"""Writes tests/golden/jpeg_cases.npz: seeded 8-bit images, their encoder parameters and cv2.imencode's bytes for them,
so the byte comparison of tests/test_gpu_jpeg_encode.py also runs where OpenCV is not installed.

    python tests/golden/make_jpeg_golden.py        (OpenCV 4.13, libjpeg-turbo 3.1.2)"""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "jpeg_cases.npz")


def cases():
    """[(image, (quality, sampling, restart_interval))]: every mode, odd sizes, noise / checkerboard / gradient."""
    rng = np.random.default_rng(2026)
    out = []
    for channels in (1, 3):
        for sampling in (("420",) if channels == 1 else ("420", "444")):
            for (h, w), quality, restart in (((1, 1), 95, 0), ((7, 9), 1, 1), ((17, 33), 100, 3), ((37, 53), 50, 8),
                                             ((64, 9), 75, 1000), ((33, 17), 10, 2)):
                shape = (h, w) if channels == 1 else (h, w, 3)
                for kind in range(3):
                    if kind == 0:
                        img = rng.integers(0, 256, shape).astype(np.uint8)
                    elif kind == 1:
                        img = np.where(rng.random(shape) < 0.5, 0, 255).astype(np.uint8)
                    else:
                        g = np.add.outer(np.arange(h) * 3, np.arange(w) * 5) % 256
                        img = (g if channels == 1 else np.stack([g, 255 - g, (2 * g) % 256], axis=-1)).astype(np.uint8)
                    out.append((img, (quality, sampling, restart)))
    return out


def encode_all():
    import cv2
    res = {}
    for k, (img, (quality, sampling, restart)) in enumerate(cases()):
        params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
        if img.ndim == 3:
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == "420"
                       else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
        ok, b = cv2.imencode(".jpg", img, params)
        assert ok
        res["jpeg_%d" % k] = np.frombuffer(b.tobytes(), np.uint8)
    return res


if __name__ == "__main__":
    np.savez_compressed(OUT, **encode_all())
    print("wrote", OUT)
