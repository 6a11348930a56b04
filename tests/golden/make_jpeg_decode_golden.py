"""Writes tests/golden/jpeg_decode_cases.npz: small JPEG files written by cv2.imencode and PIL (every sampling, gray,
restart intervals, optimised Huffman tables, 16-bit quantisation tables / SOF1, a real orthomosaic layer) with what
cv2.imread returns for each in colour and in gray, so tests/test_gpu_jpeg_decode.py checks the device decoder where
OpenCV is not installed, and tests/test_jpeg_decode_cpu.py checks the fixture against live OpenCV where it is.

    python tests/golden/make_jpeg_decode_golden.py        (OpenCV 4.13, libjpeg-turbo 3.1.2; Pillow)"""
import io
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "jpeg_decode_cases.npz")


def images():
    """[(name, image)]: seeded BGR (or gray) contents at sizes that leave every kind of partial MCU."""
    rng = np.random.default_rng(2026)
    out = []
    for h, w in ((1, 1), (7, 9), (17, 33)):
        noise = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
        g = np.add.outer(np.arange(h) * 3, np.arange(w) * 5) % 256
        grad = np.stack([g, 255 - g, (2 * g) % 256], axis=-1).astype(np.uint8)
        checker = np.where((np.add.outer(np.arange(h), np.arange(w)) & 1)[:, :, None] == 0, 255, 0) * np.ones(3, int)
        out += [("noise_%dx%d" % (h, w), noise), ("gradient_%dx%d" % (h, w), grad),
                ("checker_%dx%d" % (h, w), checker.astype(np.uint8)), ("gray_%dx%d" % (h, w), noise[:, :, 1].copy())]
    z = np.load(os.path.join(HERE, "ortho_color_96x80.npz"))
    packed = z["out"].astype(np.uint32)
    bgr = np.stack([packed & 255, (packed >> 8) & 255, (packed >> 16) & 255], -1).astype(np.uint8)
    out.append(("ortho_40x34", np.ascontiguousarray(bgr[30:70, 20:54])))
    return out


def files():
    """[(name, bytes)]: each image through the encoders and settings the decoder supports."""
    import cv2
    from PIL import Image
    samp = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    out = []
    for name, img in images():
        for k, (q, s, rst, opt) in enumerate(((95, "420", 0, 0), (50, "422", 3, 0), (100, "444", 1, 1), (10, "420", 8, 1))):
            params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_OPTIMIZE, opt]
            if img.ndim == 3:
                params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp[s]]
            ok, b = cv2.imencode(".jpg", img, params)
            assert ok
            out.append(("cv2_%s_%d" % (name, k), b.tobytes()))
        pil = Image.fromarray(img[:, :, ::-1] if img.ndim == 3 else img)
        for k, kw in enumerate((dict(quality=75, subsampling=2, optimize=True), dict(quality=90, subsampling=1),
                                dict(qtables=[[300] * 64, [1000] * 64], subsampling=0))):  # 16-bit DQT: SOF1
            bio = io.BytesIO()
            pil.save(bio, "JPEG", **kw)
            out.append(("pil_%s_%d" % (name, k), bio.getvalue()))
    return out


def decode_all():
    import cv2
    res = {}
    for k, (name, b) in enumerate(files()):
        a = np.frombuffer(b, np.uint8)
        res["file_%d" % k] = a
        res["bgr_%d" % k] = cv2.imdecode(a, cv2.IMREAD_COLOR)
        res["gray_%d" % k] = cv2.imdecode(a, cv2.IMREAD_GRAYSCALE)
    return res


if __name__ == "__main__":
    np.savez_compressed(OUT, **decode_all())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
