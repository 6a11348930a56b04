"""Writes tests/golden/cog_jpeg_cases.npz: the JPEG COG tiles OpenCV's encoder gives for a small raster (56 x 40, tiles
of 16, three levels), gray, 4:2:0 and 4:4:4 at qualities 50 and 75, split into the tables stream and the abbreviated
tile streams as tests/test_cog_jpeg_cpu.py does; the CPU tests use it where OpenCV is not installed.
Run from the repository root: python tests/golden/make_cog_jpeg_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import test_cog_jpeg_cpu as t  # noqa: E402

assert t.cv2 is not None, "the fixture records OpenCV's encoder"


def main():
    rng = np.random.default_rng(11)
    yy, xx = np.mgrid[0:40, 0:56]
    base = (np.sin(xx / 5.0) * 60 + np.cos(yy / 7.0) * 50 + 120)[..., None] + rng.normal(0, 12, (40, 56, 3))
    bgr = np.clip(base + np.array([0, 30, -30]), 0, 255).astype(np.uint8)
    gray = bgr[:, :, 1].copy()
    mask = np.where((xx - 20) ** 2 + (yy - 15) ** 2 < 150, 0, 255).astype(np.uint8)
    mask[:, 50:] = 0
    out = {"bgr": bgr, "gray": gray, "mask": mask, "tile": np.int32(16)}
    for kind, (fmt, sampling) in t.KINDS.items():
        for q in t.FIXTURE_QUALITIES:
            tables, streams = t.cv2_tiles(bgr if fmt == "bgr8" else gray, fmt, 16, q, sampling)
            key = "%s_q%d" % (kind, q)
            out[key + "_tables"] = np.frombuffer(tables, np.uint8)
            out[key + "_tiles"] = np.frombuffer(b"".join(streams), np.uint8)
            out[key + "_lens"] = np.array([len(s) for s in streams], np.int64)
    np.savez_compressed(os.path.join(HERE, "cog_jpeg_cases.npz"), **out)


if __name__ == "__main__":
    main()
