"""Writes tests/golden/jpeg_extreme_cases.npz: the files of tests/jpeg_synth.py's case set (coefficients no encoder
writes: 16-bit IDCT lanes, extreme Huffman categories, 16-bit codes, DC predictors past int16, scans that never
self-synchronise) with what cv2.imread returns for each in colour and in gray.  Where the IDCT's 16-bit lanes wrap,
the decode is that of libjpeg-turbo's x86 SIMD code; an ARM or non-SIMD build may round differently, so the device is
held to this fixture (made on x86) and to the restatement in tests/jpeg_synth.py, not to the live cv2 of its host.

    python tests/golden/make_jpeg_extreme_golden.py        (x86-64, OpenCV 4.13, libjpeg-turbo 3.1.2)"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_synth  # noqa: E402

OUT = os.path.join(HERE, "jpeg_extreme_cases.npz")


def decode_all():
    import cv2
    res = {}
    for name, b in jpeg_synth.cases():
        a = np.frombuffer(b, np.uint8)
        res["file_" + name] = a
        res["bgr_" + name] = cv2.imdecode(a, cv2.IMREAD_COLOR)
        res["gray_" + name] = cv2.imdecode(a, cv2.IMREAD_GRAYSCALE)
    return res


if __name__ == "__main__":
    np.savez_compressed(OUT, **decode_all())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
