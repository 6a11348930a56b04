"""Memory-safety pass over the JPEG decoder's kernel source (csrc/jpeg_decode.cu, csrc/jpeg_header.cc): the emulated
library (tests/emu) rebuilt with AddressSanitizer, as tools/emu_asan_check.py does, driven through the inputs a decoder
must survive whatever their bytes: truncated scans, flipped bits, bad and missing restart markers, overlong runs, codes
no table holds, spliced restart markers, scans shifted by 1..127 bytes, refused headers, and the orthomosaic from JPEG
files with corrupt frames.

    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 \\
        python tools/emu_asan_jpeg_decode.py
"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import numpy as np  # noqa: E402
import cv2  # noqa: E402
import build_emu  # noqa: E402
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402

build_emu.build()
ASAN_LIB = "/tmp/libamb_emu_jpeg_asan.so"
B = build_emu.OUT
subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-w", "-pthread",
                       "-fsanitize=address", "-fno-omit-frame-pointer", "-I" + os.path.join(build_emu.HERE, "include"),
                       "-I" + B, "-I" + build_emu.CSRC, "-I" + os.path.join(ROOT, "include")] +
                      sorted(os.path.join(B, f) for f in os.listdir(B) if f.endswith("_emu.cc")) +
                      sorted(os.path.join(build_emu.CSRC, f) for f in os.listdir(build_emu.CSRC) if f.endswith(".cc")) +
                      [os.path.join(build_emu.HERE, "emu_runtime.cc"), "-ldl", "-o", ASAN_LIB])
L = C.CDLL(ASAN_LIB)
for name, (restype, argtypes) in _lib.SYMBOLS.items():
    fn = getattr(L, name)
    fn.restype = restype
    fn.argtypes = argtypes
_lib._lib = L
os.environ["AMB_TEST_EMU"] = "1"   # the test helpers' device buffers are host arrays
import test_gpu_jpeg_decode as T  # noqa: E402
from test_jpeg_decode_cpu import refused_files, segment  # noqa: E402

rng = np.random.default_rng(21)
counts = {}


def run(files, channels, shapes):
    _, status, _ = T.decode(files, channels, shapes=shapes)
    for s in status:
        counts[s] = counts.get(s, 0) + 1


for s in T.SAMPLINGS:
    for restart in (0, 1, 3):
        b = T.cv2_file(T.content("smooth", 37, 53, seed=restart), 90, s, restart)
        start = segment(b, 0xDA)[1]
        cuts = [b[:k] for k in range(start, len(b), max(1, (len(b) - start) // 40))]
        flips = []
        for _ in range(40):
            a = bytearray(b)
            for _ in range(int(rng.integers(1, 4))):
                a[int(rng.integers(start, len(b)))] ^= 1 << int(rng.integers(0, 8))
            flips.append(bytes(a))
        junk = [b[:start] + bytes(rng.integers(0, 256, n).astype(np.uint8)) for n in (0, 1, 7, 300, 3000)]
        junk += [b[:p] + bytes([0xFF, 0xD0 + p % 8]) + b[p:] for p in range(start + 1, len(b) - 2, 97)
                 if b[p - 1] != 0xFF]   # restart markers spliced in
        for ch in (1, 3):
            run(cuts + flips + junk, ch, [(37, 53)] * (len(cuts) + len(flips) + len(junk)))
    print("sampling", s, counts)
shifted = T.cv2_file(T.content("smooth", 64, 96, seed=7), 95, "420", 0)
run([shifted[:2] + b"\xFF\xFE" + bytes([0, n + 2]) + bytes(n) + shifted[2:] for n in range(1, 128)], 3, [(64, 96)] * 127)
named = T.corrupt_files()
run([f for _, f in named], 3, [(8, 8) if n in ("run_past_63", "no_such_code") else (40, 56) for n, _ in named])
run([f for _, f in refused_files()], 3, [(17, 33)] * len(refused_files()))
print("decode", counts)

# the orthomosaic from JPEG files: corrupt contributing and non-contributing frames
camd, poses, files = T.ortho_case(True, 2)
far = poses[0].copy()
far[:2] += 5000.0
cut = files[0][:(segment(files[0], 0xDA)[1] + len(files[0])) // 2]
for extra, bad in ((far, cut), (poses[1], cut)):
    gm = T.new_map()
    try:
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=True), gm).process_jpeg(
            np.vstack([poses, extra]), files + [bad], gm)
        print("ortho: ok")
    except amb.AmbError as e:
        print("ortho:", e.status)
print("clean: no AddressSanitizer report above")
