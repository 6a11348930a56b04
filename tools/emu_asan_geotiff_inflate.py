"""Memory-safety pass over the TIFF chunk decoder's kernel source (csrc/deflate_decode.cu): the emulated library
(tests/emu) rebuilt with AddressSanitizer, as tools/emu_asan_check.py does, driven through the inputs an inflater must
survive whatever their bytes: truncated streams, flipped bits, junk streams, every corrupt class of the GPU tests, and
layouts inconsistent with the file (counts and offsets past its end, short uncompressed chunks, bad windows).

    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 \\
        python tools/emu_asan_geotiff_inflate.py
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
import build_emu  # noqa: E402
from aerial_mapper_b200 import _lib, io  # noqa: E402

build_emu.build()
ASAN_LIB = "/tmp/libamb_emu_inflate_asan.so"
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
import test_gpu_geotiff_inflate as T  # noqa: E402
from test_geotiff_inflate_cpu import (corrupt_streams, dynamic_stream, make_tiff, match_stream, predict,  # noqa: E402
                                      sample_raster, zstream)

rng = np.random.default_rng(31)
counts = {}


def run(data, window=None, layout=None):
    st = T.decode(data, window=window, layout=layout)[0]
    counts[st] = counts.get(st, 0) + 1


a = sample_raster(np.float32, 24, 40, seed=3)[:, :, 0]
raw = predict(a[8:16, :, None], 3)
lit = bytes(rng.integers(0, 256, 34000).astype(np.uint8))
far = match_stream([lit[:200], lit[1000:34000], (258, 32768), (258, 32767), (3, 32768), lit[:9]])[0]   # the ring
streams = [zstream(raw, lv, st) for lv in (0, 1, 6, 9) for st in (0, 1, 2, 3, 4)] + [dynamic_stream(raw[:900], d)
                                                                                    for d in ("none", "single")] + [far]
for s in streams:
    cases = [s[:k] for k in range(0, len(s), max(1, len(s) // 25))]
    for _ in range(25):
        b = bytearray(s)
        for _ in range(int(rng.integers(1, 4))):
            b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
        cases.append(bytes(b))
    cases += [s[:2] + bytes(rng.integers(0, 256, n).astype(np.uint8)) for n in (0, 1, 5, 64, 3000)]
    for bad in cases:
        run(make_tiff(a, 3, ("strips", 8), encode=lambda r, k: bad if k == 1 else zstream(r)))
for _, bad in corrupt_streams(raw):
    run(make_tiff(a, 3, ("strips", 8), encode=lambda r, k: bad if k == 1 else zstream(r)))
print("streams", counts)

good = make_tiff(a, 3, ("tiles", 16, 16))
t = io.tiff_layout(good)
for field, value in (("n_chunks", 1), ("band", 3), ("chunk_height", 0), ("sample", -1), ("tiled", 0)):
    Lc = t.c_layout()
    setattr(Lc, field, value)
    run(good, layout=Lc)
for k in range(3):
    Lc = t.c_layout()
    Lc._keep[0][k] = len(good) - 1
    run(good, layout=Lc)
    Lc = t.c_layout()
    Lc._keep[1][k] = len(good)
    run(good, layout=Lc)
run(make_tiff(a, 3, ("strips", 8), compression=1, encode=lambda r, k: r[:-3]))
for win in ((0, 25, 0, 40), (3, 3, 0, 40), (-1, 2, 0, 4), (0, 2, 39, 41)):
    run(good, window=win)
print("layouts and windows", counts)
print("clean: no AddressSanitizer report above")
