"""Memory-safety pass over the longitude/latitude import (csrc/raster_import.cu, raster_lonlat_kernel): the emulated
library (tests/emu) rebuilt with AddressSanitizer, as tools/emu_asan_geotiff_inflate.py does, driven through host bands
and TIFFs whose window sits at the raster's edges and corners (one-pixel rasters, rasters that end inside the map on
every side, rasters that barely touch it) with both methods, so that a tap past the copied window or a window past the
raster would be reported.  The host band of every call is allocated to its exact size.

    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 \\
        python tools/emu_asan_lonlat_import.py
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
ASAN_LIB = "/tmp/libamb_emu_lonlat_asan.so"
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
import test_gpu_lonlat_import as T  # noqa: E402

counts = {}
E = _lib.LAYER_ID["elevation"]
rows, cols = 64, 24
for centre, epsg, res in [(T.RAFZ, 32632, 7.0), ((725000.0, 5262000.0), 32632, 40.0), ((620000.0, 0.0), 32631, 30.0),
                          ((380000.0, 10000000.0), 32733, 30.0)]:
    gm = T.lonlat_map(rows, cols, res, centre)
    ctx = gm.context()
    lon, lat = T.positions(gm, epsg)
    west, east, south, north = lon.min(), lon.max(), lat.min(), lat.max()
    for step in ((east - west) / 7.0, (east - west) / 61.0, (east - west) / 400.0):
        # rasters ending at each fraction of the map on each side, and one-pixel rasters at the corners
        for fw in (-0.5, 0.0, 0.37, 0.999, 1.0):
            for fn in (1.5, 1.0, 0.61, 0.001, 0.0):
                for w, h in ((1, 1), (2, 3), (int((east - west) / step) + 2, int((north - south) / step) + 2)):
                    gt = (west + fw * (east - west), step, 0.0, south + fn * (north - south), 0.0, -step)
                    band = T.terrain(h, w, seed=w + h)
                    exact = np.empty(band.size, np.float32)   # no slack after the band for ASan to miss
                    exact[:] = band.ravel()
                    for rs in (0, 1):
                        st = L.amb_import_raster_lonlat(ctx, E, exact.ctypes.data, w, h, 4 * w, (C.c_double * 6)(*gt),
                                                        0, 0.0, rs, epsg)
                        counts[st] = counts.get(st, 0) + 1
                        b = T.lonlat_tiff(band, gt, ("tiles", 16, 16))
                        f = T.HostFile(b)
                        layout = io.tiff_layout(b).c_layout()
                        st = L.amb_import_tiff_lonlat(ctx, E, C.c_void_p(f.ptr), f.size, C.byref(layout),
                                                      (C.c_double * 6)(*gt), 0, 0.0, rs, epsg)
                        counts[st] = counts.get(st, 0) + 1
    gm.sync()
print("statuses:", counts)
assert set(counts) == {0}, counts
print("ASan: clean")
