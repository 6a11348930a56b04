"""Write tests/golden/utm_reference.json: the reference's own UTM::UTMtoLL (gps-conversions.h, built from the reference
sources by oracle/refsrc_glue_utm.cc) at fixed UTM positions, so that test_lonlat_import_cpu.py compares the order-6
series oracle with it without the reference or the build.

    python tests/golden/make_utm_golden.py [REF_ROOT]

The bound stored with the points is the largest distance measured between the two, rounded up; DESIGN.md states it."""
import ctypes as C
import json
import os
import subprocess
import sys

import mpmath as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
import utm_oracle as U  # noqa: E402

POINTS = [  # (easting, northing, epsg)
    (464980.0, 5272260.0, 32632),      # the reference's Rafz demo
    (500000.0, 5272260.0, 32632), (465000.0, 5272000.0, 32632), (400000.0, 5300000.0, 32632),
    (166000.0, 5262000.0, 32632),      # 334 km west of the central meridian at 47.5 N
    (834000.0, 5262000.0, 32632), (725000.0, 5262000.0, 32632), (955000.0, 5280000.0, 32632),
    (500000.0, 0.0, 32631), (620000.0, 50000.0, 32631), (300000.0, 1000.0, 32631),
    (500000.0, 8000000.0, 32633),      # 72 N
    (300000.0, 8000000.0, 32633), (600000.0, 9300000.0, 32633), (700000.0, 6600000.0, 32610),
    (380000.0, 9990000.0, 32733), (401000.0, 7300000.0, 32733), (620000.0, 6000000.0, 32756),
    (200000.0, 4000000.0, 32718), (500000.0, 5000000.0, 32760), (800000.0, 3000000.0, 32601),
    (250000.0, 2500000.0, 32645), (550000.0, 4400000.0, 32717), (450000.0, 1200000.0, 32738),
]


def build(ref_root):
    out = os.path.join(ROOT, "oracle", "_ref", "libamb_refsrc_utm.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-std=c++11", "-pthread", "-ffp-contract=off", "-fPIC", "-fvisibility=hidden", "-shared",
                           "-I" + os.path.join(ref_root, "aerial_mapper_thirdparty", "include"),
                           os.path.join(ROOT, "oracle", "refsrc_glue_utm.cc"), "-o", out])
    return out


def main():
    ref_root = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    lib = C.CDLL(build(ref_root))
    lib.ambo_ref_utm_to_ll.argtypes = [C.c_double, C.c_double, C.c_char_p, C.POINTER(C.c_double),
                                       C.POINTER(C.c_double)]
    points, worst = [], 0.0
    for e, n, epsg in POINTS:
        zone = ("%d%s" % (epsg % 100, "N" if epsg < 32700 else "M")).encode()
        lat, lon = C.c_double(), C.c_double()
        lib.ambo_ref_utm_to_ll(n, e, zone, C.byref(lat), C.byref(lon))
        olon, olat = U.inverse(e, n, epsg)
        d = float(mp.hypot((lat.value - olat) * 111320, (lon.value - olon) * 111320 * mp.cos(mp.radians(olat))))
        worst = max(worst, d)
        points.append({"easting": e, "northing": n, "epsg": epsg, "lat": lat.value, "lon": lon.value})
        print("%9.1f %10.1f %d  ref - oracle %.3g m" % (e, n, epsg, d))
    bound = float("%.2g" % (worst * 1.5))
    with open(os.path.join(HERE, "utm_reference.json"), "w") as f:
        json.dump({"source": "UTM::UTMtoLL, aerial_mapper_thirdparty/.../gps-conversions.h", "bound_m": bound,
                   "points": points}, f, indent=1)
    print("largest %.3g m, bound %.2g m" % (worst, bound))


if __name__ == "__main__":
    main()
