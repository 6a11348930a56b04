"""The MUFU-seeded reciprocals of csrc/approx_math.h, swept on the device over their whole domains through the test
probe tests/cuda/libamb_approx_probe.so (tests/cuda/approx_probe.cu, built by __graft_entry__.build()):

  * rcp_f32, every positive float whose reciprocal is normal, against __frcp_rn: the 2^-23 relative error the FP32
    gather's weights and its height bound assume (DESIGN.md §4.1), and the factor that bound carries for it;
  * rsqrt_f32, every positive normal float, against 1/sqrt in double: the slack of the per-neighbour height bound,
    rsqrt_f32(d2) (1 + kRsqrtSlackUlps u) >= sqrt(rcp_f32(d2)), decided exactly for every d2;
  * fast_rcp, every high word of its domain [2^-1022, 2^1022) (the seed reads the high word only) with three low words
    each, against __drcp_rn: within 1 ulp; and, input by input, the subnormals (never below 2^1022, which the FP64
    gather's hand-over relies on), 2^-1022 and the doubles near DBL_MAX, printed as a table.

Each sweep prints its largest error, its count of results that are not correctly rounded and its time."""
import ctypes as C
import math
import os
import struct
import time

import numpy as np
import pytest

from common import ROOT

PROBE = os.path.join(ROOT, "tests", "cuda", "libamb_approx_probe.so")
U = 2.0 ** -24   # unit roundoff of float32


class ProbeResult(C.Structure):
    _fields_ = [("max_err", C.c_double), ("aux", C.c_double), ("n_not_rn", C.c_uint64), ("n_bad", C.c_uint64),
                ("first_bad", C.c_uint64)]


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(PROBE):   # a GPU run without the probe is a broken build, not a skip
        pytest.fail("%s is missing: __graft_entry__.build() compiles it" % PROBE)
    L = C.CDLL(PROBE)
    for name in ("amb_probe_rcp_f32", "amb_probe_rsqrt_f32", "amb_probe_fast_rcp"):
        getattr(L, name).argtypes = [C.c_uint32, C.c_uint32, C.POINTER(ProbeResult), C.POINTER(C.c_float)]
        getattr(L, name).restype = C.c_int
    L.amb_probe_values.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int]
    L.amb_probe_values.restype = C.c_int
    L.amb_probe_constants.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.amb_probe_constants.restype = None
    return L


def sweep(fn, lo, hi, what):
    r, ms = ProbeResult(), C.c_float()
    t0 = time.perf_counter()
    st = fn(lo, hi, C.byref(r), C.byref(ms))
    wall = time.perf_counter() - t0
    assert st == 0, "CUDA error %d" % st
    print("%s: max error %.4g, %d not correctly rounded, %d breaking the claim; kernel %.1f ms, call %.1f ms"
          % (what, r.max_err, r.n_not_rn, r.n_bad, ms.value, wall * 1e3))
    return r


def values(probe, which, xs):
    x = (C.c_double * len(xs))(*xs)
    y = (C.c_double * len(xs))()
    assert probe.amb_probe_values(which, x, y, len(xs)) == 0
    return list(y)


def constants(probe):
    slack, factor = C.c_float(), C.c_float()
    probe.amb_probe_constants(C.byref(slack), C.byref(factor))
    return slack.value, factor.value


def f32_bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f32(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


F32_MIN_NORMAL, F32_MAX = 0x00800000, 0x7F7FFFFF
F32_2P126 = f32_bits(2.0 ** 126)   # above it, 1/x is subnormal and rcp.approx.ftz flushes it to 0


@pytest.mark.gpu
def test_rcp_f32_is_within_the_relative_error_the_height_bound_assumes(probe):
    r = sweep(probe.amb_probe_rcp_f32, F32_MIN_NORMAL, F32_2P126, "rcp_f32 on [2^-126, 2^126], error in u")
    assert r.n_bad == 0, "first x with |rcp_f32(x) x - 1| > 2^-23: %r" % f32(r.first_bad)
    rel = r.max_err * U
    _, factor = constants(probe)
    # E's own evaluation: three rcp_f32 among a dozen rounded float32 operations, all inside the factor
    assert (1.0 + rel) ** 3 * (1.0 + U) ** 12 - 1.0 < factor - 1.0, factor
    # the tile form's r = x rcp_f32(c) (1 - 1e-5) (two roundings) must not exceed x / c
    assert (1.0 + rel) * (1.0 - 1e-5) * (1.0 + U) ** 2 <= 1.0
    # beyond 2^126 the reciprocal is subnormal: flushed to 0 (no caller divides by such a float)
    top = sweep(probe.amb_probe_rcp_f32, F32_2P126 + 1, F32_MAX, "rcp_f32 on (2^126, FLT_MAX]")
    assert top.n_bad == F32_MAX - F32_2P126
    assert values(probe, 1, [f32(F32_2P126 + 1), 1e-40, 2.0 ** -149]) == [0.0, math.inf, math.inf]


@pytest.mark.gpu
def test_rsqrt_f32_times_its_slack_bounds_the_square_root_of_every_weight(probe):
    slack, _ = constants(probe)
    r = sweep(probe.amb_probe_rsqrt_f32, F32_MIN_NORMAL, F32_MAX, "rsqrt_f32 on every positive normal float, in u")
    print("sqrt(rcp_f32(d2)) / rsqrt_f32(d2) - 1 <= %.4g u (slack %g u)" % (r.aux, slack))
    assert r.n_bad == 0, "first d2 with rsqrt_f32(d2) (1 + %g u) < sqrt(rcp_f32(d2)): %r" % (slack, f32(r.first_bad))
    assert r.max_err <= 4.0   # "~2 ulp"
    assert r.aux <= 5.0       # the header's sqrt(w) <= (1 + 5u) rsqrt_f32(d2); the other 3u round t
    assert values(probe, 2, [1e-40]) == [math.inf]


@pytest.mark.gpu
def test_fast_rcp_is_within_one_ulp_on_its_domain(probe):
    r = sweep(probe.amb_probe_fast_rcp, 0x00100000, 0x7FCFFFFF, "fast_rcp on [2^-1022, 2^1022), high words x 3, in ulp")
    assert r.n_bad == 0, "first x with fast_rcp(x) more than 1 ulp from 1/x: %r" % f64(r.first_bad)
    assert r.max_err <= 1.0


FAST_RCP_EDGES = [
    ("2^-1074 (smallest subnormal)", 2.0 ** -1074),
    ("4.9e-309 (1/x overflows)", 4.9e-309),
    ("2^-1024 (1/x = 2^1024 overflows)", 2.0 ** -1024),
    ("2^-1024 + 2^-1074 (smallest x with a finite 1/x)", 2.0 ** -1024 + 2.0 ** -1074),
    ("2^-1023", 2.0 ** -1023),
    ("largest subnormal", f64(0x000FFFFFFFFFFFFF)),
    ("2^-1022 (smallest normal)", 2.0 ** -1022),
    ("2^-1022 + 1 ulp", f64(0x0010000000000001)),
    ("2^1022 - 1 ulp", f64(0x7FCFFFFFFFFFFFFF)),
    ("2^1022 (1/x = 2^-1022)", 2.0 ** 1022),
    ("2^1022 + 1 ulp (1/x subnormal)", f64(0x7FD0000000000001)),
    ("2^1023", 2.0 ** 1023),
    ("DBL_MAX", f64(0x7FEFFFFFFFFFFFFF)),
]


@pytest.mark.gpu
def test_fast_rcp_at_subnormals_the_smallest_normal_and_near_dbl_max(probe):
    """The table of fast_rcp at the ends of the double range (approx_math.h documents it).  Asserted: a subnormal gives
    NaN or at least 2^1022, never a plausible weight, so the FP64 gather hands its cell to the exact kernel; the ends
    of the domain are within 1 ulp."""
    got = values(probe, 0, [x for _, x in FAST_RCP_EDGES])
    rows, wrong = [], []
    with np.errstate(over="ignore", divide="ignore"):
        for (name, x), y in zip(FAST_RCP_EDGES, got):
            want = float(np.float64(1.0) / np.float64(x))
            rows.append("%-50s x = %-24r fast_rcp = %-24r 1/x = %r" % (name, x, y, want))
            ulps = abs(np.float64(y).view(np.int64) - np.float64(want).view(np.int64)) if math.isfinite(y) else None
            if x < 2.0 ** -1022 and y < 2.0 ** 1022:
                wrong.append(name)
            if 2.0 ** -1022 <= x < 2.0 ** 1022 and not (ulps is not None and ulps <= 1):
                wrong.append(name)
    print("\n".join(rows))
    assert not wrong, wrong
