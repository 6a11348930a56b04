"""The stereo kernels through their device entry points, amb_stereo_reproject_device and amb_stereo_rectify_maps_device:
the ABI a GPU pipeline uses (disparities in HBM -> world points -> Dsm / OrthoFromPcl process_device).

  A. reprojection (csrc/stereo_kernels.cu: count, one-block scan over chunks of 1024 block counts, ordered write):
     pitched and misaligned inputs, frame sizes at the scan's edges, the capacity contract, scratch and stream,
     non-finite disparities and thresholds, the float32-overflow drop rule at its exact boundary, the argument contract.
  B. rectification maps (csrc/rectify_kernels.cu): the scalar-store kernel (odd strides, misaligned planes), row
     padding, the zero-w flag.
  C. both stages chained on the device with the DSM and OrthoFromPcl: against the oracle chain and the geometry.

Outputs are compared with the oracle (oracle/stereo_oracle.cc) bit for bit, with one exception: where an output is NaN
only its NaN-ness is compared.  IEEE 754 leaves the payload of a NaN an operation creates open, and the two sides
differ (x86 gives 0xfff8... / 0xffc00000, the GPU 0x7fff... / 0x7fffffff).

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and
they are numpy arrays.  Every buffer is filled with a canary byte first: bytes a call must not write are checked."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from common import UTM, UTM_SHIFT, ulp_diff  # noqa: E402
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
PRECISION = os.environ.get("AMB_DSM_PRECISION", "f32").lower()
MAX_ULP = 1 if PRECISION == "f64" else 4
CANARY = 0xA5
THREADS = 256          # kRpThreads: pixels per block of the count and write kernels
SCAN_CHUNK = 1024      # block counts per round of reproject_scan_kernel
F32_MAX = float(np.finfo(np.float32).max)
F32_MIN_SUB = float(np.nextafter(np.float32(0), np.float32(1)))


# ---- device buffers ---------------------------------------------------------------------------------------------------
def sync():
    if not EMULATED:
        import torch
        torch.cuda.synchronize()


class Dev(object):
    """`nbytes` of device memory at a 64-byte aligned .ptr, followed by a 64-byte tail; every byte starts as CANARY."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes) + 64
        n = self.nbytes + 64
        if EMULATED:
            self.raw = np.full(n, CANARY, np.uint8)
            p = self.raw.ctypes.data
        else:
            import torch
            self.raw = torch.full((n,), CANARY, dtype=torch.uint8, device="cuda:0")
            p = self.raw.data_ptr()
        self.base = (-p) % 64
        self.ptr = p + self.base

    def put(self, a, off=0):
        b = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
        lo = self.base + off
        assert off + len(b) <= self.nbytes
        if EMULATED:
            self.raw[lo:lo + len(b)] = b
        else:
            import torch
            self.raw[lo:lo + len(b)].copy_(torch.from_numpy(b.copy()))
        return self

    def get(self, dtype=np.uint8, off=0, count=None):
        """`count` elements of `dtype` at byte `off` (default: to the end of the tail)."""
        size = np.dtype(dtype).itemsize
        count = (self.nbytes - off) // size if count is None else int(count)
        seg = self.raw[self.base + off:self.base + off + count * size]
        return (seg.copy() if EMULATED else seg.cpu().numpy()).view(dtype)


def ptr(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data


def stream_handles():
    """The NULL stream and a torch stream (NULL under emulation: there streams are no-ops)."""
    if EMULATED:
        return [("null", None, None), ("torch", None, None)]
    import torch
    s = torch.cuda.Stream(device=0)
    return [("null", None, None), ("torch", s.cuda_stream, s)]


def same(got, want):
    """Bit for bit, except that a NaN only has to be a NaN (its payload is open, see the module docstring)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return False
    gn, wn = np.isnan(got), np.isnan(want)
    u = np.uint64 if got.dtype.itemsize == 8 else np.uint32
    return np.array_equal(gn, wn) and np.array_equal(np.ascontiguousarray(got[~gn]).view(u),
                                                     np.ascontiguousarray(want[~wn]).view(u))


def untouched(words, written, what):
    """Every byte of `words` outside the mask `written` still holds the canary."""
    b = np.ascontiguousarray(words).view(np.uint8).reshape(len(words), -1)
    bad = np.flatnonzero((b[~written] != CANARY).any(axis=1))
    assert len(bad) == 0, "%s: %d elements outside the output were written" % (what, len(bad))


# ---- A. reprojection --------------------------------------------------------------------------------------------------
def camera(h, w, baseline=0.37):
    """k4 = (fx, fy, cx, cy), baseline, R_G_C (row-major), t_G_C1 of a rectified frame at map scale."""
    from scipy.spatial.transform import Rotation
    k4 = np.array([1200.5, 1190.25, w / 2 + 0.3, h / 2 - 0.7])
    R = np.ascontiguousarray(Rotation.from_euler("xyz", [3.05, 0.04, -0.6]).as_matrix().reshape(9))
    return k4, float(baseline), R, np.array([464000.5, 5248000.25, 820.0])


FILLS = ("all", "none", "last", "random")


def frame(h, w, fill, seed=0):
    rng = np.random.default_rng([h, w, FILLS.index(fill), seed])
    img = rng.integers(0, 256, (h, w), dtype=np.uint8)
    if fill == "all":
        disp = rng.uniform(1.5, 40.0, (h, w)).astype(np.float32)
    elif fill in ("none", "last"):       # the block matcher's invalid marker and exactly kMaxInvalidDisparity (strict >)
        disp = np.where(rng.random((h, w)) < 0.5, np.float32(-1.0), np.float32(1.0)).astype(np.float32)
        if fill == "last":
            disp[-1, -1] = 7.25
    else:
        disp = rng.uniform(-2.0, 40.0, (h, w)).astype(np.float32)
        disp[rng.random((h, w)) < 0.2] = -1.0
        disp[rng.random((h, w)) < 0.05] = 1.0
    return disp, img


def padded(a, stride, fill):
    out = np.full((a.shape[0], stride), fill, a.dtype)
    out[:, :a.shape[1]] = a
    return out


def blocks_of(h, w):
    return -(-(h * w) // THREADS)


def reproject_device(disp, img, cam, thr=1.0, cap=None, dpad=0, ipad=0, dshift=0, stream=None, launches=1):
    """amb_stereo_reproject_device on device copies of (disp, img): disparity rows `dpad` floats longer than the frame
    (the padding holds 20.0, a valid disparity), image rows `ipad` bytes longer (padding 200), the disparity buffer
    starting `dshift` floats into its allocation.  Outputs of capacity + 16 points, scratch of exactly ceil(W*H/256)
    words and the count start as canaries.  `launches` > 1: back-to-back calls on the same scratch, each into its own
    outputs.  Returns the status and, per launch, the count and the raw output buffers."""
    h, w = disp.shape
    k4, b, R, t = cam
    ds, ist = w + dpad, w + ipad
    cap = h * w if cap is None else int(cap)
    nb = blocks_of(h, w)
    D = Dev(4 * (h * ds + dshift)).put(padded(disp, ds, np.float32(20.0)), off=4 * dshift)
    I = Dev(h * ist).put(padded(img, ist, np.uint8(200)))
    S = Dev(4 * nb)
    outs = [(Dev(24 * (cap + 16)), Dev(4 * (cap + 16)), Dev(8)) for _ in range(launches)]
    sync()
    for X, N, K in outs:
        st = amb.lib().amb_stereo_reproject_device(0, stream, D.ptr + 4 * dshift, ds, I.ptr, ist, w, h, ptr(k4), b,
                                                   ptr(R), ptr(t), float(thr), X.ptr, N.ptr, cap, S.ptr, K.ptr)
        if st != 0:
            return st, None
    sync()
    scratch = S.get(np.uint32)
    return 0, [dict(count=int(K.get(np.uint64, count=1)[0]), xyz=X.get(np.float64), inten=N.get(np.int32), cap=cap,
                    scratch=scratch) for X, N, K in outs]


def check_outputs(r, want_xyz, want_inten, what=""):
    """The first min(count, capacity) points equal the oracle's; every byte beyond them is still the canary."""
    n, cap = len(want_xyz), r["cap"]
    assert r["count"] == n, "%s: *d_count = %d, the oracle counts %d" % (what, r["count"], n)
    k = min(n, cap)
    xyz = r["xyz"]
    assert same(xyz[:3 * k].reshape(-1, 3), want_xyz[:k]), what + ": points differ from the oracle"
    assert np.array_equal(r["inten"][:k], want_inten[:k]), what + ": intensities differ from the oracle"
    written = np.zeros(len(xyz), bool)
    written[:3 * k] = True
    untouched(xyz, written, what + ": d_out_xyz")
    written = np.zeros(len(r["inten"]), bool)
    written[:k] = True
    untouched(r["inten"], written, what + ": d_out_intensity")


def check_scratch(r, disp, thr):
    """The scratch holds the exclusive scan of the per-block valid counts, and nothing beyond its last word changed.
    (The frames of these tests overflow no depth: a pixel is valid iff its disparity is > thr.)"""
    h, w = disp.shape
    nb = blocks_of(h, w)
    valid = np.flatnonzero(disp.ravel() > np.float32(thr))
    per_block = np.bincount(valid // THREADS, minlength=nb).astype(np.int64)
    assert per_block.sum() == r["count"]
    sc = r["scratch"]
    assert np.array_equal(sc[:nb].astype(np.int64), np.cumsum(per_block) - per_block), "block offsets differ"
    untouched(sc, np.arange(len(sc)) < nb, "d_block_scratch")


def oracle(disp, img, cam, thr=1.0):
    k4, b, R, t = cam
    st, xyz, inten = po.stereo_reproject(disp, img, k4, b, R.reshape(3, 3), t, max_invalid_disparity=thr)
    assert st == 0
    return xyz, inten


# 1. pitched and misaligned inputs
@pytest.mark.parametrize("h,w,dshift", [(37, 53, 1), (300, 1000, 1), (1, 7, 1), (64, 300, 0)])
def test_reproject_pitched_and_misaligned_inputs(h, w, dshift):
    disp, img = frame(h, w, "random", seed=1)
    cam = camera(h, w)
    xyz, inten = oracle(disp, img, cam)
    assert len(xyz) > 0
    st, res = reproject_device(disp, img, cam, dpad=5, ipad=3, dshift=dshift)
    assert st == 0
    check_outputs(res[0], xyz, inten, "disparity stride W + 5, image stride W + 3")
    check_scratch(res[0], disp, 1.0)


# 2. frame sizes at the scan's edges: ceil(W*H/256) block counts, scanned in chunks of 1024
SCAN_SHAPES = [(1, 1), (16, 16), (255, 1), (341, 768), (1, 261887), (512, 512), (1, 261889), (5, 52429), (512, 1024),
               (524287, 1), (3, 174763)]


def test_scan_shapes_cover_the_chunk_edges():
    blocks = {blocks_of(h, w) for h, w in SCAN_SHAPES}
    assert {1, SCAN_CHUNK - 1, SCAN_CHUNK, SCAN_CHUNK + 1, 2 * SCAN_CHUNK, 2 * SCAN_CHUNK + 1} <= blocks
    assert {0, 1, THREADS - 1} <= {h * w % THREADS for h, w in SCAN_SHAPES}
    assert {(1, 1)} < set(SCAN_SHAPES) and any(h == 1 and w > 1 for h, w in SCAN_SHAPES) and \
        any(w == 1 and h > 1 for h, w in SCAN_SHAPES)


def check_all_fills(h, w):
    cam = camera(h, w)
    for fill in FILLS:
        disp, img = frame(h, w, fill)
        xyz, inten = oracle(disp, img, cam)
        assert len(xyz) == {"all": h * w, "none": 0, "last": 1}.get(fill, len(xyz))
        st, res = reproject_device(disp, img, cam)
        assert st == 0
        check_outputs(res[0], xyz, inten, "%dx%d %s" % (h, w, fill))
        check_scratch(res[0], disp, 1.0)


@pytest.mark.parametrize("h,w", SCAN_SHAPES, ids=["%dx%d" % s for s in SCAN_SHAPES])
def test_reproject_frame_sizes_at_the_scan_edges(h, w):
    check_all_fills(h, w)


@pytest.mark.skipif(EMULATED, reason="12 M pixels: minutes on the emulated kernels")
def test_reproject_large_benchmark_camera_frame():
    # the benchmark cameras' 4000 x 3000 frames: 46875 blocks, 46 chunks of the scan
    assert blocks_of(3000, 4000) == 46875
    check_all_fills(3000, 4000)


# 3. the capacity contract
@pytest.mark.parametrize("h,w", [(61, 83), (300, 1000)])
def test_reproject_capacity_contract(h, w):
    disp, img = frame(h, w, "random", seed=3)
    cam = camera(h, w)
    k4, b, R, t = cam
    xyz, inten = oracle(disp, img, cam)
    n = len(xyz)
    assert n > 2
    for cap in (0, 1, n - 1, n, n + 7):
        st, res = reproject_device(disp, img, cam, cap=cap)
        assert st == 0
        check_outputs(res[0], xyz, inten, "capacity %d of %d" % (cap, n))
        # the host entry: the same count in out_count, the same rows, nothing written beyond them
        hx = np.full(3 * (cap + 16), np.frombuffer(bytes([CANARY]) * 8, np.float64)[0])
        hi = np.full(cap + 16, np.frombuffer(bytes([CANARY]) * 4, np.int32)[0])
        cnt = C.c_size_t(0xDEADBEEF)
        st = amb.lib().amb_stereo_reproject(0, ptr(disp), w, ptr(img), w, w, h, ptr(k4), b, ptr(R), ptr(t), 1.0,
                                            ptr(hx), ptr(hi), cap, C.byref(cnt))
        assert st == 0 and cnt.value == n
        check_outputs(dict(count=cnt.value, xyz=hx, inten=hi, cap=cap), xyz, inten, "host entry, capacity %d" % cap)


# 4. scratch and stream
@pytest.mark.parametrize("h,w", [(300, 1000), (512, 1024)])
def test_reproject_scratch_and_streams(h, w):
    disp, img = frame(h, w, "random", seed=4)
    cam = camera(h, w)
    xyz, inten = oracle(disp, img, cam)
    for name, handle, _keep in stream_handles():
        st, res = reproject_device(disp, img, cam, stream=handle, launches=2)
        assert st == 0, name
        for k, r in enumerate(res):
            check_outputs(r, xyz, inten, "%s stream, launch %d" % (name, k))
        check_scratch(res[1], disp, 1.0)
        assert np.array_equal(res[0]["xyz"].view(np.uint64), res[1]["xyz"].view(np.uint64))


# 5. non-finite and boundary values
SPECIALS = [np.nan, np.inf, -np.inf, 0.0, -0.0, F32_MIN_SUB, -F32_MIN_SUB, F32_MAX, -F32_MAX, 1.0, -1.0, 0.5, -0.5,
            2.0, 37.0]
THRESHOLDS = [1.0, 0.0, -1.0, -np.inf, np.inf, np.nan]


def special_frame(thr):
    """Every special value (and thr, its float successor and predecessor) in every row and in the column u = cx; the
    row v = cy holds them all too: there (u - cx) or (fx/fy v - cy fx/fy) is exactly 0, so d = +-0 gives 0/0."""
    vals = list(SPECIALS)
    if np.isfinite(thr):
        f = np.float32(thr)
        vals += [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    vals = np.array(vals, np.float32)
    L = len(vals)
    h, w = L, 41
    v, u = np.mgrid[0:h, 0:w]
    disp = vals[(u + v) % L]
    img = ((u * 7 + v * 3) % 256).astype(np.uint8)
    k4 = np.array([1200.5, 1190.25, 20.0, 4.0])
    return disp, img, k4


@pytest.mark.parametrize("baseline", [0.37, -0.37])
@pytest.mark.parametrize("thr", THRESHOLDS, ids=["thr=%s" % t for t in THRESHOLDS])
def test_reproject_non_finite_and_boundary_disparities(thr, baseline):
    disp, img, k4 = special_frame(thr)
    h, w = disp.shape
    _, _, R, t = camera(h, w)
    cam = (k4, baseline, R, t)
    xyz, inten = oracle(disp, img, cam, thr)
    st, res = reproject_device(disp, img, cam, thr=thr, dpad=5, ipad=3, dshift=1)
    assert st == 0
    check_outputs(res[0], xyz, inten, "thr %s, baseline %s" % (thr, baseline))
    with np.errstate(invalid="ignore"):
        n_valid = int((disp > np.float32(thr)).sum())
    if np.isnan(thr) or thr == np.inf:
        assert len(xyz) == 0                          # nothing is > NaN or > +inf
    else:
        assert 0 < len(xyz) <= n_valid
    if thr < 0:                                       # zero disparities are valid: 0/0 at u = cx, inf - inf elsewhere
        assert np.isnan(xyz).any()
    if thr == 1.0 and po.have_refsrc_stereo():        # the reference's own densifier (kMaxInvalidDisparity = 1)
        st2, rxyz, rinten = po.refsrc_stereo_reproject(disp, img, k4, baseline, R.reshape(3, 3), t)
        assert st2 == 0 and same(rxyz, xyz) and np.array_equal(rinten, inten)
        assert same(res[0]["xyz"][:3 * len(xyz)].reshape(-1, 3), rxyz)


# 6. the float32-overflow drop rule at its exact boundary
MID = F32_MAX + 2.0 ** 103      # halfway between FLT_MAX and 2^128: rounds to even, i.e. to 2^128 = inf


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_reproject_float32_overflow_drop_rule_at_its_boundary(sign):
    with np.errstate(over="ignore"):
        assert np.isinf(np.float32(MID)) and np.float32(np.nextafter(MID, 0.0)) == np.float32(F32_MAX)
    h, w = 23, 67
    disp, img = frame(h, w, "random", seed=6)
    k4, b, R, t = camera(h, w)
    R = R.copy()
    R[6:] = 0.0                          # Z = ((0 x1 + 0 y1) + 0 z1) + t[2] = t[2] exactly
    n_valid = int((disp > 1.0).sum())
    for tz, kept in ((F32_MAX, True), (MID, False), (np.nextafter(MID, 0.0), True), (2.0 ** 128, False)):
        cam = (k4, b, R, np.array([t[0], t[1], sign * tz]))
        xyz, inten = oracle(disp, img, cam)
        assert len(xyz) == (n_valid if kept else 0), tz
        st, res = reproject_device(disp, img, cam)
        assert st == 0
        check_outputs(res[0], xyz, inten, "t_z = %r" % (sign * tz))
        if kept:
            assert (res[0]["xyz"][2:3 * n_valid:3] == sign * tz).all()


# 7. the argument contract
def test_reproject_argument_contract():
    h, w = 4, 8
    disp, img = frame(h, w, "random", seed=7)
    k4, b, R, t = camera(h, w)
    D, I = Dev(4 * h * w).put(disp), Dev(h * w).put(img)
    X, N, S, K = Dev(24 * h * w), Dev(4 * h * w), Dev(4), Dev(8)
    L = amb.lib()
    INVALID, CHECK = _lib.AMB_ERR_INVALID_ARGUMENT, _lib.AMB_ERR_CHECK_FAILED

    def dev(**kw):
        a = dict(d=D.ptr, ds=w, i=I.ptr, ist=w, w=w, h=h, k=ptr(k4), b=b, R=ptr(R), t=ptr(t), x=X.ptr, n=N.ptr,
                 s=S.ptr, c=K.ptr)
        a.update(kw)
        st = L.amb_stereo_reproject_device(0, None, a["d"], a["ds"], a["i"], a["ist"], a["w"], a["h"], a["k"], a["b"],
                                           a["R"], a["t"], 1.0, a["x"], a["n"], h * w, a["s"], a["c"])
        sync()
        return st

    hx, hi = np.zeros((h * w, 3)), np.zeros(h * w, np.int32)

    def host(**kw):
        a = dict(d=ptr(disp), ds=w, i=ptr(img), ist=w, w=w, h=h, b=b, x=ptr(hx), n=ptr(hi), cnt=C.byref(C.c_size_t()))
        a.update(kw)
        return L.amb_stereo_reproject(0, a["d"], a["ds"], a["i"], a["ist"], a["w"], a["h"], ptr(k4), a["b"], ptr(R),
                                      ptr(t), 1.0, a["x"], a["n"], h * w, a["cnt"])

    assert dev() == 0 and host() == 0
    for arg in ("d", "i", "k", "R", "t", "x", "n", "s", "c"):
        assert dev(**{arg: None}) == INVALID, arg
    for arg in ("d", "i", "x", "n"):
        assert host(**{arg: None}) == INVALID, arg
    assert host(cnt=None) == INVALID
    for f in (dev, host):
        for kw in (dict(w=0), dict(w=-1), dict(h=0), dict(h=-3), dict(ds=w - 1), dict(ist=w - 1), dict(ds=0)):
            assert f(**kw) == INVALID, (f.__name__, kw)
        assert f(b=0.0) == CHECK and f(b=-0.0) == CHECK, f.__name__
    # a stride longer than the row is a pitched frame
    assert dev(ds=w + 1, w=w - 1) == 0 and dev(ist=w + 9) == 0
    # the oracle keeps the same contract
    cnt = C.c_size_t(0)
    O = po.lib().ambo_stereo_reproject
    for ds, ist, ww, hh in ((w - 1, w, w, h), (w, w - 1, w, h), (w, w, 0, h), (w, w, w, 0)):
        assert O(ptr(disp), ds, ptr(img), ist, ww, hh, ptr(k4), b, ptr(R), ptr(t), 1.0, ptr(hx), ptr(hi), h * w,
                 C.byref(cnt)) == INVALID, (ds, ist, ww, hh)


# ---- B. rectification maps --------------------------------------------------------------------------------------------
def round_up(a, b):
    return (a + b - 1) // b * b


def rectify_device(T1, T2, w, h, stride, shift=0, one_alloc=False, flag=0, stream=None):
    """amb_stereo_rectify_maps_device into maps of row stride `stride` floats whose planes start `shift` floats past a
    64-byte aligned address: in four allocations, or back to back in one.  flag: the value the zero-w flag starts as
    (None: a NULL flag pointer).  Checks that no byte outside the maps' W x H cells changed (row padding, the bytes
    before and after the planes); returns the status, the four maps [h, w] and the flag."""
    plane = stride * h
    T1 = np.ascontiguousarray(T1, np.float32).reshape(9)
    T2 = np.ascontiguousarray(T2, np.float32).reshape(9)
    if one_alloc:
        bufs = [Dev(4 * (4 * plane + shift))]
        where = [(0, shift + k * plane) for k in range(4)]
    else:
        bufs = [Dev(4 * (plane + shift)) for _ in range(4)]
        where = [(k, shift) for k in range(4)]
    F = None if flag is None else Dev(4).put(np.array([flag], np.int32))
    sync()
    st = amb.lib().amb_stereo_rectify_maps_device(0, stream, ptr(T1), ptr(T2), w, h, stride,
                                                  *[bufs[b].ptr + 4 * o for b, o in where],
                                                  None if F is None else F.ptr)
    sync()
    words = [B.get(np.uint32) for B in bufs]
    written = [np.zeros(len(x), bool) for x in words]
    maps = []
    for b, o in where:
        written[b][o:o + plane].reshape(h, stride)[:, :w] = True
        maps.append(words[b][o:o + plane].reshape(h, stride)[:, :w].view(np.float32))
    for x, m in zip(words, written):
        untouched(x, m, "maps of stride %d, %d floats past alignment" % (stride, shift))
    return st, maps, None if F is None else int(F.get(np.int32, count=1)[0])


def homographies(w, h, seed=2):
    from test_stereo_rectify import rig
    K, R1, R2, t1, t2 = rig(seed, w, h)
    _, _, T1, T2 = amb.rectify_stereo_setup(K, R1, R2, t1, t2)
    return T1, T2


def check_maps(maps, want, what):
    for k in range(4):
        assert same(maps[k], want[k]), "%s: map %d differs from the oracle" % (what, k)


# 1. the scalar-store instantiation: strides that are no multiple of 4 floats, planes 4 bytes past 16-byte alignment
RECT_SHAPES = [(1, 1), (2, 5), (3, 1), (4, 3), (5, 1), (8, 2), (37, 9), (64, 1), (66, 17), (63, 20)]


@pytest.mark.parametrize("one_alloc", [False, True], ids=["four_allocations", "one_allocation"])
@pytest.mark.parametrize("w,h", RECT_SHAPES, ids=["%dx%d" % s for s in RECT_SHAPES])
def test_rectify_scalar_stores_pitched_and_misaligned(w, h, one_alloc):
    T1, T2 = homographies(w, h)
    st, want = po.stereo_rectify_maps(T1, T2, w, h)
    assert st == 0
    for stride, shift in ((w + 1, 0), (w + 2, 0), (round_up(w, 4), 1), (round_up(w, 4) + 4, 1)):
        st, maps, flag = rectify_device(T1, T2, w, h, stride, shift, one_alloc)
        assert st == 0 and flag == 0
        check_maps(maps, want, "stride %d, shift %d" % (stride, shift))


# 2. a large frame on the scalar path: several grid-stride iterations per thread
@pytest.mark.skipif(EMULATED, reason="12 M pixels: minutes on the emulated kernels")
def test_rectify_large_frame_on_the_scalar_path():
    w, h = 4000, 3000
    T1, T2 = homographies(w, h, 4)
    st, want = po.stereo_rectify_maps(T1, T2, w, h)
    assert st == 0
    st, maps, flag = rectify_device(T1, T2, w, h, w + 1)
    assert st == 0 and flag == 0
    check_maps(maps, want, "4000x3000, stride 4001")


# 3. the zero-w flag
@pytest.mark.parametrize("w", [1, 2, 3, 5, 6, 7, 13])
def test_rectify_zero_w_flag(w):
    h = 3
    eye = np.eye(3, dtype=np.float32)

    def with_third_row(row):
        T = eye.copy()
        T[2] = row
        return T

    # w = u - c vanishes at u = c: c = W lies in a masked lane of the last group of 4 (W % 4 != 0), c = W - 1 does not;
    # (0, 1, -(H - 1)) vanishes on the last row only
    cases = [((1.0, 0.0, -float(w)), 0), ((1.0, 0.0, -float(w - 1)), 1), ((0.0, 1.0, -float(h - 1)), 1)]
    for row, flagged in cases:
        T = with_third_row(row)
        for T1, T2 in ((T, eye), (eye, T)):
            st, want = po.stereo_rectify_maps(T1, T2, w, h)
            assert st == (_lib.AMB_ERR_CHECK_FAILED if flagged else 0)
            for stride, shift in ((round_up(w, 4), 0), (w + 1, 0), (round_up(w, 4), 1)):
                what = "third row %s, stride %d, shift %d" % (row, stride, shift)
                st, maps, flag = rectify_device(T1, T2, w, h, stride, shift)
                assert st == 0 and flag == flagged, what
                check_maps(maps, want, what)
                if not flagged:
                    assert all(np.isfinite(m).all() for m in maps), what
                st, maps, _ = rectify_device(T1, T2, w, h, stride, shift, flag=None)      # a NULL flag pointer
                assert st == 0
                check_maps(maps, want, what + ", no flag")
                st, _, flag = rectify_device(T1, T2, w, h, stride, shift, flag=1)         # the kernel only sets it
                assert st == 0 and flag == 1, what
            if flagged:
                with pytest.raises(amb.AmbError) as ei:
                    amb.rectify_stereo_maps(T1, T2, w, h)
                assert ei.value.status == _lib.AMB_ERR_CHECK_FAILED
            else:
                check_maps(amb.rectify_stereo_maps(T1, T2, w, h), want, "host entry")


# 4. the rig's homographies, pitched maps, both streams
@pytest.mark.parametrize("w,h,seed", [(640, 480, 2), (333, 77, 3), (5, 3, 5)])
def test_rectify_rig_homographies_through_the_device_entry(w, h, seed):
    T1, T2 = homographies(w, h, seed)
    st, want = po.stereo_rectify_maps(T1, T2, w, h)
    assert st == 0
    for name, handle, _keep in stream_handles():
        for stride, shift, one in ((w + 3, 1, True), (round_up(w, 4) + 8, 0, False)):
            st, maps, flag = rectify_device(T1, T2, w, h, stride, shift, one, stream=handle)
            assert st == 0 and flag == 0
            check_maps(maps, want, "%s stream, stride %d" % (name, stride))
    assert po.lib().ambo_stereo_rectify_maps(ptr(T1), ptr(T2), w, h, w - 1, *[ptr(m) for m in want]) == \
        _lib.AMB_ERR_INVALID_ARGUMENT
    dummy = Dev(16)
    assert amb.lib().amb_stereo_rectify_maps_device(0, None, ptr(T1), ptr(T2), w, h, w - 1, *[dummy.ptr] * 4,
                                                    None) == _lib.AMB_ERR_INVALID_ARGUMENT


# ---- C. both stages chained on the device ---------------------------------------------------------------------------
PLANES = {"horizontal": (0.0, 0.0), "tilted": (0.15, -0.1)}


def plane_disparity(h, w, k4, b, R, t, z0, grad, X0, Y0):
    """The rectified disparity of the plane z = z0 + gx (X - X0) + gy (Y - Y0): pixel (u, v)'s ray R q,
    q = ((u - cx)/fx, (v - cy)/fy, 1), from t meets it at depth s; d = (float)(fx b / s)."""
    fx, fy, cx, cy = k4
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    q = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], -1)
    r = q @ R.reshape(3, 3).T
    gx, gy = grad
    s = (z0 + gx * (t[0] - X0) + gy * (t[1] - Y0) - t[2]) / (r[..., 2] - gx * r[..., 0] - gy * r[..., 1])
    assert (s > 0).all()
    return (fx * b / s).astype(np.float32)


@pytest.mark.parametrize("plane", sorted(PLANES))
def test_disparity_to_dsm_and_ortho_on_the_device(plane):
    from scipy.spatial.transform import Rotation
    h, w = 150, 200
    k4 = np.array([250.0, 250.0, 99.75, 74.2])
    b = 12.0
    R = np.ascontiguousarray((Rotation.from_euler("z", 0.3) * Rotation.from_euler("x", np.pi)).as_matrix().reshape(9))
    rows, cols, res = 60, 80, 1.0
    ce, cn = UTM_SHIFT
    X0, Y0 = UTM[0] + cn, UTM[1] + ce            # the map centre in raw (unshifted) coordinates
    z0, grad = 420.0, PLANES[plane]
    t = np.array([X0 + 1.3, Y0 - 2.1, z0 + 100.0])
    disp = plane_disparity(h, w, k4, b, R, t, z0, grad, X0, Y0)
    gray = 137
    img = np.full((h, w), gray, np.uint8)
    cam = (k4, b, R, t)

    # the GPU pipeline: disparities in device memory, reprojected into a buffer of capacity W * H
    D, I = Dev(4 * h * w).put(disp), Dev(h * w).put(img)
    X, N, S, K = Dev(24 * h * w), Dev(4 * h * w), Dev(4 * blocks_of(h, w)), Dev(8)
    sync()
    assert amb.lib().amb_stereo_reproject_device(0, None, D.ptr, w, I.ptr, w, w, h, ptr(k4), b, ptr(R), ptr(t), 1.0,
                                                 X.ptr, N.ptr, h * w, S.ptr, K.ptr) == 0
    sync()
    n = int(K.get(np.uint64, count=1)[0])
    oxyz, ointen = oracle(disp, img, cam)
    assert n == len(oxyz) == h * w
    assert same(X.get(np.float64, count=3 * n).reshape(-1, 3), oxyz)
    assert np.array_equal(N.get(np.int32, count=n), ointen)

    gm = amb.AerialGridMap(amb.GridMapSettings(UTM[0], UTM[1], rows * res, cols * res, res)).getMutable()
    gm.to_device(0, names=("elevation",))
    amb.Dsm(amb.DsmSettings(interpolation_radius=1, center_easting=ce, center_northing=cn), gm).process_device(
        X.ptr, n, gm)
    gm.sync()
    gm.download(("elevation",))
    elev = gm["elevation"].copy()
    go = amb.AerialGridMap(amb.GridMapSettings(X0, Y0, rows * res, cols * res, res)).getMutable()
    go.to_device(0, names=("ortho",))
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=2)).process_device(X.ptr, N.ptr, n, go)
    go.sync()
    go.download(("ortho",))
    ortho = go["ortho"].copy()

    # against the oracle chain
    e = np.full((rows, cols), np.nan, np.float32, order="F")
    st, _, lvl, _ = po.dsm_process(po.make_geometry(rows, cols, res, UTM[0], UTM[1]), e, oxyz, radius=1,
                                   center_easting=ce, center_northing=cn, debug=True)
    assert st == 0
    assert np.array_equal(np.isnan(elev), np.isnan(e))
    ok = ~np.isnan(e)
    assert np.allclose(elev[ok], e[ok], rtol=1e-6, atol=0.0)
    assert ulp_diff(elev, e).max() <= MAX_ULP
    o = np.full((rows, cols), 255.0, np.float32, order="F")
    assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res, X0, Y0), o, oxyz, ointen, radius=2) == 0
    filled = o != 255.0
    assert np.array_equal(filled, ortho != 255.0)
    assert ulp_diff(ortho, o).max() <= 1

    # against the geometry, in float64: a cell resolved at level 0 averages heights within sqrt(radius) = 1 m
    qx, qy = synth.grid_positions(rows, cols, res, UTM[0], UTM[1])
    zc = z0 + grad[0] * ((qx[:, None] + cn) - X0) + grad[1] * ((qy[None, :] + ce) - Y0)
    covered = lvl == 0
    assert covered.sum() > 0.3 * rows * cols
    bound = math.hypot(*grad) * 1.0 + 1e-3
    assert np.abs(elev[covered] - zc[covered]).max() <= bound
    if plane == "horizontal":
        assert np.abs(elev[ok] - z0).max() <= 1e-3
    assert filled.sum() > 0.3 * rows * cols and (ortho[filled] == gray).all()
