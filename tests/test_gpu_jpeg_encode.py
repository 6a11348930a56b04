"""Baseline JPEG on the device (amb_jpeg_encode_device, amb_export_jpeg, csrc/jpeg_encode.cu; convention in
include/aerial_mapper_b200.h): every file is compared byte for byte with cv2.imencode(".jpg", img, params) of the same
8-bit image.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last tests run this file's `gpu` tests on the emulated kernels, so the kernel logic is checked on
every CPU run too (the 10000 x 10000 case and the torch wrapper need a GPU)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, synth  # noqa: E402

cv2 = pytest.importorskip("cv2")

gpu = pytest.mark.gpu
EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
CANARY = 0xA5
QUALITIES = (1, 10, 50, 75, 95, 100)
RESTARTS = (0, 1, 3, 8, 1000)
SMALL = [(1, 1), (1, 37), (37, 1), (7, 9), (8, 8), (9, 8), (15, 17), (16, 16), (17, 33)]   # (height, width)
GOLDEN = os.path.join(HERE, "golden", "jpeg_cases.npz")


def cv2_jpeg(img, quality=95, sampling="420", restart=0):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == "420" else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
    ok, b = cv2.imencode(".jpg", img, params)
    assert ok
    return b.tobytes()


def content(kind, h, w, channels, seed):
    rng = np.random.default_rng(seed)
    shape = (h, w) if channels == 1 else (h, w, 3)
    if kind == "noise":
        return rng.integers(0, 256, shape).astype(np.uint8)
    if kind == "constant":
        return np.full(shape, int(rng.integers(0, 256)), np.uint8)
    if kind == "checker":
        a = np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, 255, 0).astype(np.uint8)
        return a if channels == 1 else np.repeat(a[:, :, None], 3, axis=2) ^ np.uint8([0, 255, 0])
    # smooth gradient
    a = np.add.outer(np.arange(h) * 3, np.arange(w) * 2)
    if channels == 1:
        return (a % 256).astype(np.uint8)
    return np.stack([(a + 40 * k) % 256 for k in range(3)], axis=-1).astype(np.uint8)


class Dev(object):
    """A device copy of `img` with rows `pitch` bytes apart at byte offset `off` from 16-byte alignment."""

    def __init__(self, img, pitch=None, off=0):
        img = np.ascontiguousarray(img)
        h = img.shape[0]
        row = img[0].nbytes
        self.pitch = pitch or row
        host = np.full(64 + off + h * self.pitch + 64, CANARY, np.uint8)
        for r in range(h):
            host[64 + off + r * self.pitch:64 + off + r * self.pitch + row] = img[r].reshape(-1)
        if EMULATED:
            self.raw = host
            p = host.ctypes.data
            self.ptr = p + 64 + off   # numpy allocations are 16-byte aligned
        else:
            import torch
            self.raw = torch.empty(len(host) + 16, dtype=torch.uint8, device="cuda:0")
            base = (-self.raw.data_ptr()) % 16
            self.raw[base:base + len(host)].copy_(torch.from_numpy(host))
            self.ptr = self.raw.data_ptr() + base + 64 + off


def encode_dev(d, h, w, channels, quality=95, sampling="420", restart=0, out=None, capacity=None):
    L = _lib.lib()
    ctx = api._jpeg_context(0)
    cap = L.amb_jpeg_max_size(w, h, channels, quality, api.JPEG_SAMPLING[sampling], restart)
    buf = np.empty(cap, np.uint8) if out is None else out
    size = C.c_size_t(0)
    st = L.amb_jpeg_encode_device(ctx, d.ptr, w, h, d.pitch, channels, quality, api.JPEG_SAMPLING[sampling], restart,
                                  buf.ctypes.data, cap if capacity is None else capacity, C.byref(size))
    return st, buf, size.value


def encode(img, quality=95, sampling="420", restart=0, pitch=None, off=0):
    h, w = img.shape[:2]
    channels = 1 if img.ndim == 2 else 3
    st, buf, n = encode_dev(Dev(img, pitch, off), h, w, channels, quality, sampling, restart)
    amb.check(st, api._jpeg_context(0))
    return buf[:n].tobytes()


def first_difference(a, b):
    n = min(len(a), len(b))
    k = next((i for i in range(n) if a[i] != b[i]), n)
    return "sizes %d / %d, first difference at byte %d" % (len(a), len(b), k)


def check_same(img, quality=95, sampling="420", restart=0, **kw):
    got, want = encode(img, quality, sampling, restart, **kw), cv2_jpeg(img, quality, sampling, restart)
    assert got == want, (img.shape, quality, sampling, restart, first_difference(got, want))


# ---- the whole parameter grid -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mode", ["gray", "420", "444"])
@pytest.mark.parametrize("quality", QUALITIES)
def test_parameter_grid_on_small_sizes(mode, quality):
    channels = 1 if mode == "gray" else 3
    sampling = "444" if mode == "444" else "420"
    for restart in RESTARTS:
        for k, (h, w) in enumerate(SMALL):
            img = content(("noise", "smooth", "checker", "constant")[k % 4], h, w, channels, seed=quality * 100 + k)
            check_same(img, quality, sampling, restart)


@gpu
@pytest.mark.parametrize("mode", ["gray", "420", "444"])
@pytest.mark.parametrize("kind", ["noise", "constant", "checker", "smooth"])
def test_every_content_at_every_small_size(mode, kind):
    channels = 1 if mode == "gray" else 3
    sampling = "444" if mode == "444" else "420"
    for k, (h, w) in enumerate(SMALL):
        img = content(kind, h, w, channels, seed=k)
        for quality, restart in ((95, 0), (100, 1), (50, 3)):
            check_same(img, quality, sampling, restart)


@gpu
@pytest.mark.parametrize("mode", ["gray", "420", "444"])
def test_333_by_250(mode):
    channels = 1 if mode == "gray" else 3
    sampling = "444" if mode == "444" else "420"
    for kind in ("noise", "smooth", "checker"):
        img = content(kind, 333, 250, channels, seed=7)
        for quality, restart in ((95, 0), (75, 8), (100, 1000), (10, 1)):
            check_same(img, quality, sampling, restart)


@gpu
def test_10000_by_10000():
    if EMULATED:
        return   # minutes on the emulated kernels; every path it takes is covered by the smaller cases
    rng = np.random.default_rng(3)
    base = np.add.outer(np.arange(10000) // 7, np.arange(10000) // 5).astype(np.uint8)
    img = np.stack([base, base ^ 0x5A, base + rng.integers(0, 4, base.shape).astype(np.uint8)], axis=-1)
    for sampling in ("420", "444"):
        check_same(img, 95, sampling, 0)
    check_same(np.ascontiguousarray(img[:, :, 1]), 95, "420", 1000)


# ---- device layout ------------------------------------------------------------------------------------------------------
@gpu
def test_pitched_and_misaligned_inputs():
    for channels in (1, 3):
        img = content("noise", 19, 27, channels, seed=channels)
        row = img[0].nbytes
        for off in range(16):
            check_same(img, 90, "420", 2, pitch=row + 5 + off, off=off)
        check_same(img, 90, "444", 0, pitch=row + 64, off=3)


# ---- real layers of a DSM + orthomosaic run -------------------------------------------------------------------------
def ortho_run(rows=72, cols=56, col_range=None):
    res = 1.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0, col_range=col_range)
    xyz = synth.point_cloud(8000, rows * res / 2, cols * res / 2, seed=21, holes=2, hole_sides=(4.0, 10.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, agl=60.0, seed=4, jitter_pos=0.5)
    for colored in (False, True):
        ch = 3 if colored else 1
        imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(poses))]
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm).process(poses, imgs, gm)
    return gm


@gpu
def test_ortho_layers_of_a_dsm_and_ortho_run():
    gm = ortho_run()
    gm.sync()
    for name, fmt in (("ortho", "gray8"), ("colored_ortho", "bgr8")):
        band = gm.to_raster(name, fmt)
        assert (band == 0).any(), "NaN cells export as black"
        for sampling, restart in (("420", 0), ("444", 5)):
            got = gm.to_jpeg(name, quality=95, sampling=sampling, restart_interval=restart)
            assert got == cv2_jpeg(band, 95, sampling, restart), (name, sampling, restart)
    assert gm.to_jpeg("elevation", fmt="gray8", quality=80) == cv2_jpeg(gm.to_raster("elevation", "gray8"), 80)


@gpu
def test_stripe_context_encodes_its_band():
    whole = ortho_run()
    full = whole.to_raster("colored_ortho", "bgr8")
    src = {"colored_ortho": None}
    whole.download(("colored_ortho",))
    src["colored_ortho"] = whole["colored_ortho"].copy(order="F")
    rows, cols = whole.getSize()
    for c0, c1 in ((0, 1), (1, 20), (20, cols)):
        gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * 1.0, cols * 1.0, 1.0)).getMutable()
        gm["colored_ortho"] = src["colored_ortho"]
        gm.to_device(0, col_range=(c0, c1), names=("colored_ortho",))
        for sampling in ("420", "444"):
            assert gm.to_jpeg("colored_ortho", 90, sampling, 2) == cv2_jpeg(full[c0:c1], 90, sampling, 2), (c0, c1)


@gpu
def test_encode_enqueued_right_after_process_equals_one_after_sync():
    rows, cols, res = 300, 260, 0.5
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(60000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    first = gm.to_jpeg("elevation", fmt="gray8", quality=75)   # no amb_sync in between: ordered on the context's stream
    gm.sync()
    assert gm.to_jpeg("elevation", fmt="gray8", quality=75) == first
    assert first == cv2_jpeg(gm.to_raster("elevation", "gray8"), 75)


@gpu
def test_pinned_and_pageable_destinations_are_identical():
    img = content("noise", 700, 900, 3, seed=5)     # ~2-5 MB file: large enough for the staged pageable copy
    d = Dev(img)
    L = _lib.lib()
    cap = L.amb_jpeg_max_size(900, 700, 3, 100, 1, 0)
    p = C.c_void_p()
    amb.check(L.amb_host_alloc(C.byref(p), cap))
    try:
        pinned = np.frombuffer((C.c_uint8 * cap).from_address(p.value), np.uint8)
        st, _, n = encode_dev(d, 700, 900, 3, 100, "444", 0, out=pinned)
        assert st == 0
        st, pageable, m = encode_dev(d, 700, 900, 3, 100, "444", 0)
        assert st == 0 and n == m and pinned[:n].tobytes() == pageable[:m].tobytes()
        assert pageable[:m].tobytes() == cv2_jpeg(img, 100, "444", 0)
    finally:
        L.amb_host_free(p)


# ---- the argument contract ------------------------------------------------------------------------------------------
@gpu
def test_too_small_a_capacity_returns_the_size_and_writes_nothing():
    img = content("smooth", 40, 50, 3, seed=1)
    want = cv2_jpeg(img, 95, "420", 4)
    d = Dev(img)
    for cap in (0, 1, len(want) - 1):
        buf = np.full(len(want) + 64, CANARY, np.uint8)
        st, _, n = encode_dev(d, 40, 50, 3, 95, "420", 4, out=buf, capacity=cap)
        assert st == _lib.AMB_ERR_SIZE_MISMATCH and n == len(want) and (buf == CANARY).all(), cap
    buf = np.full(len(want) + 64, CANARY, np.uint8)
    st, _, n = encode_dev(d, 40, 50, 3, 95, "420", 4, out=buf, capacity=len(want))
    assert st == 0 and buf[:n].tobytes() == want and (buf[n:] == CANARY).all()


@gpu
def test_invalid_and_unsupported_arguments_write_nothing():
    L = _lib.lib()
    ctx = api._jpeg_context(0)
    d = Dev(content("noise", 9, 9, 3, seed=2))
    buf = np.full(4096, CANARY, np.uint8)
    size = C.c_size_t(12345)
    INV, UNS = _lib.AMB_ERR_INVALID_ARGUMENT, _lib.AMB_ERR_UNSUPPORTED
    # (ctx, image, w, h, stride, channels, quality, sampling, restart, out given, size given) -> status
    good = [ctx, d.ptr, 9, 9, 27, 3, 95, 0, 0, True, True]
    cases = [((0, None), INV), ((1, None), INV), ((9, False), INV), ((10, False), INV), ((2, 0), INV), ((3, -1), INV),
             ((4, 26), INV), ((2, 65536), UNS), ((3, 65536), UNS), ((5, 2), UNS), ((5, 4), UNS), ((6, 0), UNS),
             ((6, 101), UNS), ((7, 2), UNS), ((7, -1), UNS), ((8, -1), UNS), ((8, 65536), UNS)]
    for (k, v), want in cases:
        a = list(good)
        a[k] = v
        if k == 2 and v == 65536:
            a[4] = 65536 * 3
        st = L.amb_jpeg_encode_device(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8],
                                      buf.ctypes.data if a[9] else None, len(buf), C.byref(size) if a[10] else None)
        assert st == want, (k, v, st)
    assert (buf == CANARY).all() and size.value == 12345
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable()
    gm.to_device(0)
    gc = gm.context()
    for layer, fmt in ((-1, 1), (len(_lib.LAYER_NAMES), 1), (0, 0), (0, 3), (0, 4)):
        assert L.amb_export_jpeg(gc, layer, fmt, 95, 0, 0, buf.ctypes.data, len(buf), C.byref(size)) == INV
    assert L.amb_export_jpeg(gc, 0, 1, 0, 0, 0, buf.ctypes.data, len(buf), C.byref(size)) == UNS
    assert L.amb_export_jpeg(None, 0, 1, 95, 0, 0, buf.ctypes.data, len(buf), C.byref(size)) == INV
    gm.sync()
    assert (buf == CANARY).all() and size.value == 12345
    with pytest.raises(ValueError):
        gm.to_jpeg("elevation")
    with pytest.raises(ValueError):
        gm.to_jpeg("ortho", sampling="422")
    with pytest.raises(ValueError):
        gm.to_jpeg("ortho", quality=0)
    with pytest.raises(amb.AmbError):
        amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable().to_jpeg("ortho")


@gpu
def test_torch_wrapper():
    if EMULATED:
        return   # the wrapper takes torch CUDA tensors; its C entry point is what every other test here calls
    import torch
    img = content("smooth", 123, 77, 3, seed=4)
    t = torch.from_numpy(img).cuda()
    assert amb.encode_jpeg(t, 85, "444", 3) == cv2_jpeg(img, 85, "444", 3)
    big = torch.zeros((123, 100, 3), dtype=torch.uint8, device="cuda")
    big[:, :77] = t
    assert amb.encode_jpeg(big[:, :77]) == cv2_jpeg(img)                    # padded rows
    assert amb.encode_jpeg(t[:, :, 0].contiguous(), 60) == cv2_jpeg(np.ascontiguousarray(img[:, :, 0]), 60)
    with pytest.raises(ValueError):
        amb.encode_jpeg(t.float())
    with pytest.raises(ValueError):
        amb.encode_jpeg(t[:, ::2])


# ---- the fixture, for hosts without OpenCV ---------------------------------------------------------------------------
@gpu
def test_golden_cases_equal_the_fixture():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_jpeg_golden as mg
    z = np.load(GOLDEN)
    for k, (img, params) in enumerate(mg.cases()):
        assert encode(img, *params) == z["jpeg_%d" % k].tobytes(), (k, img.shape, params)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_jpeg_encode.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
