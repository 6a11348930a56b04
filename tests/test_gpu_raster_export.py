"""North-up raster export of map layers (amb_export_raster*, csrc/raster_export.cu; convention in
include/aerial_mapper_b200.h): every format against a numpy restatement of the convention, bit for bit.

    pixel (r, c) = layer(i = rows - 1 - c, j = r);   a stripe [c0, c1) owns image rows [c0, c1)

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels, so the kernel logic is checked on
every CPU run too."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402

gpu = pytest.mark.gpu
EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
FORMATS = ("f32", "gray8", "bgr8", "mask8")
CANARY = 0xA5
UTM = (464500.0, 5272500.0)


# ---- the convention, restated (test-only) -----------------------------------------------------------------------------
def restate(layer, fmt):
    """layer: float32 [rows, band_cols] (column-major slab) -> the exported band, as the header defines it."""
    img = np.ascontiguousarray(np.asarray(layer, np.float32).T[:, ::-1])   # (r, c) = layer[rows - 1 - c, r]
    bits = img.view(np.uint32)
    nan = (bits & 0x7FFFFFFF) > 0x7F800000
    if fmt == "f32":
        return img
    if fmt == "mask8":
        return np.where(nan, 0, 255).astype(np.uint8)
    if fmt == "bgr8":
        v = np.where(nan, 0, bits)
        return np.stack([(v >> s) & 0xFF for s in (0, 8, 16)], axis=-1).astype(np.uint8)
    # gray8: OpenCV saturate_cast<uchar>(float) = cvRound (half to even; NaN / outside int32 -> INT_MIN), clamp to [0, 255]
    with np.errstate(invalid="ignore"):
        out_of_int = nan | ~(img < np.float32(2.0 ** 31))
        r = np.rint(np.where(out_of_int, 0, img).astype(np.float64))
    return np.where(out_of_int, 0, np.clip(r, 0, 255)).astype(np.uint8)


def same(got, want):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    return got.shape == want.shape and got.dtype == want.dtype and got.tobytes() == want.tobytes()


def special_layer(rows, cols, seed):
    """A layer mixing NaN payloads, +-0, +-inf, packed-colour denormals, gray ties and out-of-range values."""
    rng = np.random.default_rng(seed)
    special_bits = np.array([0x7FC00000, 0xFFC00001, 0x7F800001, 0x00000000, 0x80000000, 0x7F800000, 0xFF800000,
                             0x00FF8040, 0x00000001, 0x00123456, 0x00FFFFFF, 0x4F000000, 0x4EFFFFFF, 0xCF000000],
                            np.uint32).view(np.float32)
    ties = np.arange(-3, 259, dtype=np.float32) + np.float32(0.5)
    pool = np.concatenate([special_bits, ties, np.float32([-0.4, -0.6, 254.5, 255.4, 255.5, 256.0, 1e9, 3e9, -1e10,
                                                           0.49999997, 127.49999])])
    n = rows * cols
    v = rng.uniform(-20.0, 280.0, n).astype(np.float32)
    pick = rng.random(n) < 0.6
    v[pick] = pool[rng.integers(0, len(pool), int(pick.sum()))]
    colours = rng.integers(0, 1 << 24, n).astype(np.uint32).view(np.float32)   # packed 0x00RRGGBB: denormals
    colour = rng.random(n) < 0.2
    v[colour] = colours[colour]
    return np.asfortranarray(v.reshape(rows, cols, order="F"))


def resident_map(layers, col_range=None, res=1.0, center=(0.0, 0.0)):
    """A device-resident map (whole map or one stripe) holding the given float32 [rows, cols] layers."""
    rows, cols = next(iter(layers.values())).shape
    gm = amb.AerialGridMap(amb.GridMapSettings(center[0], center[1], rows * res, cols * res, res)).getMutable()
    assert gm.getSize() == (rows, cols)
    for name, a in layers.items():
        gm[name] = a
    gm.to_device(0, col_range=col_range, names=tuple(layers))
    return gm


class Dev(object):
    """`nbytes` of device memory at .ptr (16-byte aligned + `off`), 64 guard bytes on each side, every byte CANARY."""

    def __init__(self, nbytes, off=0):
        n = int(nbytes) + 160
        if EMULATED:
            self.raw = np.full(n, CANARY, np.uint8)
            p = self.raw.ctypes.data
        else:
            import torch
            self.raw = torch.full((n,), CANARY, dtype=torch.uint8, device="cuda:0")
            p = self.raw.data_ptr()
        self.lo = (-p) % 16 + 64 + off
        self.ptr = p + self.lo
        self.nbytes = int(nbytes)

    def all(self):
        return self.raw.copy() if EMULATED else self.raw.cpu().numpy()


def sync_device():
    if not EMULATED:
        import torch
        torch.cuda.synchronize()


def as_fmt(buf, fmt, shape):
    if fmt == "f32":
        return buf.view(np.float32).reshape(shape)
    return buf.reshape(shape + ((3,) if fmt == "bgr8" else ()))


# ---- every format, bit for bit ----------------------------------------------------------------------------------------
SHAPES = [(1, 1), (1, 37), (37, 1), (3, 29), (17, 11), (33, 7), (1000, 9)]


@gpu
@pytest.mark.parametrize("rows,cols", SHAPES)
def test_every_format_equals_the_restatement(rows, cols):
    layer = special_layer(rows, cols, seed=rows * 131 + cols)
    gm = resident_map({"ortho": layer})
    for fmt in FORMATS:
        got = gm.to_raster("ortho", fmt)
        assert same(got, restate(layer, fmt)), (fmt, rows, cols)


@gpu
def test_gray_ties_and_saturation_exactly():
    v = np.float32([0.5, 1.5, 2.5, 3.5, -0.5, -1.5, 254.5, 255.5, 253.5, 255.49998, 256.0, 2.0 ** 31, 2.0 ** 31 - 128,
                    3e9, np.inf, -np.inf, np.nan, -0.0, 1e-45, 0.49999997, 0.50000006])
    want = np.uint8([0, 2, 2, 4, 0, 0, 254, 255, 254, 255, 255, 0, 255, 0, 0, 0, 0, 0, 0, 0, 1])
    gm = resident_map({"ortho": np.asfortranarray(v.reshape(-1, 1))})
    got = gm.to_raster("ortho", "gray8")
    assert got.shape == (1, len(v)) and np.array_equal(got[0, ::-1], want)


# ---- real layers of a DSM + gray and colour orthomosaic run -----------------------------------------------------------
@gpu
def test_layers_of_a_dsm_and_ortho_run():
    rows, cols, res = 72, 56, 1.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(8000, rows * res / 2, cols * res / 2, seed=21, holes=2, hole_sides=(4.0, 10.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, agl=60.0, seed=4, jitter_pos=0.5)
    for colored in (False, True):
        ch = 3 if colored else 1
        imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(poses))]
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm).process(poses, imgs, gm)
    gm.sync()
    names = ("elevation", "ortho", "colored_ortho", "observation_index")
    gm.download(names)
    for name, fmt in (("elevation", "f32"), ("ortho", "gray8"), ("colored_ortho", "bgr8"), ("observation_index", "mask8"),
                      ("elevation", "mask8")):
        got = gm.to_raster(name, fmt)
        assert same(got, restate(gm[name], fmt)), (name, fmt)
    assert np.isnan(gm["elevation"]).any() and (~np.isnan(gm["observation_index"])).any()
    assert (~np.isnan(gm["colored_ortho"])).any()


# ---- geolocation ------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("center", [(0.0, 0.0), (12.25, -7.5), UTM])
def test_geotransform_locates_every_cell_at_its_pixel(center):
    rows, cols, res = 41, 23, 0.5
    ids = np.arange(rows * cols, dtype=np.float32).reshape(rows, cols, order="F")   # cell (i, j) holds i + j * rows
    gm = resident_map({"elevation": np.asfortranarray(ids)}, res=res, center=center)
    img = gm.to_raster("elevation", "f32")
    gt = gm.geotransform()
    rng = np.random.default_rng(5)
    cells = [(0, 0), (rows - 1, 0), (0, cols - 1), (rows - 1, cols - 1)] + \
        [tuple(int(v) for v in rng.integers(0, (rows, cols))) for _ in range(40)]
    for i, j in cells:
        x, y = gm.getPosition((i, j))
        c, r = int(np.floor((x - gt[0]) / gt[1])), int(np.floor((y - gt[3]) / gt[5]))
        assert (r, c) == (j, rows - 1 - i)
        assert img[r, c] == i + j * rows


# ---- stripes and several GPUs -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_stripe_contexts_write_one_image(fmt):
    rows, cols = 45, 23
    layer = special_layer(rows, cols, seed=9)
    whole = resident_map({"colored_ortho": layer}).to_raster("colored_ortho", fmt)
    full = np.full_like(whole, CANARY)
    maps = []
    for c0, c1 in ((0, 1), (1, 8), (8, cols)):
        gm = resident_map({"colored_ortho": layer}, col_range=(c0, c1))
        gm.to_raster("colored_ortho", fmt, out=full[c0:c1])
        maps.append(gm)
    assert same(full, whole) and same(whole, restate(layer, fmt))


@gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_export_on_every_visible_gpu(fmt):
    L = _lib.lib()
    rows, cols = 37, 29
    layer = special_layer(rows, cols, seed=13)
    g = amb.Geometry()
    assert L.amb_geometry_init(float(rows), float(cols), 1.0, 0.0, 0.0, C.byref(g)) == 0
    m = C.c_void_p()
    n = min(L.amb_device_count(), cols)
    assert L.amb_multi_create(C.byref(g), n, C.byref(m)) == 0
    try:
        assert L.amb_multi_upload_layer(m, _lib.LAYER_ID["elevation"], layer.ctypes.data) == 0
        want = restate(layer, fmt)
        img = np.full(want.shape, CANARY, want.dtype)
        assert L.amb_multi_export_raster(m, _lib.LAYER_ID["elevation"], _lib.RASTER_FORMAT[fmt], img.ctypes.data) == 0
        assert same(img, want)
    finally:
        L.amb_multi_destroy(m)


# ---- host destinations ------------------------------------------------------------------------------------------------
@gpu
def test_pinned_and_pageable_destinations_are_identical():
    rows, cols = 1100, 1000                  # 4.4 MB as float32: above the 4 MB threshold of the staged pageable copy
    layer = special_layer(rows, cols, seed=17)
    gm = resident_map({"elevation": layer})
    p = C.c_void_p()
    nbytes = rows * cols * 4
    amb.check(_lib.lib().amb_host_alloc(C.byref(p), nbytes))
    try:
        pinned = np.frombuffer((C.c_uint8 * nbytes).from_address(p.value), np.float32).reshape(cols, rows)
        gm.to_raster("elevation", "f32", out=pinned)
        pageable = gm.to_raster("elevation", "f32")
        assert same(pinned, restate(layer, "f32")) and same(pageable, pinned)
    finally:
        _lib.lib().amb_host_free(p)


# ---- device destinations ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_device_export_at_every_byte_offset(fmt):
    L = _lib.lib()
    for rows, cols in ((33, 9), (1000, 5)):
        layer = special_layer(rows, cols, seed=rows + cols)
        want = restate(layer, fmt)
        nbytes = want.nbytes
        gm = resident_map({"ortho": layer})
        for off in range(16):
            d = Dev(nbytes, off)
            amb.check(L.amb_export_raster_device(gm.context(), _lib.LAYER_ID["ortho"], _lib.RASTER_FORMAT[fmt], d.ptr),
                      gm.context())
            gm.sync()
            raw = d.all()
            got = as_fmt(raw[d.lo:d.lo + nbytes].copy(), fmt, want.shape[:2])
            assert same(got, want), (fmt, rows, cols, off)
            assert (raw[:d.lo] == CANARY).all() and (raw[d.lo + nbytes:] == CANARY).all(), (fmt, rows, cols, off)


def device_array(a):
    if EMULATED:
        return a, a.ctypes.data
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t, t.data_ptr()


@gpu
def test_export_enqueued_right_after_process_equals_one_after_sync():
    rows, cols, res = 300, 260, 0.5
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(60000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    keep, d_xyz = device_array(np.ascontiguousarray(xyz))
    sync_device()
    L = _lib.lib()
    ctx = gm.context()
    bufs = {}
    for fmt in ("f32", "mask8"):
        want_bytes = rows * cols * _lib.RASTER_BPP[_lib.RASTER_FORMAT[fmt]]
        bufs[fmt] = Dev(want_bytes, 3)
    amb.Dsm(amb.DsmSettings(), gm).process_device(d_xyz, len(xyz), gm)
    for fmt, d in bufs.items():   # no amb_sync in between: ordered on the context's stream
        amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID["elevation"], _lib.RASTER_FORMAT[fmt], d.ptr), ctx)
    gm.sync()
    for fmt, d in bufs.items():
        got = as_fmt(d.all()[d.lo:d.lo + d.nbytes].copy(), fmt, (cols, rows))
        assert same(got, gm.to_raster("elevation", fmt)), fmt
    gm.download(("elevation",))
    assert same(gm.to_raster("elevation", "f32"), restate(gm["elevation"], "f32"))
    assert np.isfinite(gm["elevation"]).mean() > 0.5
    del keep


# ---- the argument contract --------------------------------------------------------------------------------------------
@gpu
def test_invalid_arguments_write_nothing():
    L = _lib.lib()
    layer = special_layer(5, 4, seed=3)
    gm = resident_map({"ortho": layer})
    ctx = gm.context()
    buf = np.full(5 * 4 * 4 + 64, CANARY, np.uint8)
    p = buf.ctypes.data
    d = Dev(len(buf))
    # (ctx, layer, format, destination given)
    bad = [(ctx, -1, 0, True), (ctx, len(_lib.LAYER_NAMES), 0, True), (ctx, 0, -1, True), (ctx, 0, 4, True),
           (ctx, 0, 0, False), (None, 0, 0, True)]
    for c, layer_id, fmt, given in bad:
        args = (c, layer_id, fmt)
        assert L.amb_export_raster(*args, p if given else None) == _lib.AMB_ERR_INVALID_ARGUMENT, args
        assert L.amb_export_raster_device(*args, d.ptr if given else None) == _lib.AMB_ERR_INVALID_ARGUMENT, args
    gm.sync()
    assert (buf == CANARY).all() and (d.all() == CANARY).all()
    g = amb.Geometry()
    assert L.amb_raster_geotransform(None, (C.c_double * 6)()) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_raster_geotransform(C.byref(g), None) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_multi_export_raster(None, 0, 0, p) == _lib.AMB_ERR_INVALID_ARGUMENT
    with pytest.raises(KeyError):
        gm.to_raster("ortho", "png")
    with pytest.raises(amb.AmbError) as ei:
        amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable().to_raster("ortho", "gray8")
    assert "to_device()" in str(ei.value)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_raster_export.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
