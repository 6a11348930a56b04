"""North-up raster import into map layers (amb_import_raster*, csrc/raster_import.cu; convention in
include/aerial_mapper_b200.h, amb_resample): every case bit for bit against a numpy restatement of the convention, which
builds the same per-axis tables in float64 and does the same per-cell blend.

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
from aerial_mapper_b200.io import read_geotiff, write_geotiff  # noqa: E402
from test_gpu_raster_export import Dev, EMULATED, UTM, device_array, resident_map, sync_device  # noqa: E402

gpu = pytest.mark.gpu
SNAP = 2.0 ** -20
SENTINEL = np.float32(-7777.25)


# ---- the convention, restated (test-only) -----------------------------------------------------------------------------
def axis_table(pos, origin, step, n, method):
    """Source index (-1: uncovered), fraction and the unsnapped fraction of every position along one axis."""
    u = (np.asarray(pos, np.float64) - origin) / step
    covered = (u >= 0) & (u < n)
    if method == "nearest":
        k, f = np.floor(np.where(covered, u, 0.0)), np.zeros_like(u)
        raw = f.copy()
    else:
        s = np.minimum(np.maximum(u - 0.5, 0.0), n - 1.0)
        s = np.where(covered, s, 0.0)
        k = np.floor(s)
        f = s - k
        raw = f.copy()
        hi = f > 1.0 - SNAP
        f = np.where((f < SNAP) | hi, 0.0, f)
        k = np.where(hi, k + 1, k)
    return np.where(covered, k, -1).astype(np.int32), np.where(covered, f, 0.0), raw


def tables(geom, width, height, gt, method, col_range=None):
    c0, c1 = col_range or (0, geom.cols)
    qx, qy = synth.grid_positions(geom.rows, geom.cols, geom.resolution, geom.pos_x, geom.pos_y)
    return axis_table(qx, gt[0], gt[1], width, method), axis_table(qy[c0:c1], gt[3], gt[5], height, method)


def no_data(p, nodata):
    nd = np.isnan(p)
    return nd | (p == np.float32(nodata)) if nodata is not None else nd


def restate(layer, geom, band, gt, method, nodata=None, col_range=None):
    """The slab [rows, c1 - c0] after importing `band` into `layer` (the slab before)."""
    band = np.asarray(band, np.float32)
    h, w = band.shape
    (ci, fx, _), (rj, fy, _) = tables(geom, w, h, gt, method, col_range)
    out = np.array(layer, np.float32, order="F", copy=True)
    C_, R_ = ci[:, None], rj[None, :]
    cov = (C_ >= 0) & (R_ >= 0)
    Cc, Rc = np.clip(C_, 0, w - 1), np.clip(R_, 0, h - 1)
    if method == "nearest":
        p = band[Rc, Cc]
        ok = cov & ~no_data(p, nodata)
        out[ok] = p[ok]
        return out
    FX, FY = fx[:, None], fy[None, :]
    wx, wy = np.broadcast_to(FX != 0, cov.shape), np.broadcast_to(FY != 0, cov.shape)
    C1, R1 = np.clip(C_ + 1, 0, w - 1), np.clip(R_ + 1, 0, h - 1)
    p00, p01, p10, p11 = band[Rc, Cc], band[Rc, C1], band[R1, Cc], band[R1, C1]
    bad = no_data(p00, nodata) | (wx & no_data(p01, nodata)) | \
        (wy & (no_data(p10, nodata) | (wx & no_data(p11, nodata))))
    d00, d01, d10, d11 = (a.astype(np.float64) for a in (p00, p01, p10, p11))
    with np.errstate(invalid="ignore", over="ignore"):
        row0 = np.where(wx, (1.0 - FX) * d00 + FX * d01, d00)
        row1 = np.where(wx, (1.0 - FX) * d10 + FX * d11, d10)
        hgt = np.where(wy, (1.0 - FY) * row0 + FY * row1, row0).astype(np.float32)
    ok = cov & ~bad
    out[ok] = hgt[ok]
    return out


def same(got, want):
    """Bit for bit, except that a NaN the blend generated (inf - inf) is compared as NaN: IEEE leaves its payload open."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    if got.shape != want.shape:
        return False
    eq = got.view(np.uint32) == want.view(np.uint32)
    return bool((eq | (np.isnan(got) & np.isnan(want))).all())


def geometry(rows, cols, res, center=(0.0, 0.0)):
    g = amb.Geometry()
    assert _lib.lib().amb_geometry_init(rows * res, cols * res, res, center[0], center[1], C.byref(g)) == 0
    assert (g.rows, g.cols) == (rows, cols)
    return g


def sentinel_map(rows, cols, res=1.0, center=(0.0, 0.0), col_range=None, name="elevation"):
    return resident_map({name: np.full((rows, cols), SENTINEL, np.float32, order="F")}, col_range=col_range, res=res,
                        center=center)


def layer_of(gm, name="elevation"):
    gm.sync()
    gm.download((name,))
    c0, c1 = gm._col_range
    return gm[name][:, c0:c1].copy(order="F")


def dem(h, w, seed, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    a = (300.0 + 40.0 * rng.standard_normal((h, w))).astype(np.float32)
    if nan_frac:
        a[rng.random((h, w)) < nan_frac] = np.nan
    return a


# ---- round trip -------------------------------------------------------------------------------------------------------
def dsm_map(rows, cols, res):
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(8000, rows * res / 2, cols * res / 2, seed=21, holes=2, hole_sides=(4.0, 10.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    gm.sync()
    return gm


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
@pytest.mark.parametrize("center", [(0.0, 0.0), UTM])
def test_round_trip_through_geotiff(tmp_path, method, center):
    rows, cols, res = 72, 56, 1.0
    if center == UTM:   # a DSM-like layer (terrain with empty patches) on a map at UTM scale
        layer = synth.analytic_elevation(rows, cols, res, *center)
        layer[10:25, 5:40] = np.nan
        layer[60:, 50:] = np.nan
        gm = resident_map({"elevation": layer}, res=res, center=center)
    else:
        gm = dsm_map(rows, cols, res)
    gm.download(("elevation",))
    orig = gm["elevation"].copy(order="F")
    assert np.isnan(orig).any() and np.isfinite(orig).mean() > 0.5
    path = str(tmp_path / "dem.tif")
    write_geotiff(path, gm.to_raster("elevation", "f32"), gm.geotransform(), nodata="nan")
    band, gt, epsg, nodata = read_geotiff(path)
    assert gt == gm.geotransform() and epsg == 32632 and np.isnan(nodata)
    fresh = amb.AerialGridMap(amb.GridMapSettings(center[0], center[1], rows * res, cols * res, res)).getMutable()
    fresh.to_device(0)
    fresh.from_raster("elevation", band, gt, nodata=nodata, resample=method)
    got = layer_of(fresh)
    assert np.array_equal(np.isnan(got), np.isnan(orig))
    assert np.array_equal(got.view(np.uint32)[~np.isnan(got)], orig.view(np.uint32)[~np.isnan(orig)])


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
@pytest.mark.parametrize("center", [(0.0, 0.0), UTM])
def test_aligned_import_copies_bits_including_signed_zero(method, center):
    rows, cols, res = 41, 23, 0.25
    rng = np.random.default_rng(3)
    layer = rng.uniform(-50, 50, (rows, cols)).astype(np.float32)
    layer[rng.random((rows, cols)) < 0.1] = -0.0
    layer[rng.random((rows, cols)) < 0.05] = np.float32(1e-45)
    layer[rng.random((rows, cols)) < 0.05] = np.inf
    layer[rng.random((rows, cols)) < 0.05] = -np.inf
    src = resident_map({"elevation": np.asfortranarray(layer)}, res=res, center=center)
    img = src.to_raster("elevation", "f32")
    dst = sentinel_map(rows, cols, res, center)
    dst.from_raster("elevation", img, src.geotransform(), resample=method)
    assert np.array_equal(layer_of(dst).view(np.uint32), layer.view(np.uint32))


# ---- orthomosaic on an imported DEM ------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("colored", [False, True])
def test_ortho_on_the_imported_dem_equals_ortho_on_the_original(colored):
    rows, cols, res = 72, 56, 1.0
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, agl=60.0, seed=4, jitter_pos=0.5)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], 3 if colored else 1) for k in range(len(poses))]
    a = dsm_map(rows, cols, res)
    b = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    b.to_device(0)
    b.from_raster("elevation", a.to_raster("elevation", "f32"), a.geotransform(), resample="bilinear")
    names = ("ortho", "colored_ortho", "elevation_angle", "observation_index", "elevation")
    for gm in (a, b):
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm).process(poses, imgs, gm)
        gm.sync()
        gm.download(names)
    assert (~np.isnan(a["observation_index"])).any()
    for name in names:
        assert np.array_equal(a[name].view(np.uint32), b[name].view(np.uint32)) or \
            np.array_equal(a[name], b[name], equal_nan=True), name


# ---- resampled ---------------------------------------------------------------------------------------------------------
RESAMPLED = {
    "coarser 1 m onto 0.25 m": (0.25, 1.0, (0.0, 0.0)),
    "finer 0.1 m onto 0.25 m": (0.25, 0.1, (0.0, 0.0)),
    "origin offset 0.3 px": (0.5, 0.5, (0.15, -0.35)),
    "coarser at UTM": (0.25, 1.0, (0.37, 0.61)),
}


@gpu
@pytest.mark.parametrize("case", sorted(RESAMPLED))
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_resampled_equals_the_restatement_and_scipy(case, method):
    res, dem_res, shift = RESAMPLED[case]
    rows, cols = 64, 48
    center = UTM if "UTM" in case else (0.0, 0.0)
    g = geometry(rows, cols, res, center)
    # a DEM over the map and a margin, its origin shifted by `shift` pixels of the DEM
    west = center[0] - rows * res / 2 - 3 * dem_res + shift[0] * dem_res
    north = center[1] + cols * res / 2 + 3 * dem_res + shift[1] * dem_res
    w, h = int(rows * res / dem_res) + 7, int(cols * res / dem_res) + 7
    band = dem(h, w, seed=len(case))
    gt = (west, dem_res, 0.0, north, 0.0, -dem_res)
    gm = sentinel_map(rows, cols, res, center)
    gm.from_raster("elevation", band, gt, resample=method)
    got = layer_of(gm)
    want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method)
    assert same(got, want), case
    assert (got != SENTINEL).all()
    if method != "bilinear":
        return
    # independent check of the half-pixel convention: scipy's bilinear interpolation at the same coordinates
    from scipy.ndimage import map_coordinates
    (_, _, rawx), (_, _, rawy) = tables(g, w, h, gt, method)
    qx, qy = synth.grid_positions(rows, cols, res, center[0], center[1])
    u, v = (qx - gt[0]) / gt[1] - 0.5, (qy - gt[3]) / gt[5] - 0.5
    V, U = np.meshgrid(v, u)
    sc = map_coordinates(band, [V.ravel(), U.ravel()], order=1, mode="nearest").reshape(rows, cols)
    outside = lambda f: (f == 0) | ((f >= SNAP) & (f <= 1 - SNAP))   # noqa: E731
    pick = outside(rawx)[:, None] & outside(rawy)[None, :]
    assert pick.mean() > 0.5
    ulps = np.abs(got.view(np.int32).astype(np.int64) - sc.view(np.int32).astype(np.int64))
    assert ulps[pick].max() <= 2, case


# ---- partial coverage, no-data, borders --------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
@pytest.mark.parametrize("shape,offset,dem_res", [((20, 30), (5.0, 7.0), 1.0), ((90, 120), (-10.0, -8.0), 1.0),
                                                  ((1, 1), (12.0, 9.0), 3.0), ((1, 17), (2.0, 4.0), 2.0),
                                                  ((17, 1), (6.0, 1.0), 2.0), ((3, 3), (0.5, 0.5), 0.5)])
def test_partial_coverage_keeps_every_other_cell(method, shape, offset, dem_res):
    rows, cols, res = 40, 36, 1.0
    g = geometry(rows, cols, res)
    band = dem(shape[0], shape[1], seed=shape[0] * 7 + shape[1], nan_frac=0.15 if min(shape) > 1 else 0.0)
    gt = (-rows * res / 2 + offset[0], dem_res, 0.0, cols * res / 2 - offset[1], 0.0, -dem_res)
    gm = sentinel_map(rows, cols, res)
    gm.from_raster("elevation", band, gt, resample=method)
    got = layer_of(gm)
    want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method)
    assert same(got, want)
    # cells outside the raster keep the sentinel; covered cells fed only by valid taps are written
    qx, qy = synth.grid_positions(rows, cols, res)
    inside = ((qx[:, None] >= gt[0]) & (qx[:, None] < gt[0] + shape[1] * dem_res) &
              (qy[None, :] <= gt[3]) & (qy[None, :] > gt[3] - shape[0] * dem_res))
    assert (got[~inside] == SENTINEL).all()
    if not np.isnan(band).any():
        assert (got[inside] != SENTINEL).all() and inside.any()


@gpu
def test_no_data_taps_and_snapped_weights():
    # one DEM pixel per 2 x 2 cells: cells at pixel quarters have weights 1/4 and 3/4, except at the borders
    rows, cols, res = 12, 10, 0.5
    g = geometry(rows, cols, res)
    band = np.arange(30, dtype=np.float32).reshape(5, 6) + 100
    band[2, 3] = np.nan
    band[1, 1] = -9999.0
    band[3, 4] = np.inf
    band[0, 5] = -np.inf
    band[4, 0] = -0.0
    gt = (-rows * res / 2, 1.0, 0.0, cols * res / 2, 0.0, -1.0)
    for nodata in (None, -9999.0, 0.0):
        for method in ("nearest", "bilinear"):
            gm = sentinel_map(rows, cols, res)
            gm.from_raster("elevation", band, gt, nodata=nodata, resample=method)
            got = layer_of(gm)
            want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method, nodata)
            assert same(got, want), (nodata, method)
            if method == "bilinear":
                # the 4 x 4 cells around the NaN pixel read it with non-zero weight: untouched
                (ci, fx, _), (rj, fy, _) = tables(g, 6, 5, gt, method)
                reads = ((ci[:, None] == 3) | ((ci[:, None] == 2) & (fx[:, None] != 0))) & \
                        ((rj[None, :] == 2) | ((rj[None, :] == 1) & (fy[None, :] != 0)))
                assert reads.sum() == 16 and (got[reads] == SENTINEL).all()
                # border cells (half a pixel from the edge) clamp: they read one column with weight 1
                assert (fx[[0, rows - 1]] == 0).all() and (got[[0, rows - 1]] != SENTINEL).any()
            if nodata == 0.0:   # -0 compares equal to 0: the pixel is no-data
                (ci, _, _), (rj, _, _) = tables(g, 6, 5, gt, "nearest")
                assert (got[(ci[:, None] == 0) & (rj[None, :] == 4)] == SENTINEL).all()


@gpu
def test_no_data_next_to_a_snapped_tap_is_not_read():
    # aligned raster: every fraction snaps to 0, so a NaN pixel only leaves its own cell untouched
    rows, cols = 9, 7
    band = dem(cols, rows, seed=2)
    band[3, 4] = np.nan
    gm = sentinel_map(rows, cols)
    gt = gm.geotransform()
    gm.from_raster("elevation", band, gt, resample="bilinear")
    got = layer_of(gm)
    assert (got == SENTINEL).sum() == 1 and got[rows - 1 - 4, 3] == SENTINEL


# ---- strides, host memory, device bands --------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_padded_stride_pinned_and_pageable_are_identical(method):
    rows, cols, res = 300, 260, 0.25
    g = geometry(rows, cols, res)
    h, w = 80, 90
    full = dem(h, w + 13, seed=9, nan_frac=0.02)
    band = full[:, 5:5 + w]                              # a view: row stride (w + 13) * 4 bytes
    gt = (-rows * res / 2 - 3.3, 1.0, 0.0, cols * res / 2 + 2.7, 0.0, -1.0)
    want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method)
    got = {}
    p = C.c_void_p()
    amb.check(_lib.lib().amb_host_alloc(C.byref(p), full.nbytes))
    try:
        pinned = np.frombuffer((C.c_uint8 * full.nbytes).from_address(p.value), np.float32).reshape(full.shape)
        pinned[...] = full
        for label, b in (("pageable", band), ("pinned", pinned[:, 5:5 + w]), ("packed", np.ascontiguousarray(band))):
            gm = sentinel_map(rows, cols, res)
            gm.from_raster("elevation", b, gt, resample=method)
            got[label] = layer_of(gm)
    finally:
        _lib.lib().amb_host_free(p)
    for label, a in got.items():
        assert same(a, want), label


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_device_band_at_4_byte_offsets(method):
    L = _lib.lib()
    rows, cols, res = 33, 29, 0.5
    g = geometry(rows, cols, res)
    h, w = 19, 21
    band = dem(h, w, seed=11, nan_frac=0.05)
    gt = (-rows * res / 2 + 0.3, 0.75, 0.0, cols * res / 2 - 0.2, 0.0, -0.75)
    want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method)
    pitch = (w + 3) * 4
    for off in (0, 4, 8, 12):
        d = Dev(h * pitch, off)
        img = np.zeros((h, w + 3), np.float32)
        img[:, :w] = band
        raw = d.all()
        raw[d.lo:d.lo + h * pitch] = img.view(np.uint8).ravel()
        if EMULATED:
            d.raw[:] = raw
        else:
            import torch
            d.raw.copy_(torch.from_numpy(raw))
        before = d.all()
        gm = sentinel_map(rows, cols, res)
        gtc = (C.c_double * 6)(*gt)
        amb.check(L.amb_import_raster_device(gm.context(), _lib.LAYER_ID["elevation"], d.ptr, w, h, pitch, gtc, 0, 0.0,
                                             _lib.RESAMPLE[method]), gm.context())
        assert same(layer_of(gm), want), off
        assert np.array_equal(d.all(), before), off          # the band and its guard bytes are only read
        for bad in (1, 2, 3):
            assert L.amb_import_raster_device(gm.context(), _lib.LAYER_ID["elevation"], d.ptr + bad, w, h, pitch, gtc,
                                              0, 0.0, 0) == _lib.AMB_ERR_INVALID_ARGUMENT


# ---- stripes, several GPUs, ordering -----------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_stripe_contexts_equal_one_whole_map_import(method):
    rows, cols, res = 45, 23, 1.0
    band = dem(30, 50, seed=5, nan_frac=0.05)
    gt = (-rows * res / 2 - 2.6, 1.1, 0.0, cols * res / 2 + 1.3, 0.0, -0.9)
    whole = sentinel_map(rows, cols, res)
    whole.from_raster("elevation", band, gt, resample=method)
    want = layer_of(whole)
    assert same(want, restate(np.full((rows, cols), SENTINEL, np.float32), geometry(rows, cols, res), band, gt, method))
    parts = []
    for c0, c1 in ((0, 1), (1, 8), (8, cols)):
        gm = sentinel_map(rows, cols, res, col_range=(c0, c1))
        gm.from_raster("elevation", band, gt, resample=method)
        parts.append(layer_of(gm))
    assert same(np.concatenate(parts, axis=1), want)


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_multi_import_on_every_visible_gpu(method):
    L = _lib.lib()
    rows, cols, res = 37, 29, 1.0
    g = geometry(rows, cols, res)
    band = dem(40, 33, seed=13, nan_frac=0.05)
    gt = (-rows * res / 2 - 1.7, 1.2, 0.0, cols * res / 2 + 2.1, 0.0, -1.1)
    want = restate(np.full((rows, cols), SENTINEL, np.float32), g, band, gt, method)
    m = C.c_void_p()
    assert L.amb_multi_create(C.byref(g), min(L.amb_device_count(), cols), C.byref(m)) == 0
    try:
        init = np.full((rows, cols), SENTINEL, np.float32, order="F")
        assert L.amb_multi_upload_layer(m, _lib.LAYER_ID["elevation"], init.ctypes.data) == 0
        assert L.amb_multi_import_raster(m, _lib.LAYER_ID["elevation"], band.ctypes.data, band.shape[1], band.shape[0],
                                         band.strides[0], (C.c_double * 6)(*gt), 0, 0.0, _lib.RESAMPLE[method]) == 0
        got = np.empty((rows, cols), np.float32, order="F")
        assert L.amb_multi_download_layer(m, _lib.LAYER_ID["elevation"], got.ctypes.data) == 0
        assert same(got, want)
    finally:
        L.amb_multi_destroy(m)


@gpu
def test_import_enqueued_right_after_process_equals_one_after_sync():
    rows, cols, res = 120, 100, 0.5
    L = _lib.lib()
    xyz = synth.point_cloud(30000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    keep, d_xyz = device_array(np.ascontiguousarray(xyz))
    band = dem(25, 30, seed=17, nan_frac=0.1)
    gt = (-10.3, 0.7, 0.0, 8.1, 0.0, -0.7)                   # a tile inside the map: the rest is the DSM's
    keep_b, d_band = device_array(band)
    sync_device()
    gtc = (C.c_double * 6)(*gt)
    results = []
    for synced in (False, True):
        gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
        gm.to_device(0)
        ctx = gm.context()
        amb.Dsm(amb.DsmSettings(), gm).process_device(d_xyz, len(xyz), gm)
        if synced:
            gm.sync()
            dsm_only = layer_of(gm)
        amb.check(L.amb_import_raster_device(ctx, _lib.LAYER_ID["elevation"], d_band, 30, 25, 120, gtc, 0, 0.0, 1), ctx)
        results.append(layer_of(gm))
    assert same(results[0], results[1])
    assert same(results[1], restate(dsm_only, geometry(rows, cols, res), band, gt, "bilinear"))
    assert not same(results[1], dsm_only)
    del keep, keep_b


# ---- the argument contract --------------------------------------------------------------------------------------------
@gpu
def test_invalid_arguments_write_nothing():
    L = _lib.lib()
    rows, cols = 6, 5
    gm = sentinel_map(rows, cols)
    ctx = gm.context()
    band = dem(4, 4, seed=1)
    d = Dev(band.nbytes)
    good = gm.geotransform()
    E = _lib.LAYER_ID["elevation"]
    # (ctx, layer, band given, width, height, stride, gt, resample)
    cases = [(None, E, True, 4, 4, 16, good, 0), (ctx, -1, True, 4, 4, 16, good, 0),
             (ctx, len(_lib.LAYER_NAMES), True, 4, 4, 16, good, 0), (ctx, E, False, 4, 4, 16, good, 0),
             (ctx, E, True, 0, 4, 16, good, 0), (ctx, E, True, 4, 0, 16, good, 0), (ctx, E, True, -1, 4, 16, good, 0),
             (ctx, E, True, 4, 4, 12, good, 0), (ctx, E, True, 4, 4, 18, good, 0), (ctx, E, True, 4, 4, 16, good, 2),
             (ctx, E, True, 4, 4, 16, good, -1), (ctx, E, True, 4, 4, 16, None, 0)]
    for bad_gt in ((good[0], good[1], 0.1, good[3], 0.0, good[5]), (good[0], good[1], 0.0, good[3], 0.1, good[5]),
                   (good[0], -1.0, 0.0, good[3], 0.0, good[5]), (good[0], good[1], 0.0, good[3], 0.0, 1.0),
                   (good[0], 0.0, 0.0, good[3], 0.0, good[5]), (np.nan,) + good[1:], good[:3] + (np.inf,) + good[4:]):
        cases.append((ctx, E, True, 4, 4, 16, bad_gt, 1))
    for c, layer_id, given, w, h, stride, gt, rs in cases:
        gtc = None if gt is None else (C.c_double * 6)(*gt)
        args = (layer_id, w, h, stride, gtc, 0, 0.0, rs)
        assert L.amb_import_raster(c, layer_id, band.ctypes.data if given else None, *args[1:]) == \
            _lib.AMB_ERR_INVALID_ARGUMENT, (layer_id, w, h, stride, gt, rs)
        assert L.amb_import_raster_device(c, layer_id, d.ptr if given else None, *args[1:]) == \
            _lib.AMB_ERR_INVALID_ARGUMENT, (layer_id, w, h, stride, gt, rs)
    assert L.amb_multi_import_raster(None, E, band.ctypes.data, 4, 4, 16, (C.c_double * 6)(*good), 0, 0.0, 0) == \
        _lib.AMB_ERR_INVALID_ARGUMENT
    # a raster that misses the map: OK, nothing written
    far = (good[0] + 1000.0,) + good[1:]
    assert L.amb_import_raster(ctx, E, band.ctypes.data, 4, 4, 16, (C.c_double * 6)(*far), 0, 0.0, 1) == 0
    assert L.amb_import_raster_device(ctx, E, d.ptr, 4, 4, 16, (C.c_double * 6)(*far), 0, 0.0, 1) == 0
    assert (layer_of(gm) == SENTINEL).all()
    with pytest.raises(KeyError):
        gm.from_raster("elevation", band, good, resample="cubic")
    with pytest.raises(amb.AmbError):
        gm.from_raster("elevation", band.astype(np.float64), good)
    with pytest.raises(amb.AmbError):
        gm.from_raster("elevation", band[:, ::2], good)
    assert (layer_of(gm) == SENTINEL).all()
    with pytest.raises(amb.AmbError) as ei:
        amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable().from_raster("elevation", band, good)
    assert "to_device()" in str(ei.value)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_raster_import.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
