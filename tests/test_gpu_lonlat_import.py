"""Longitude/latitude rasters imported into UTM maps (amb_import_raster_lonlat*, amb_import_tiff_lonlat,
amb_lonlat_positions_device, csrc/raster_import.cu; convention in include/aerial_mapper_b200.h): the cells' positions
against the mpmath oracle of tests/utm_oracle.py within 1e-11 degrees, and every import bit for bit against the
resampling rule restated in numpy from those positions.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
import utm_oracle as U  # noqa: E402
from aerial_mapper_b200 import _lib, io, synth  # noqa: E402
from test_geotiff_inflate_cpu import make_tiff  # noqa: E402
from test_gpu_geotiff_inflate import HostFile  # noqa: E402
from test_gpu_raster_export import EMULATED, Dev, device_array, sync_device  # noqa: E402
from test_gpu_raster_import import axis_table, no_data, same  # noqa: E402
from test_lonlat_import_cpu import RAFZ, lonlat_tiff  # noqa: E402

gpu = pytest.mark.gpu
SENTINEL = np.float32(-7777.25)
ARCSEC = 1.0 / 3600.0
E_ID = _lib.LAYER_ID["elevation"]


def lonlat_map(rows, cols, res, centre, col_range=None, value=SENTINEL):
    gm = amb.AerialGridMap(amb.GridMapSettings(centre[0], centre[1], rows * res, cols * res, res)).getMutable()
    assert gm.getSize() == (rows, cols)
    gm["elevation"] = np.full((rows, cols), value, np.float32, order="F") if np.ndim(value) == 0 else value
    gm.to_device(0, col_range=col_range, names=("elevation",))
    return gm


def layer_of(gm):
    gm.sync()
    gm.download(("elevation",))
    c0, c1 = gm._col_range
    return gm["elevation"][:, c0:c1].copy(order="F")


def positions(gm, epsg):
    """(lon, lat), each float64 [rows, c1 - c0], of the context's stripe from amb_lonlat_positions_device."""
    rows = gm.geometry.rows
    c0, c1 = gm._col_range
    n = rows * (c1 - c0)
    d = Dev(16 * n)
    ctx = gm.context()
    amb.check(_lib.lib().amb_lonlat_positions_device(ctx, epsg, C.c_void_p(d.ptr)), ctx)
    gm.sync()
    raw = d.all()[d.lo:d.lo + 16 * n].view(np.float64).reshape(c1 - c0, rows, 2)
    return raw[:, :, 0].T.copy(), raw[:, :, 1].T.copy()


def restate(before, lon, lat, band, gt, method, nodata=None):
    """The layer after importing `band` (float32 [H, W], geotransform gt) at the cells' (lon, lat): amb_resample's rule
    with u = (lon - gt0) / gt1, v = (lat - gt3) / gt5 per cell."""
    band = np.asarray(band, np.float32)
    h, w = band.shape
    ci, fx, _ = axis_table(lon, gt[0], gt[1], w, method)
    rj, fy, _ = axis_table(lat, gt[3], gt[5], h, method)
    out = np.array(before, np.float32, order="F", copy=True)
    cov = (ci >= 0) & (rj >= 0)
    Cc, Rc = np.clip(ci, 0, w - 1), np.clip(rj, 0, h - 1)
    if method == "nearest":
        p = band[Rc, Cc]
        ok = cov & ~no_data(p, nodata)
        out[ok] = p[ok]
        return out
    wx, wy = fx != 0, fy != 0
    C1, R1 = np.clip(ci + 1, 0, w - 1), np.clip(rj + 1, 0, h - 1)
    p00, p01, p10, p11 = band[Rc, Cc], band[Rc, C1], band[R1, Cc], band[R1, C1]
    bad = no_data(p00, nodata) | (wx & no_data(p01, nodata)) | \
        (wy & (no_data(p10, nodata) | (wx & no_data(p11, nodata))))
    d00, d01, d10, d11 = (a.astype(np.float64) for a in (p00, p01, p10, p11))
    with np.errstate(invalid="ignore", over="ignore"):
        row0 = np.where(wx, (1.0 - fx) * d00 + fx * d01, d00)
        row1 = np.where(wx, (1.0 - fx) * d10 + fx * d11, d10)
        hgt = np.where(wy, (1.0 - fy) * row0 + fy * row1, row0).astype(np.float32)
    ok = cov & ~bad
    out[ok] = hgt[ok]
    return out


def covering_gt(lon, lat, step, margin=(0.1, 0.1, 0.1, 0.1)):
    """A north-up lon/lat geotransform and its (width, height) covering the positions with margins (fractions of the
    extent; negative margins cut into the map)."""
    west, east, south, north = lon.min(), lon.max(), lat.min(), lat.max()
    lon0 = west - margin[0] * (east - west)
    lat0 = north + margin[3] * (north - south)
    w = int(np.ceil((east + margin[1] * (east - west) - lon0) / step))
    h = int(np.ceil((lat0 - (south - margin[2] * (north - south))) / step))
    return (lon0, step, 0.0, lat0, 0.0, -step), max(w, 1), max(h, 1)


def terrain(h, w, seed, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = (400.0 + 30.0 * np.sin(x / 7.0) * np.cos(y / 11.0) + rng.standard_normal((h, w))).astype(np.float32)
    if nan_frac:
        a[rng.random((h, w)) < nan_frac] = np.nan
    return a


# ---- positions -------------------------------------------------------------------------------------------------------
POSITION_MAPS = {
    # name: (epsg, centre, rows, cols, resolution)
    "32N": (32632, (612345.5, 6012000.25), 300, 24, 40.0),
    "33S": (32733, (401000.0, 7300000.0), 280, 20, 35.0),
    "rafz": (32632, RAFZ, 400, 30, 0.25),
    "across_the_zone_edge": (32632, (725000.0, 5262000.0), 260, 24, 100.0),
    "across_the_equator": (32631, (620000.0, 0.0), 270, 22, 200.0),
}


@gpu
@pytest.mark.parametrize("name", sorted(POSITION_MAPS))
def test_positions_match_the_oracle(name):
    epsg, centre, rows, cols, res = POSITION_MAPS[name]
    gm = lonlat_map(rows, cols, res, centre)
    lon, lat = positions(gm, epsg)
    assert np.isfinite(lon).all() and np.isfinite(lat).all()
    rng = np.random.default_rng(rows)
    cells = {(i, j) for i in (0, 1, rows - 2, rows - 1) for j in (0, 1, cols - 2, cols - 1)}
    cells |= {(i, j) for i in range(0, rows, 7) for j in (0, cols - 1)}
    cells |= {(i, j) for i in (0, rows - 1) for j in range(cols)}
    n_random = 300 if EMULATED else 2000 - len(cells)
    cells |= {(int(i), int(j)) for i, j in zip(rng.integers(0, rows, n_random), rng.integers(0, cols, n_random))}
    worst = 0.0
    for i, j in sorted(cells):
        x, y = gm.getPosition((i, j))
        want_lon, want_lat = U.inverse(x, y, epsg)
        worst = max(worst, abs(float(want_lon - lon[i, j])), abs(float(want_lat - lat[i, j])))
    print("%s: largest position error %.3g degrees over %d cells" % (name, worst, len(cells)))
    assert worst < 1e-11


# ---- heights, bit for bit ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_heights_equal_the_restatement(method):
    rows, cols, res = 300, 40, 2.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    cases = []
    # one arc-second tile around the map; a raster finer than the cells; rasters whose edges cut through the map
    for step, margin in [(ARCSEC, (0.1, 0.1, 0.1, 0.1)), (0.2 * ARCSEC, (0.05, 0.05, 0.05, 0.05)),
                         (0.5 * ARCSEC, (-0.3, 0.1, 0.1, -0.45)), (ARCSEC, (0.1, -0.6, -0.2, 0.1))]:
        cases.append(covering_gt(lon, lat, step, margin))
    # an origin on a cell's own position: that cell's fractions are 0 up to rounding, and snap
    gt, w, h = cases[0]
    i0, j0 = 123, 17
    snapped = (lon[i0, j0] - 20.5 * gt[1], gt[1], 0.0, lat[i0, j0] + 15.5 * gt[1], 0.0, -gt[1])
    cases.append((snapped, w + 40, h + 40))
    for k, (gt, w, h) in enumerate(cases):
        band = terrain(h, w, seed=k, nan_frac=0.03)
        before = layer_of(gm)
        gm.from_lonlat_raster("elevation", band, gt, 32632, resample=method)
        got = layer_of(gm)
        want = restate(before, lon, lat, band, gt, method)
        assert same(got, want), (method, k)
        assert not same(got, before)
    _, fx, raw = axis_table(lon, snapped[0], snapped[1], cases[-1][1], "bilinear")
    assert raw[i0, j0] < 2.0 ** -20 or raw[i0, j0] > 1 - 2.0 ** -20


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_no_data_nan_and_int16_minimum(method):
    rows, cols, res = 260, 16, 5.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    gt, w, h = covering_gt(lon, lat, ARCSEC)
    rng = np.random.default_rng(5)
    band = terrain(h, w, seed=9)
    band[rng.random((h, w)) < 0.15] = -32768.0
    band[rng.random((h, w)) < 0.05] = np.nan
    for nodata in (None, -32768.0):
        gm = lonlat_map(rows, cols, res, RAFZ)
        gm.from_lonlat_raster("elevation", band, gt, 32632, nodata=nodata, resample=method)
        want = restate(np.full((rows, cols), SENTINEL, np.float32), lon, lat, band, gt, method, nodata)
        got = layer_of(gm)
        assert same(got, want)
        assert (got == SENTINEL).any() and (got != SENTINEL).any()
        assert (got == -32768.0).any() == (nodata is None)


@gpu
def test_an_analytic_surface_within_the_bilinear_bound():
    # independent of the restatement: h(lon, lat) sampled at pixel centres, read back at the oracle's positions
    rows, cols, res = 256, 12, 20.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    step = ARCSEC
    gt, w, h = covering_gt(lon, lat, step)
    kx, ky = 2 * np.pi / 0.01, 2 * np.pi / 0.013

    def surface(x, y):
        return 500.0 + 100.0 * np.sin(kx * x) * np.cos(ky * y)

    xc = gt[0] + (np.arange(w) + 0.5) * step
    yc = gt[3] - (np.arange(h) + 0.5) * step
    band = surface(xc[None, :], yc[:, None]).astype(np.float32)
    gm.from_lonlat_raster("elevation", band, gt, 32632)
    got = layer_of(gm)
    bound = (100.0 * kx * kx * step * step + 100.0 * ky * ky * step * step) / 8 + 1e-4
    rng = np.random.default_rng(3)
    for i, j in zip(rng.integers(0, rows, 200), rng.integers(0, cols, 200)):
        x, y = gm.getPosition((int(i), int(j)))
        lo, la = (float(v) for v in U.inverse(x, y, 32632))
        assert abs(float(got[i, j]) - surface(lo, la)) <= bound, (i, j)


# ---- input paths ------------------------------------------------------------------------------------------------------
def pair(b, rows, cols, res, centre, method="bilinear", col_range=None, epsg=32632, kind=None):
    """(from_geotiff(map_epsg) layer, from_lonlat_raster of read_geotiff's array) on fresh maps."""
    import tempfile
    with tempfile.NamedTemporaryFile(suffix=".tif") as fh:
        fh.write(b)
        fh.flush()
        a, gt, file_epsg, nd = io.read_geotiff(fh.name)
    assert file_epsg == 4326
    g1 = lonlat_map(rows, cols, res, centre, col_range)
    g1.from_geotiff("elevation", b if kind is None else kind(b), resample=method, map_epsg=epsg)
    g2 = lonlat_map(rows, cols, res, centre, col_range)
    g2.from_lonlat_raster("elevation", a.astype(np.float32), gt, epsg, nodata=nd, resample=method)
    return layer_of(g1), layer_of(g2)


@gpu
@pytest.mark.parametrize("dtype,predictor", [(np.int16, 1), (np.int16, 2), (np.float32, 1), (np.float32, 3)])
@pytest.mark.parametrize("chunk", [("strips", 8), ("tiles", 32, 16)])
def test_geotiff_equals_from_lonlat_raster(dtype, predictor, chunk):
    rows, cols, res = 270, 20, 4.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    gt, w, h = covering_gt(lon, lat, 0.5 * ARCSEC, (0.4, 0.3, 0.5, 0.2))
    a = terrain(h, w, seed=2)
    if dtype == np.int16:
        a = np.round(a).astype(np.int16)
        a[::7, ::5] = -32768
        nd = -32768
    else:
        a[::9, ::4] = np.nan
        nd = None
    b = lonlat_tiff(a, gt, chunk, predictor, nodata=nd)
    for method in ("bilinear", "nearest"):
        got, want = pair(b, rows, cols, res, RAFZ, method)
        assert same(got, want)
        assert (got != SENTINEL).any()


@gpu
def test_srtm_tile_as_shipped():
    # a 3601 x 3601 one-arc-second int16 tile with PixelIsPoint georeferencing, its south-west corner at 47N 8E
    n = 3601
    y, x = np.mgrid[0:n, 0:n]
    a = (400 + 200 * np.sin(x / 300.0) * np.cos(y / 420.0)).astype(np.int16)
    a[1500:1510, 1800:1830] = -32768
    corner = (8.0 - 0.5 * ARCSEC, ARCSEC, 0.0, 48.0 + 0.5 * ARCSEC, 0.0, -ARCSEC)
    b = lonlat_tiff(a, (8.0, ARCSEC, 0.0, 48.0, 0.0, -ARCSEC), ("strips", 16), 2, point=True, nodata=-32768)
    gt, epsg, _ = io.tiff_layout(b).georeferencing()
    assert epsg == 4326 and np.allclose(gt, corner, rtol=0, atol=1e-12)
    got, want = pair(b, 400, 64, 1.0, RAFZ)
    assert same(got, want) and (got != SENTINEL).all()


@gpu
def test_projected_files_take_the_projected_import():
    rows, cols, res = 40, 30, 1.0
    gm = lonlat_map(rows, cols, res, RAFZ, value=np.asfortranarray(terrain(rows, cols, 4)))
    b = make_tiff(terrain(50, 50, 1), gt=(RAFZ[0] - 25.0, 1.0, 0.0, RAFZ[1] + 25.0, 0.0, -1.0))
    g1, g2 = lonlat_map(rows, cols, res, RAFZ), lonlat_map(rows, cols, res, RAFZ)
    g1.from_geotiff("elevation", b, map_epsg=32632)
    g2.from_geotiff("elevation", b)
    assert same(layer_of(g1), layer_of(g2))
    with pytest.raises(ValueError):
        g1.from_geotiff("elevation", b, map_epsg=32633)


@gpu
def test_from_geotiff_refuses_codes_it_cannot_import():
    from test_lonlat_import_cpu import refused_files
    gm = lonlat_map(8, 8, 1.0, RAFZ)
    for b, epsg, words in refused_files():
        with pytest.raises(ValueError) as e:
            gm.from_geotiff("elevation", b, map_epsg=epsg)
        for w in words:
            assert w in str(e.value)
    assert (layer_of(gm) == SENTINEL).all()


@gpu
def test_corrupt_chunks_outside_the_window_are_never_read():
    rows, cols, res = 260, 20, 2.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    gt, w, h = covering_gt(lon, lat, 0.5 * ARCSEC, (0.1, 0.1, 2.0, 0.1))    # rows far south of the map
    win = (C.c_int32 * 4)()
    assert _lib.lib().amb_lonlat_import_window(C.byref(gm.geometry), 0, cols, 32632, w, h, (C.c_double * 6)(*gt),
                                               win) == 0
    a = terrain(h, w, seed=3)
    rps = 8
    outside = [k for k in range((h + rps - 1) // rps) if k * rps > win[3] or (k + 1) * rps <= win[2]]
    inside = [k for k in range((h + rps - 1) // rps) if k * rps <= win[3] and (k + 1) * rps > win[2]]
    assert outside and inside
    from test_geotiff_inflate_cpu import zstream

    def bad(ks):
        return lonlat_tiff(a, gt, ("strips", rps), encode=lambda raw, k: raw[:3] + b"\xff" * 9 if k in ks else zstream(raw))

    got, want = pair(bad(set()), rows, cols, res, RAFZ)
    assert same(got, want) and (got != SENTINEL).any()
    g = lonlat_map(rows, cols, res, RAFZ)
    g.from_geotiff("elevation", bad(set(outside)), map_epsg=32632)
    assert same(layer_of(g), want)
    g = lonlat_map(rows, cols, res, RAFZ)
    with pytest.raises(amb.AmbError) as e:
        g.from_geotiff("elevation", bad({inside[len(inside) // 2]}), map_epsg=32632)
    assert e.value.status == _lib.AMB_ERR_CORRUPT_DATA
    assert (layer_of(g) == SENTINEL).all()


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_pinned_pageable_and_device_bands_are_identical(method):
    rows, cols, res = 270, 24, 3.0
    gm = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(gm, 32632)
    gt, w, h = covering_gt(lon, lat, 0.7 * ARCSEC)
    band = terrain(h, w, seed=8, nan_frac=0.02)
    padded = np.full((h, w + 5), np.float32(1e30))
    padded[:, :w] = band
    results = []
    gm.from_lonlat_raster("elevation", band, gt, 32632, resample=method)
    results.append(layer_of(gm))
    gm = lonlat_map(rows, cols, res, RAFZ)
    gm.from_lonlat_raster("elevation", padded[:, :w], gt, 32632, resample=method)
    results.append(layer_of(gm))
    p = C.c_void_p()
    assert _lib.lib().amb_host_alloc(C.byref(p), band.nbytes) == 0
    try:
        pinned = np.frombuffer((C.c_float * band.size).from_address(p.value), np.float32).reshape(h, w)
        pinned[...] = band
        gm = lonlat_map(rows, cols, res, RAFZ)
        gm.from_lonlat_raster("elevation", pinned, gt, 32632, resample=method)
        results.append(layer_of(gm))
    finally:
        _lib.lib().amb_host_free(p)
    keep, d_band = device_array(padded)
    sync_device()
    gm = lonlat_map(rows, cols, res, RAFZ)
    ctx = gm.context()
    amb.check(_lib.lib().amb_import_raster_lonlat_device(ctx, E_ID, C.c_void_p(d_band), w, h, 4 * (w + 5),
                                                         (C.c_double * 6)(*gt), 0, 0.0, _lib.RESAMPLE[method], 32632),
              ctx)
    results.append(layer_of(gm))
    del keep
    want = restate(np.full((rows, cols), SENTINEL, np.float32), lon, lat, band, gt, method)
    for r in results:
        assert same(r, want)


@gpu
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_stripes_and_multi_equal_one_whole_map_import(method):
    rows, cols, res = 260, 40, 3.0
    whole = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(whole, 32632)
    gt, w, h = covering_gt(lon, lat, 0.6 * ARCSEC, (0.1, -0.3, 0.1, 0.1))
    band = terrain(h, w, seed=6, nan_frac=0.02)
    whole.from_lonlat_raster("elevation", band, gt, 32632, resample=method)
    want = layer_of(whole)
    b = lonlat_tiff(band, gt, ("tiles", 16, 16))
    for c0, c1 in [(0, 13), (13, 14), (14, 40)]:
        s = lonlat_map(rows, cols, res, RAFZ, col_range=(c0, c1))
        s.from_lonlat_raster("elevation", band, gt, 32632, resample=method)
        assert same(layer_of(s), want[:, c0:c1])
        s2 = lonlat_map(rows, cols, res, RAFZ, col_range=(c0, c1))
        s2.from_geotiff("elevation", b, resample=method, map_epsg=32632)
        assert same(layer_of(s2), want[:, c0:c1])
    L = _lib.lib()
    if L.amb_device_count() < 2:
        pytest.skip("amb_multi_import_*_lonlat over stripes needs two devices")
    g = whole.geometry
    m = C.c_void_p()
    assert L.amb_multi_create(C.byref(g), 2, C.byref(m)) == 0
    try:
        host = np.full(g.rows * g.cols, SENTINEL)
        for call in ("raster", "tiff"):
            assert L.amb_multi_upload_layer(m, E_ID, host.ctypes.data_as(C.c_void_p)) == 0
            gtc = (C.c_double * 6)(*gt)
            if call == "raster":
                st = L.amb_multi_import_raster_lonlat(m, E_ID, band.ctypes.data_as(C.c_void_p), w, h, 4 * w, gtc, 0,
                                                      0.0, _lib.RESAMPLE[method], 32632)
            else:
                f = HostFile(b)
                layout = io.tiff_layout(b).c_layout()
                st = L.amb_multi_import_tiff_lonlat(m, E_ID, C.c_void_p(f.ptr), f.size, C.byref(layout), gtc, 0, 0.0,
                                                    _lib.RESAMPLE[method], 32632)
            assert st == 0
            out = np.empty_like(host)
            assert L.amb_multi_download_layer(m, E_ID, out.ctypes.data_as(C.c_void_p)) == 0
            assert same(out.reshape(g.rows, g.cols, order="F"), want), call
    finally:
        L.amb_multi_destroy(m)


@gpu
def test_import_enqueued_right_after_process_equals_one_after_sync():
    rows, cols, res = 280, 40, 0.5
    L = _lib.lib()
    xyz = synth.point_cloud(30000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    xyz[:, 0] += RAFZ[0]
    xyz[:, 1] += RAFZ[1]
    keep, d_xyz = device_array(np.ascontiguousarray(xyz))
    probe = lonlat_map(rows, cols, res, RAFZ)
    lon, lat = positions(probe, 32632)
    gt, w, h = covering_gt(lon, lat, 0.05 * ARCSEC, (-0.3, -0.3, -0.3, -0.3))   # a tile inside the map
    band = terrain(h, w, seed=17, nan_frac=0.1)
    keep_b, d_band = device_array(band)
    sync_device()
    gtc = (C.c_double * 6)(*gt)
    results = []
    for synced in (False, True):
        gm = amb.AerialGridMap(amb.GridMapSettings(RAFZ[0], RAFZ[1], rows * res, cols * res, res)).getMutable()
        gm.to_device(0)
        ctx = gm.context()
        amb.Dsm(amb.DsmSettings(), gm).process_device(d_xyz, len(xyz), gm)
        if synced:
            gm.sync()
            dsm_only = layer_of(gm)
        amb.check(L.amb_import_raster_lonlat_device(ctx, E_ID, d_band, w, h, 4 * w, gtc, 0, 0.0, 1, 32632), ctx)
        results.append(layer_of(gm))
    assert same(results[0], results[1])
    assert same(results[1], restate(dsm_only, lon, lat, band, gt, "bilinear"))
    assert not same(results[1], dsm_only)
    del keep, keep_b


@gpu
def test_invalid_arguments_write_nothing():
    L = _lib.lib()
    rows, cols = 8, 6
    gm = lonlat_map(rows, cols, 10.0, RAFZ)
    ctx = gm.context()
    lon, lat = positions(gm, 32632)
    good, w, h = covering_gt(lon, lat, ARCSEC)
    band = terrain(h, w, seed=1)
    d = Dev(band.nbytes)
    b = lonlat_tiff(band, good)
    f = HostFile(b)
    layout = io.tiff_layout(b).c_layout()
    stride = 4 * w
    cases = []   # (ctx, layer, band given, stride, gt, resample, epsg)
    for epsg in (4326, 0, 32600, 32661, 32700, 32761, 25832, 2056, 3857):
        cases.append((ctx, E_ID, True, stride, good, 1, epsg))
    for bad_gt in ((good[0], good[1], 0.1, good[3], 0.0, good[5]), (good[0], good[1], 0.0, good[3], 0.0, -good[5]),
                   (good[0], -good[1], 0.0, good[3], 0.0, good[5]), (np.nan,) + good[1:], None):
        cases.append((ctx, E_ID, True, stride, bad_gt, 1, 32632))
    cases += [(ctx, -1, True, stride, good, 1, 32632), (ctx, len(_lib.LAYER_NAMES), True, stride, good, 1, 32632),
              (ctx, E_ID, True, stride - 4, good, 1, 32632), (ctx, E_ID, True, stride + 2, good, 1, 32632),
              (ctx, E_ID, True, stride, good, 2, 32632), (ctx, E_ID, False, stride, good, 1, 32632),
              (None, E_ID, True, stride, good, 1, 32632)]
    for c, layer_id, given, s, gt, rs, epsg in cases:
        gtc = None if gt is None else (C.c_double * 6)(*gt)
        what = (layer_id, s, gt, rs, epsg)
        assert L.amb_import_raster_lonlat(c, layer_id, band.ctypes.data if given else None, w, h, s, gtc, 0, 0.0, rs,
                                          epsg) == _lib.AMB_ERR_INVALID_ARGUMENT, what
        assert L.amb_import_raster_lonlat_device(c, layer_id, d.ptr if given else None, w, h, s, gtc, 0, 0.0, rs,
                                                 epsg) == _lib.AMB_ERR_INVALID_ARGUMENT, what
        if s == stride:
            assert L.amb_import_tiff_lonlat(c, layer_id, C.c_void_p(f.ptr) if given else None, f.size,
                                            C.byref(layout), gtc, 0, 0.0, rs, epsg) == _lib.AMB_ERR_INVALID_ARGUMENT, what
    assert L.amb_import_raster_lonlat_device(ctx, E_ID, d.ptr + 2, w, h, stride, (C.c_double * 6)(*good), 0, 0.0, 1,
                                             32632) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_lonlat_positions_device(ctx, 4326, d.ptr) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_lonlat_positions_device(ctx, 32632, None) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_multi_import_raster_lonlat(None, E_ID, band.ctypes.data, w, h, stride, (C.c_double * 6)(*good), 0,
                                            0.0, 1, 32632) == _lib.AMB_ERR_INVALID_ARGUMENT
    # a raster that misses the map: OK, nothing written
    far = (good[0] + 5.0,) + good[1:]
    assert L.amb_import_raster_lonlat(ctx, E_ID, band.ctypes.data, w, h, stride, (C.c_double * 6)(*far), 0, 0.0, 1,
                                      32632) == 0
    assert L.amb_import_raster_lonlat_device(ctx, E_ID, d.ptr, w, h, stride, (C.c_double * 6)(*far), 0, 0.0, 1,
                                             32632) == 0
    f.free()
    assert (layer_of(gm) == SENTINEL).all()


# ---- the orthomosaic on an imported DEM --------------------------------------------------------------------------------
@gpu
def test_ortho_on_the_imported_dem_equals_ortho_on_the_uploaded_layer():
    rows, cols, res = 72, 56, 1.0
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, agl=60.0, seed=4, jitter_pos=0.5)
    for p in poses:
        p[0] += RAFZ[0]
        p[1] += RAFZ[1]
    imgs = [synth.procedural_image(k, camd["width"], camd["height"]) for k in range(len(poses))]
    a = amb.AerialGridMap(amb.GridMapSettings(RAFZ[0], RAFZ[1], rows * res, cols * res, res)).getMutable()
    a.to_device(0)
    lon, lat = positions(a, 32632)
    gt, w, h = covering_gt(lon, lat, 0.1 * ARCSEC)
    a.from_lonlat_raster("elevation", terrain(h, w, seed=12) - np.float32(300), gt, 32632)
    dem = layer_of(a)
    assert np.isfinite(dem).all()
    b = amb.AerialGridMap(amb.GridMapSettings(RAFZ[0], RAFZ[1], rows * res, cols * res, res)).getMutable()
    b["elevation"] = dem
    b.to_device(0)
    names = ("ortho", "elevation_angle", "observation_index", "elevation")
    for gm in (a, b):
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm).process(poses, imgs, gm)
        gm.sync()
        gm.download(names)
    assert (~np.isnan(a["observation_index"])).any()
    for name in names:
        assert np.array_equal(a[name], b[name], equal_nan=True), name


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_lonlat_import.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail
