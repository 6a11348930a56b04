"""The longitude/latitude import without a GPU (convention: include/aerial_mapper_b200.h, amb_import_raster_lonlat):
the mpmath oracle of tests/utm_oracle.py pinned to the exact transverse Mercator by three independent checks, the
reference's UTMtoLL against it, the host window of amb_lonlat_import_window against every tap of the oracle's positions,
and from_geotiff's refusals of EPSG codes it cannot import."""
import ctypes as C
import json
import os
import struct

import mpmath as mp
import numpy as np
import pytest

import utm_oracle as U
from aerial_mapper_b200 import _lib
from test_geotiff_inflate_cpu import make_tiff
from test_gpu_raster_import import axis_table, geometry

HERE = os.path.dirname(os.path.abspath(__file__))
RAFZ = (464980.0, 5272260.0)   # the reference's real demo, UTM 32N


def lonlat_tiff(a, gt, chunk=("strips", 16), predictor=1, point=False, nodata=None, encode=None):
    """make_tiff with the GeoKeys of a geographic WGS84 raster: GTModelType 2, GTRasterType 1 (area) or 2 (point),
    GeographicType 2048 = 4326."""
    b = make_tiff(a, predictor, chunk, gt=gt, nodata=nodata, encode=encode)
    old = struct.pack("<16H", 1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32632)
    new = struct.pack("<16H", 1, 1, 0, 3, 1024, 0, 1, 2, 1025, 0, 1, 2 if point else 1, 2048, 0, 1, 4326)
    assert b.count(old) == 1
    return b.replace(old, new)


# ---- the oracle against the exact projection ------------------------------------------------------------------------
def test_central_meridian_is_the_meridian_arc():
    # on the central meridian the projection is N = k0 M(phi), M the meridian arc: the forward series meets it, and the
    # inverse series returns the latitude
    for lat in [0.0, 1.0, 10.0, 23.4, 47.60280, 60.0, 72.0, 80.0, 84.0]:
        n = U.K0 * U.meridian_arc(lat)
        e, n_fwd = U.forward(9, lat, 32632)
        assert abs(e - 500000) < mp.mpf("1e-12")
        assert abs(n_fwd - n) < mp.mpf("1e-9"), lat
        lon, lat_inv = U.inverse(500000, n, 32632)
        assert abs(lon - 9) < mp.mpf("1e-20")
        assert abs(lat_inv - lat) * mp.pi / 180 * 6.4e6 < mp.mpf("1e-9"), lat


def test_psi_and_lambda_satisfy_cauchy_riemann():
    # psi + i lambda is an analytic function of N + i E: with the meridian values above, that pins the whole projection
    rng = np.random.default_rng(7)
    h = mp.mpf("1e-3")
    for _ in range(12):
        lat = rng.uniform(0.5, 80.0)
        dlon = rng.uniform(-3.0, 3.0)
        e0, n0 = U.forward(9 + dlon, lat, 32632)

        def f(de, dn):
            lon, la = U.inverse(e0 + de, n0 + dn, 32632)
            return U.isometric_latitude(la), mp.radians(lon)

        pn1, ln1 = f(0, h)
        pn0, ln0 = f(0, -h)
        pe1, le1 = f(h, 0)
        pe0, le0 = f(-h, 0)
        psi_n, lam_n = (pn1 - pn0) / (2 * h), (ln1 - ln0) / (2 * h)
        psi_e, lam_e = (pe1 - pe0) / (2 * h), (le1 - le0) / (2 * h)
        scale = abs(psi_n) + abs(psi_e)
        assert abs(psi_n - lam_e) < mp.mpf("1e-15") * scale, (lat, dlon)
        assert abs(psi_e + lam_n) < mp.mpf("1e-15") * scale, (lat, dlon)


@pytest.mark.parametrize("epsg", [32632, 32733])
def test_forward_then_inverse_is_the_identity(epsg):
    rng = np.random.default_rng(epsg)
    for _ in range(40):
        e = rng.uniform(160000.0, 840000.0)
        n = rng.uniform(0.0, 9300000.0) if epsg < 32700 else rng.uniform(1000000.0, 10000000.0)
        lon, lat = U.inverse(e, n, epsg)
        e2, n2 = U.forward(lon, lat, epsg)
        assert abs(e2 - e) < mp.mpf("1e-9") and abs(n2 - n) < mp.mpf("1e-9"), (e, n)


def test_rafz_origin():
    lon, lat = U.inverse(RAFZ[0], RAFZ[1], 32632)
    assert abs(lat - mp.mpf("47.603")) < 1e-3 and abs(lon - mp.mpf("8.534")) < 1e-3


def test_reference_utmtoll_agrees_within_the_stated_bound():
    # tests/golden/utm_reference.json: the reference's UTMtoLL (a truncated series with a 10-digit eccentricity) at fixed
    # points, recorded by tests/golden/make_utm_golden.py; DESIGN.md states the bound
    path = os.path.join(HERE, "golden", "utm_reference.json")
    data = json.load(open(path))
    cases = data["points"]
    assert len(cases) >= 20
    worst = 0.0
    for c in cases:
        lon, lat = U.inverse(c["easting"], c["northing"], c["epsg"])
        # metres on the ellipsoid, roughly
        d = float(mp.hypot((c["lat"] - lat) * 111320, (c["lon"] - lon) * 111320 * mp.cos(mp.radians(lat))))
        assert d < data["bound_m"], c
        worst = max(worst, d)
    print("largest reference - oracle distance: %.4g m" % worst)


# ---- the host window -------------------------------------------------------------------------------------------------
WINDOW_MAPS = {
    # name: (epsg, centre, cells, resolution)
    "rafz": (32632, RAFZ, (48, 40), 250.0),
    "across_the_zone_edge": (32632, (725000.0, 5262000.0), (40, 30), 500.0),
    "3_degrees_past_the_edge": (32632, (955000.0, 5280000.0), (40, 30), 500.0),
    "equator_north_zone": (32631, (620000.0, 0.0), (36, 44), 1000.0),
    "equator_south_zone": (32733, (380000.0, 10000000.0), (36, 44), 1000.0),
}


def oracle_positions(g, epsg, c0=0, c1=None):
    """lon, lat [rows, c1 - c0] of every cell, by the oracle (float64 of the mpmath values)."""
    c1 = g.cols if c1 is None else c1
    lon = np.empty((g.rows, c1 - c0))
    lat = np.empty_like(lon)
    for i in range(g.rows):
        for j in range(c0, c1):
            x, y = C.c_double(), C.c_double()
            _lib.lib().amb_geometry_position(C.byref(g), i, j, C.byref(x), C.byref(y))
            a, b = U.inverse(x.value, y.value, epsg)
            lon[i, j - c0], lat[i, j - c0] = float(a), float(b)
    return lon, lat


def window(g, epsg, w, h, gt, c0=0, c1=None):
    win = (C.c_int32 * 4)()
    st = _lib.lib().amb_lonlat_import_window(C.byref(g), c0, g.cols if c1 is None else c1, epsg, w, h,
                                             (C.c_double * 6)(*gt), win)
    return st, tuple(win)


@pytest.mark.parametrize("name", sorted(WINDOW_MAPS))
def test_window_covers_every_tap_of_the_oracle_positions(name):
    epsg, centre, (rows, cols), res = WINDOW_MAPS[name]
    g = geometry(rows, cols, res, centre)
    half = cols // 2
    pos = {(0, cols): oracle_positions(g, epsg)}
    pos[(half, cols)] = (pos[(0, cols)][0][:, half:], pos[(0, cols)][1][:, half:])
    lon, lat = pos[(0, cols)]
    west, east, south, north = lon.min(), lon.max(), lat.min(), lat.max()
    covered_some = 0
    # rasters covering the map with a margin, cutting through it on every side, and missing it
    for step in (1 / 3600.0, 0.004, 0.05):
        for (fw, fe, fs, fn) in [(-0.1, 1.1, -0.1, 1.1), (0.3, 1.2, -0.2, 0.6), (-0.2, 0.45, 0.55, 1.3),
                                 (0.4, 0.6, 0.4, 0.6), (1.05, 1.5, 0.0, 1.0)]:
            lon0 = west + fw * (east - west)
            lat0 = south + fn * (north - south)
            w = max(1, int(np.ceil((fe - fw) * (east - west) / step)))
            h = max(1, int(np.ceil((fn - fs) * (north - south) / step)))
            gt = (lon0, step, 0.0, lat0, 0.0, -step)
            for (c0, c1), (lo, la) in pos.items():
                st, win = window(g, epsg, w, h, gt, c0, c1)
                assert st == 0
                for method in ("nearest", "bilinear"):
                    ci, fx, _ = axis_table(lo, gt[0], gt[1], w, method)
                    rj, fy, _ = axis_table(la, gt[3], gt[5], h, method)
                    cov = (ci >= 0) & (rj >= 0)
                    if not cov.any():
                        continue
                    assert win[0] >= 0, (name, step, fw, method)
                    covered_some += 1
                    assert win[0] <= ci[cov].min() and (ci + (fx != 0))[cov].max() <= win[1], (name, step, win)
                    assert win[2] <= rj[cov].min() and (rj + (fy != 0))[cov].max() <= win[3], (name, step, win)
                    assert 0 <= win[0] <= win[1] < w and 0 <= win[2] <= win[3] < h
    assert covered_some > 20


def test_window_of_a_raster_that_misses_the_map_and_bad_arguments():
    g = geometry(20, 20, 100.0, RAFZ)
    gt = (20.0, 0.001, 0.0, 47.7, 0.0, -0.001)
    assert window(g, 32632, 100, 100, gt) == (0, (-1, -1, -1, -1))
    for epsg in (4326, 32600, 32661, 32700, 32761, 25832, 2056):
        assert window(g, epsg, 100, 100, gt)[0] == _lib.AMB_ERR_INVALID_ARGUMENT
    for bad in [(8.0, 0.001, 0.0, 47.7, 0.0, 0.001), (8.0, 0.001, 0.1, 47.7, 0.0, -0.001), (8.0, np.nan, 0, 47, 0, -1)]:
        assert window(g, 32632, 100, 100, bad)[0] == _lib.AMB_ERR_INVALID_ARGUMENT


# ---- from_geotiff's EPSG codes ---------------------------------------------------------------------------------------
def refused_files():
    """(file, map_epsg, words the ValueError names) that from_geotiff(map_epsg=...) refuses."""
    a = np.zeros((8, 8), np.float32)
    ll = lonlat_tiff(a, (8.5, 0.001, 0.0, 47.61, 0.0, -0.001))
    utm = (464000.0, 1.0, 0.0, 5273000.0, 0.0, -1.0)
    utm33 = make_tiff(a, gt=utm).replace(struct.pack("<4H", 3072, 0, 1, 32632), struct.pack("<4H", 3072, 0, 1, 32633))
    no_code = make_tiff(a, gt=utm).replace(   # user-defined: no EPSG code
        struct.pack("<4H", 3072, 0, 1, 32632), struct.pack("<4H", 3072, 0, 1, 32767))
    return [(utm33, 32632, ("32633", "32632")), (ll, 25832, ("25832",)), (ll, 4326, ("4326",)),
            (no_code, 32632, ("none", "32632")), (ll, 32600, ("32600",))]


def test_the_epsg_decision_of_from_geotiff():
    # the decision from_geotiff takes on the file's code (the GPU tests run from_geotiff itself on these files)
    from aerial_mapper_b200 import api, io
    for b, epsg, words in refused_files():
        with pytest.raises(ValueError) as e:
            api._lonlat_source(io.tiff_layout(b).georeferencing()[1], epsg)
        for w in words:
            assert w in str(e.value)
    a = np.zeros((8, 8), np.float32)
    ll = lonlat_tiff(a, (8.5, 0.001, 0.0, 47.61, 0.0, -0.001))
    utm = make_tiff(a, gt=(464000.0, 1.0, 0.0, 5273000.0, 0.0, -1.0))
    for b, epsg, want in [(ll, 32632, True), (ll, 32733, True), (utm, 32632, False), (utm, None, False),
                          (ll, None, False)]:
        assert api._lonlat_source(io.tiff_layout(b).georeferencing()[1], epsg) is want


def test_point_geokeys_are_shifted_by_read_geotiff(tmp_path):
    from aerial_mapper_b200 import io
    a = np.arange(12, dtype=np.int16).reshape(3, 4)
    step = 1 / 3600.0
    for point in (False, True):
        b = lonlat_tiff(a, (8.0, step, 0.0, 48.0, 0.0, -step), point=point)
        gt, epsg, _ = io.tiff_layout(b).georeferencing()
        assert epsg == 4326
        shift = step / 2 if point else 0.0
        assert gt[0] == 8.0 - shift and gt[3] == 48.0 + shift
