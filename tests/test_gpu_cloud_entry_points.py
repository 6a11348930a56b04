"""Every DSM and OrthoFromPcl entry point of the C ABI on the same cloud: host, `_device`, `_device_ids`, the sharded
ones on a context without a communicator, and amb_multi_* with one device must write the same layer bits, return the
statuses of their argument checks, report the same timings fields, and end the way each is documented to end
(synchronous or not, coincident points reported at once or by amb_sync).  A Dsm's own settings reach all its calls.

The tests also run on the emulated kernels (tests/emu) through tests/test_emulated_kernels.py."""
import ctypes as C
import os

import numpy as np
import pytest

import aerial_mapper_b200 as amb
from aerial_mapper_b200 import _lib, synth

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
ROWS, COLS, RES = 72, 56, 0.5
RADIUS, CE, CN = 2, 0.75, -0.5
OK, EMPTY, COINCIDENT, INVALID = (_lib.AMB_OK, _lib.AMB_ERR_EMPTY, _lib.AMB_ERR_COINCIDENT_POINT,
                                  _lib.AMB_ERR_INVALID_ARGUMENT)


def L():
    return amb.lib()


def cloud(n=4000, seed=17):
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(-ROWS * RES / 2 - 1.0, ROWS * RES / 2 + 1.0, n) + CN,
                rng.uniform(-COLS * RES / 2 - 1.0, COLS * RES / 2 + 1.0, n) + CE, rng.uniform(0.0, 5.0, n)]
    inten = rng.integers(0, 256, n).astype(np.int32)
    return np.ascontiguousarray(xyz), inten, np.arange(n, dtype=np.uint64)


def on_device(a):
    """(keep-alive object, device pointer) of a copy of `a`; the emulated kernels take host memory as device memory."""
    a = np.ascontiguousarray(a)
    if EMULATED:
        return a, a.ctypes.data
    import torch
    t = torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).to("cuda:0")
    return t, t.data_ptr()


def grid_map():
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, ROWS * RES, COLS * RES, RES)).getMutable()
    gm.context(0)
    return gm


def layer(gm, name):
    gm.sync()
    gm.download((name,))
    return gm[name].copy()


def host(a):
    return a.ctypes.data


DSM_ROUTES = ("host", "device", "device_ids", "sharded_device", "sharded", "multi")


def run_dsm(route, xyz, ids):
    n = len(xyz)
    if route == "multi":
        return run_multi(lambda m: L().amb_multi_dsm_process(m, host(xyz), n, RADIUS, CE, CN), "elevation")
    gm = grid_map()
    ctx = gm.context()
    dx, px = on_device(xyz)
    di, pi = on_device(ids)
    st = {"host": lambda: L().amb_dsm_process(ctx, host(xyz), n, RADIUS, CE, CN),
          "device": lambda: L().amb_dsm_process_device(ctx, px, n, RADIUS, CE, CN),
          "device_ids": lambda: L().amb_dsm_process_device_ids(ctx, px, pi, n, RADIUS, CE, CN),
          "sharded_device": lambda: L().amb_dsm_process_sharded_device(ctx, px, pi, n, RADIUS, CE, CN, 1000),
          "sharded": lambda: L().amb_dsm_process_sharded(ctx, host(xyz), host(ids), n, RADIUS, CE, CN, 1000)}[route]()
    assert st == OK, route
    return layer(gm, "elevation"), gm


PCL_ROUTES = ("host", "device", "device_ids", "sharded_device", "sharded", "multi")


def run_pcl(route, xyz, inten, ids, adaptive):
    n = len(xyz)
    if route == "multi":
        return run_multi(lambda m: L().amb_multi_ortho_from_pcl_process(m, host(xyz), host(inten), n, RADIUS, adaptive),
                         "ortho")
    gm = grid_map()
    ctx = gm.context()
    dx, px = on_device(xyz)
    dv, pv = on_device(inten)
    di, pi = on_device(ids)
    st = {"host": lambda: L().amb_ortho_from_pcl_process(ctx, host(xyz), host(inten), n, RADIUS, adaptive),
          "device": lambda: L().amb_ortho_from_pcl_process_device(ctx, px, pv, n, RADIUS, adaptive),
          "device_ids": lambda: L().amb_ortho_from_pcl_process_device_ids(ctx, px, pv, pi, n, RADIUS, adaptive),
          "sharded_device": lambda: L().amb_ortho_from_pcl_process_sharded_device(ctx, px, pv, pi, n, RADIUS, 1000),
          "sharded": lambda: L().amb_ortho_from_pcl_process_sharded(ctx, host(xyz), host(inten), host(ids), n, RADIUS,
                                                                    1000)}[route]()
    assert st == OK, route
    return layer(gm, "ortho"), gm


def run_multi(process, name):
    gm = grid_map()                                   # for its geometry
    m = C.c_void_p()
    amb.check(L().amb_multi_create(C.byref(gm.geometry), 1, C.byref(m)))
    try:
        assert L().amb_multi_size(m) == 1
        assert process(m) == OK
        assert L().amb_multi_sync(m) == OK
        out = np.full((ROWS, COLS), np.nan, np.float32, order="F")
        amb.check(L().amb_multi_download_layer(m, _lib.LAYER_ID[name], out.ctypes.data))
    finally:
        L().amb_multi_destroy(m)
    return out, None


def same_bits(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- the same layer bits from every route ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_dsm_every_entry_point_writes_the_same_elevation():
    xyz, _, ids = cloud()
    ref, _ = run_dsm("host", xyz, ids)
    assert np.isfinite(ref).sum() > 0.9 * ref.size
    for route in DSM_ROUTES[1:]:
        got, _ = run_dsm(route, xyz, ids)
        assert same_bits(got, ref), route


@pytest.mark.gpu
@pytest.mark.parametrize("adaptive", [0, 1])
def test_ortho_from_pcl_every_entry_point_writes_the_same_ortho(adaptive):
    xyz, inten, ids = cloud(seed=23)
    ref, _ = run_pcl("host", xyz, inten, ids, adaptive)
    assert (ref != 255.0).sum() > 0.9 * ref.size
    # the sharded entry points take no adaptive interpolation (no rank of a sharded cloud holds the whole cloud)
    routes = [r for r in PCL_ROUTES[1:] if not (adaptive and r.startswith("sharded"))]
    for route in routes:
        got, _ = run_pcl(route, xyz, inten, ids, adaptive)
        assert same_bits(got, ref), (route, adaptive)


# ---- argument checks, in their order ---------------------------------------------------------------------------------
@pytest.mark.gpu
def test_status_of_every_argument_check():
    xyz, inten, ids = cloud(n=64)
    n = len(xyz)
    gm = grid_map()
    ctx = gm.context()
    dx, px = on_device(xyz)
    dv, pv = on_device(inten)
    di, pi = on_device(ids)
    hx, hv, hi = host(xyz), host(inten), host(ids)
    cases = [
        # no context
        (L().amb_dsm_process(None, hx, n, RADIUS, CE, CN), INVALID),
        (L().amb_dsm_process_device(None, px, n, RADIUS, CE, CN), INVALID),
        (L().amb_dsm_process_sharded(None, hx, hi, n, RADIUS, CE, CN, 1000), INVALID),
        (L().amb_ortho_from_pcl_process(None, hx, hv, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_sharded_device(None, px, pv, pi, n, RADIUS, 1000), INVALID),
        # n == 0 is checked before the pointers of a whole cloud ...
        (L().amb_dsm_process(ctx, None, 0, RADIUS, CE, CN), EMPTY),
        (L().amb_dsm_process_device(ctx, None, 0, RADIUS, CE, CN), EMPTY),
        (L().amb_dsm_process_device_ids(ctx, None, None, 0, RADIUS, CE, CN), EMPTY),
        (L().amb_ortho_from_pcl_process(ctx, None, None, 0, RADIUS, 0), EMPTY),
        (L().amb_ortho_from_pcl_process_device(ctx, None, None, 0, RADIUS, 1), EMPTY),
        # ... except the ids of amb_ortho_from_pcl_process_device_ids, which are required
        (L().amb_ortho_from_pcl_process_device_ids(ctx, px, pv, None, 0, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_device_ids(ctx, px, pv, None, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_device_ids(ctx, px, pv, pi, 0, RADIUS, 0), EMPTY),
        # null inputs
        (L().amb_dsm_process(ctx, None, n, RADIUS, CE, CN), INVALID),
        (L().amb_dsm_process_device(ctx, None, n, RADIUS, CE, CN), INVALID),
        (L().amb_dsm_process_device_ids(ctx, None, pi, n, RADIUS, CE, CN), INVALID),
        (L().amb_ortho_from_pcl_process(ctx, None, hv, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process(ctx, hx, None, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_device(ctx, None, pv, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_device(ctx, px, None, n, RADIUS, 0), INVALID),
        (L().amb_ortho_from_pcl_process_device_ids(ctx, px, None, pi, n, RADIUS, 0), INVALID),
        # sharded: every pointer (ids included) and the radius before n; without a communicator n == 0 is empty
        (L().amb_dsm_process_sharded_device(ctx, None, pi, 0, RADIUS, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded_device(ctx, px, None, 0, RADIUS, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded_device(ctx, px, pi, 0, 0, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded_device(ctx, px, pi, n, 0, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded_device(ctx, px, pi, 0, RADIUS, CE, CN, 1000), EMPTY),
        (L().amb_dsm_process_sharded(ctx, None, hi, 0, RADIUS, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded(ctx, hx, None, 0, RADIUS, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded(ctx, hx, hi, 0, 0, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded(ctx, hx, hi, n, 0, CE, CN, 1000), INVALID),
        (L().amb_dsm_process_sharded(ctx, hx, hi, 0, RADIUS, CE, CN, 1000), EMPTY),
        (L().amb_ortho_from_pcl_process_sharded_device(ctx, None, pv, pi, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded_device(ctx, px, None, pi, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded_device(ctx, px, pv, None, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded_device(ctx, px, pv, pi, n, 0, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded_device(ctx, px, pv, pi, 0, RADIUS, 1000), EMPTY),
        (L().amb_ortho_from_pcl_process_sharded(ctx, None, hv, hi, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded(ctx, hx, None, hi, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded(ctx, hx, hv, None, 0, RADIUS, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded(ctx, hx, hv, hi, n, 0, 1000), INVALID),
        (L().amb_ortho_from_pcl_process_sharded(ctx, hx, hv, hi, 0, RADIUS, 1000), EMPTY),
        # the DSM's device ids are optional (array positions)
        (L().amb_dsm_process_device_ids(ctx, px, None, n, RADIUS, CE, CN), OK),
    ]
    for k, (got, want) in enumerate(cases):
        assert got == want, (k, got, want)
    assert L().amb_sync(ctx) == OK


# ---- a point on a cell centre: reported at once by amb_dsm_process only ----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("route", ["host", "device", "sharded"])
def test_coincident_point_is_reported_at_once_by_the_host_dsm_entry_only(route):
    xyz, _, ids = cloud(n=800, seed=31)
    qx, qy = synth.grid_positions(ROWS, COLS, RES)
    xyz[7, :2] = (qx[20] + CN, qy[30] + CE)          # shifted by the centre, exactly on the centre of cell (20, 30)
    gm = grid_map()
    ctx = gm.context()
    n = len(xyz)
    if route == "host":
        assert L().amb_dsm_process(ctx, host(xyz), n, RADIUS, CE, CN) == COINCIDENT
    elif route == "device":
        dx, px = on_device(xyz)
        assert L().amb_dsm_process_device(ctx, px, n, RADIUS, CE, CN) == OK
        assert L().amb_sync(ctx) == COINCIDENT
    else:
        assert L().amb_dsm_process_sharded(ctx, host(xyz), host(ids), n, RADIUS, CE, CN, 1000) == OK
        assert L().amb_sync(ctx) == COINCIDENT
    assert L().amb_sync(ctx) == OK                   # reported once, then cleared


# ---- timings ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="events of the emulated runtime measure nothing")
def test_h2d_time_only_for_host_clouds_and_the_same_launches_on_every_route():
    xyz, inten, ids = cloud(seed=41)
    t = {}
    for route in ("host", "device", "device_ids", "sharded_device", "sharded"):
        t["dsm", route] = run_dsm(route, xyz, ids)[1].timings()
        t["pcl", route] = run_pcl(route, xyz, inten, ids, 0)[1].timings()
    for kind in ("dsm", "pcl"):
        assert t[kind, "host"]["dsm_h2d_ms"] > 0.0, kind
        # a sharded share is uploaded before the timed region, whose "h2d" phase is the halo exchange: none here
        for route in ("device", "device_ids", "sharded_device", "sharded"):
            assert t[kind, route]["dsm_h2d_ms"] == 0.0, (kind, route)
            assert t[kind, route]["dsm_kernel_launches"] == t[kind, "host"]["dsm_kernel_launches"], (kind, route)
        assert t[kind, "host"]["dsm_kernel_launches"] > 0


# ---- a Dsm's own settings reach every one of its calls ---------------------------------------------------------------
@pytest.mark.gpu
def test_a_dsm_without_debug_leaves_no_debug_record_on_the_map_after_its_sharded_call():
    xyz, _, ids = cloud(n=1500, seed=43)
    gm = grid_map()
    first = amb.Dsm(amb.DsmSettings(interpolation_radius=RADIUS), gm)
    first.debug = True
    first.process(xyz, gm)
    assert first.last_debug is not None
    second = amb.Dsm(amb.DsmSettings(interpolation_radius=RADIUS), gm)
    second.process_sharded(xyz, ids, gm, 1000)
    gm.sync()
    assert L().amb_dsm_download_debug(gm.context(), None, None) == INVALID
