"""GPU parity of the DSM path: the CUDA library through the C ABI (aerial_mapper_b200.Dsm = dsm::Dsm mirror)
against the CPU oracle on the same seeded inputs, the golden fixture, and size-independent properties at scale.

Bars: neighbour counts, retry-threshold indices and the NaN mask are integer-exact in BOTH arithmetic modes of the gather
(amb_dsm_set_precision; the whole module runs once per mode, AMB_DSM_PRECISION):
  f64  elevation <= 1 float32 ulp from the oracle (bit-identical up to double summation order)
  f32  (library default) float32 weights / sums from tile-local coordinates: elevation within 1e-6 relative and <= 4 ulp
       on these terrain-like clouds.  The library guarantees 1e-4 relative in every cell: a cell whose float32 height a
       rounding-error bound cannot place within it is evaluated in double (test_gpu_dsm_heights.py tests that bound
       where float32 fails).  Measured: > 99.9 % of the cells bit-identical to the f64 mode."""
import ctypes as C
import os

import numpy as np
import pytest

from common import GOLDEN, ulp_diff
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

REL = 1e-6
PRECISION = os.environ.get("AMB_DSM_PRECISION", "f32").lower()
MAX_ULP = 1 if PRECISION == "f64" else 4


def gpu_dsm(rows, cols, res, xyz, radius=1, ce=0.0, cn=0.0, pos=(0.0, 0.0), elevation=None, col_range=None):
    gm = amb.AerialGridMap(amb.GridMapSettings(pos[0], pos[1], rows * res, cols * res, res)).getMutable()
    assert gm.getSize() == (rows, cols)
    if elevation is not None:
        gm["elevation"] = elevation
    if col_range is not None:
        gm.context(0, col_range)
    d = amb.Dsm(amb.DsmSettings(interpolation_radius=radius, center_easting=ce, center_northing=cn), gm)
    d.debug = True
    d.process(xyz, gm)
    return gm, d.last_debug


def oracle_dsm(rows, cols, res, xyz, radius=1, ce=0.0, cn=0.0, pos=(0.0, 0.0), elevation=None):
    g = po.make_geometry(rows, cols, res, pos[0], pos[1])
    e = np.full((rows, cols), np.nan, np.float32, order="F")
    if elevation is not None:
        e[...] = elevation
    st, cnt, lvl, _ = po.dsm_process(g, e, xyz, radius=radius, center_easting=ce, center_northing=cn, debug=True)
    assert st == 0
    return e, cnt, lvl


def assert_parity(gm, dbg, e, cnt, lvl):
    gc, gl = dbg
    ge = gm["elevation"]
    assert np.array_equal(gl, lvl), "retry-threshold index differs in %d cells" % int((gl != lvl).sum())
    touched = lvl >= 0
    assert np.array_equal(gc[touched], cnt[touched]), "neighbour count differs"
    assert (gc[~touched] == 0).all()
    assert np.array_equal(np.isnan(ge), np.isnan(e))
    ok = ~np.isnan(e)
    assert np.allclose(ge[ok], e[ok], rtol=REL, atol=0.0)
    assert ulp_diff(ge, e).max() <= MAX_ULP


CASES = [
    # rows, cols, res, n, seed, holes, radius
    (256, 256, 1.0, 100000, 1, 0, 1),      # BASELINE config C1
    (300, 200, 0.25, 40000, 5, 6, 1),      # holes -> every retry level and permanent NaN
    (100, 130, 0.5, 20000, 6, 0, 2),       # radius 2 m^2
    (97, 61, 0.4, 9000, 8, 2, 1),          # tile-unaligned sizes, odd resolution
    (33, 500, 1.0, 30000, 9, 0, 3),
    (64, 64, 0.1, 3000, 10, 0, 1),         # window half-width 10 cells
    (40, 40, 2.0, 20000, 11, 0, 1),        # cells larger than the search radius
    (50, 50, 1.0, 12000, 12, 0, 8),        # radius > 7: exactly one retry, no growth
]


@pytest.mark.parametrize("rows,cols,res,n,seed,holes,radius", CASES)
def test_matches_oracle(rows, cols, res, n, seed, holes, radius):
    xyz = synth.point_cloud(n, rows * res / 2 + 2.0, cols * res / 2 + 2.0, seed, holes=holes,
                            hole_sides=(rows * res / 30, rows * res / 6))
    gm, dbg = gpu_dsm(rows, cols, res, xyz, radius)
    assert_parity(gm, dbg, *oracle_dsm(rows, cols, res, xyz, radius))


def test_golden_fixture():
    z = np.load(os.path.join(GOLDEN, "dsm_96x80.npz"))
    rows, cols, res = int(z["rows"]), int(z["cols"]), float(z["res"])
    gm, (gc, gl) = gpu_dsm(rows, cols, res, z["xyz"])
    assert np.array_equal(gl, z["threshold_index"])
    t = gl >= 0
    assert np.array_equal(gc[t], z["neighbour_count"][t])
    assert np.array_equal(np.isnan(gm["elevation"]), np.isnan(z["elevation"]))
    assert ulp_diff(gm["elevation"], z["elevation"]).max() <= MAX_ULP


def test_map_offset_and_center_shift():
    xyz = synth.point_cloud(15000, 30.0, 20.0, seed=14, center=(5000.0 + 7.0, -3000.0 - 2.0))
    kw = dict(ce=-2.0, cn=7.0, pos=(5000.0, -3000.0))
    gm, dbg = gpu_dsm(110, 70, 0.5, xyz, 1, **kw)
    assert_parity(gm, dbg, *oracle_dsm(110, 70, 0.5, xyz, 1, **kw))


def test_non_finite_heights_only_touch_the_cells_they_reach():
    # the reference keeps z = +-inf / NaN points (its loader only requires z > -100): they poison exactly the cells whose
    # ball contains them — a point out of reach must leave a cell's sums untouched (round-1 advisor finding)
    xyz = synth.point_cloud(4000, 34.0, 34.0, seed=23)
    xyz[7, 2] = np.inf
    xyz[1234, 2] = -np.inf
    xyz[2500, 2] = np.nan
    gm, dbg = gpu_dsm(64, 64, 1.0, xyz)
    e, cnt, lvl = oracle_dsm(64, 64, 1.0, xyz)
    ge = gm["elevation"]
    assert np.array_equal(dbg[1], lvl)
    assert np.array_equal(np.isnan(ge), np.isnan(e)) and np.array_equal(np.isinf(ge), np.isinf(e))
    fin = np.isfinite(e)
    assert fin.sum() > 3000 and (~fin).sum() >= 3
    assert np.array_equal(np.sign(ge[~fin & ~np.isnan(e)]), np.sign(e[~fin & ~np.isnan(e)]))
    assert ulp_diff(ge[fin], e[fin]).max() <= MAX_ULP


def test_points_outside_the_map_still_count():
    # the reference's kd-tree holds every point: points beyond the border contribute to edge cells
    xyz = synth.point_cloud(8000, 30.0, 30.0, seed=15)   # map is 40 x 40 m, cloud 60 x 60 m
    gm, dbg = gpu_dsm(40, 40, 1.0, xyz)
    assert_parity(gm, dbg, *oracle_dsm(40, 40, 1.0, xyz))


def test_repeated_process_keeps_untouched_cells():
    a = synth.point_cloud(3000, 10.0, 20.0, seed=16, center=(-10.0, 0.0))
    b = synth.point_cloud(3000, 10.0, 20.0, seed=17, center=(10.0, 0.0))
    b[:, 2] += 40.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 40.0, 40.0, 0.5)).getMutable()
    d = amb.Dsm(amb.DsmSettings(), gm)
    d.process(a, gm)
    d.process(b, gm)
    e, _, _ = oracle_dsm(80, 80, 0.5, a)
    e, _, _ = oracle_dsm(80, 80, 0.5, b, elevation=e)
    assert np.array_equal(np.isnan(gm["elevation"]), np.isnan(e))
    assert ulp_diff(gm["elevation"], e).max() <= MAX_ULP


def test_resident_map_matches_host_mode():
    xyz = synth.point_cloud(20000, 25.0, 25.0, seed=18, holes=3, hole_sides=(2.0, 8.0))
    host, _ = gpu_dsm(100, 100, 0.5, xyz)
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 50.0, 50.0, 0.5)).getMutable()
    gm.to_device(0)
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    assert np.isnan(gm["elevation"]).all()          # host copy untouched until download
    gm.download(("elevation",))
    assert np.array_equal(gm["elevation"].view(np.uint32), host["elevation"].view(np.uint32))


def test_run_to_run_and_stripe_determinism():
    # the in-bin canonical order makes every output bit independent of atomic scheduling and of the striping
    xyz = synth.point_cloud(60000, 40.0, 30.0, seed=19, holes=4, hole_sides=(2.0, 9.0))
    full1, _ = gpu_dsm(160, 120, 0.5, xyz)
    full2, _ = gpu_dsm(160, 120, 0.5, xyz)
    assert np.array_equal(full1["elevation"].view(np.uint32), full2["elevation"].view(np.uint32))
    for c0, c1 in [(0, 30), (30, 77), (77, 120)]:
        part, (pc, pl) = gpu_dsm(160, 120, 0.5, xyz, col_range=(c0, c1))
        assert np.array_equal(part["elevation"][:, c0:c1].view(np.uint32),
                              full1["elevation"][:, c0:c1].view(np.uint32))
        outside = np.ones(120, bool)
        outside[c0:c1] = False
        assert np.isnan(part["elevation"][:, outside]).all()   # other stripes are not this context's to write


def test_errors():
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 8.0, 8.0, 1.0)).getMutable()
    d = amb.Dsm(amb.DsmSettings(), gm)
    gm["elevation"] = 3.25
    d.process(np.zeros((0, 3)), gm)                      # dsm.cc:189-192: warn + return
    assert (gm["elevation"] == 3.25).all()
    qx, qy = synth.grid_positions(8, 8, 1.0)
    with pytest.raises(amb.AmbError) as ei:
        d.process(np.array([[qx[2], qy[5], 1.0], [0.1, 0.2, 0.3]]), gm)
    assert ei.value.status == -3                         # CHECK(distances[i] > 0.0), dsm.cc:165
    with pytest.raises(amb.AmbError):
        amb.Dsm(amb.DsmSettings(interpolation_radius=0), gm).process(np.ones((2, 3)), gm)


def test_clustered_points_overflow_the_shared_memory_stage():
    # 40k points inside one 32x32 tile: the tile falls back to reading its bins from global memory
    rng = np.random.default_rng(20)
    xyz = np.c_[rng.uniform(-3, 3, 40000), rng.uniform(-3, 3, 40000), rng.uniform(90, 110, 40000)]
    gm, dbg = gpu_dsm(64, 64, 0.25, xyz)
    assert_parity(gm, dbg, *oracle_dsm(64, 64, 0.25, xyz))


# ---- size-independent properties at BASELINE-scale densities (no oracle needed) ----
def test_property_constant_height_and_bounds_large():
    import torch
    rows = cols = 4000
    res, n = 0.25, 8_000_000
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(3)
    xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
    xyz[:, 0] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * 500
    xyz[:, 1] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * 500
    xyz[:, 2] = 123.25
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res),
                           layer_names=("elevation",)).getMutable()
    gm.to_device(0, names=("elevation",))
    d = amb.Dsm(amb.DsmSettings(), gm)
    d.process_device(xyz.data_ptr(), n, gm)
    gm.sync()
    gm.download(("elevation",))
    e = gm["elevation"]
    assert not np.isnan(e).any()
    assert (e == np.float32(123.25)).all()               # IDW of a constant is that constant
    # bounds: IDW is a convex combination of the neighbours' heights
    xyz[:, 2] = 100.0 + 10.0 * torch.sin(0.01 * xyz[:, 0]) * torch.cos(0.01 * xyz[:, 1])
    d.process_device(xyz.data_ptr(), n, gm)
    gm.sync()
    gm.download(("elevation",))
    e = gm["elevation"].astype(np.float64)
    qx, qy = synth.grid_positions(rows, cols, res)
    truth = synth.terrain(qx[:, None], qy[None, :])
    assert np.abs(e - truth).max() < 0.11                # |grad| <= 0.1 per metre, neighbours within 1 m
    assert e.min() >= 90.0 - 1e-3 and e.max() <= 110.0 + 1e-3


def test_property_neighbour_checksum_large():
    """Sum over cells of the neighbour count == sum over points of the number of cell centres within the radius,
    the latter evaluated independently with torch (same un-fused double expression)."""
    import torch
    rows, cols, res, n = 3000, 2000, 0.25, 3_000_000
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(4)
    xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
    xyz[:, 0] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * (rows * res / 2 + 3)
    xyz[:, 1] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * (cols * res / 2 + 3)
    xyz[:, 2] = 50.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res),
                           layer_names=("elevation",)).getMutable()
    gm.to_device(0, names=("elevation",))
    d = amb.Dsm(amb.DsmSettings(), gm)
    d.debug = True
    d.process_device(xyz.data_ptr(), n, gm)
    gm.sync()
    d._fetch_debug(gm)
    cnt, lvl = d.last_debug
    assert (lvl == 0).all()      # 8 points / m^2: the primary radius is never empty
    base_x = 0.0 + (0.5 * rows * res - 0.5 * res)
    base_y = 0.0 + (0.5 * cols * res - 0.5 * res)
    px, py = xyz[:, 0], xyz[:, 1]
    ci = torch.floor((base_x - px) / res + 0.5).to(torch.int64)
    cj = torch.floor((base_y - py) / res + 0.5).to(torch.int64)
    total = 0
    for di in range(-5, 6):
        for dj in range(-5, 6):
            i, j = ci + di, cj + dj
            inside = (i >= 0) & (i < rows) & (j >= 0) & (j < cols)
            qx = base_x + res * (-(i.to(torch.float64)))
            qy = base_y + res * (-(j.to(torch.float64)))
            dx, dy = qx - px, qy - py
            d2 = dx * dx + dy * dy
            total += int(((d2 < 1.0) & inside).sum().item())
    assert int(cnt.astype(np.int64).sum()) == total


@pytest.mark.parametrize("on_library_stream", [False, True])
def test_sharded_cloud_with_border_halos_is_bit_identical_to_the_undivided_map(on_library_stream):
    """SURVEY §8e: every rank holds only the points of its own stripe; the border halos are compacted by
    amb_dsm_extract_halo and exchanged (here: three ranks simulated one after the other on one GPU)."""
    import torch
    from aerial_mapper_b200 import sharding
    # tests/emu (AMB_TEST_EMU=1, the kernel source on a CPU): host memory is "device" memory there, so CPU tensors do
    emulated = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
    if emulated and on_library_stream:
        pytest.skip("torch.cuda.ExternalStream needs a real device")
    rows, cols, res, world = 150, 200, 0.5, 3
    xyz_np = synth.point_cloud(120000, rows * res / 2 + 3.0, cols * res / 2 + 3.0, seed=71, holes=5,
                               hole_sides=(3.0, 12.0))
    full, _ = gpu_dsm(rows, cols, res, xyz_np)
    dev = torch.device("cpu" if emulated else "cuda:0")
    device_sync = (lambda: None) if emulated else torch.cuda.synchronize
    xyz = torch.from_numpy(xyz_np).to(dev)
    ids = torch.arange(xyz.shape[0], dtype=torch.int64, device=dev)
    gms, exch = [], []
    for r in range(world):
        c0, c1 = sharding.stripe_range(cols, r, world)
        gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
        gm.to_device(0, col_range=(c0, c1), names=("elevation",))
        y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
        m = sharding.owner_mask(xyz[:, 1], y_lo, y_hi, r, world)
        hx = sharding.HaloExchange(torch, world, r, 60000, xyz[m], ids[m], dev)
        if on_library_stream:  # torch plumbing ordered on the context's own stream, no host syncs
            hx.use_stream(torch.cuda.ExternalStream(amb.lib().amb_stream(gm.context()), device=dev))
        reach = amb.lib().amb_dsm_halo_reach(ctypes_byref(gm.geometry), 1)
        amb.check(amb.lib().amb_dsm_set_density_hint(gm.context(), xyz.shape[0] / float(rows * cols)), gm.context())
        hx.extract(gm.context(), y_lo, y_hi, reach)
        gms.append((gm, c0, c1))
        exch.append(hx)
    assert sum(h.n_local for h in exch) == xyz.shape[0]          # the stripes partition the cloud
    device_sync()
    for gm, _, _ in gms:
        gm.sync()
    gathered = torch.stack([h.send for h in exch])               # what the all-gather would deliver
    device_sync()
    for r, (hx, (gm, c0, c1)) in enumerate(zip(exch, gms)):
        hx.gathered.copy_(gathered)
        device_sync()
        assert (hx.counts() <= hx.cap).all() and (hx.counts() > 0).all()
        hx.assemble()
        d = amb.Dsm(amb.DsmSettings(), gm)
        d.process_device(hx.big_xyz.data_ptr(), hx.n_total, gm, d_ids=hx.big_ids.data_ptr())
        gm.sync()
        gm.download(("elevation",))
        assert np.array_equal(gm["elevation"][:, c0:c1].view(np.uint32), full["elevation"][:, c0:c1].view(np.uint32))
    assert np.isnan(full["elevation"]).any()


def ctypes_byref(x):
    import ctypes
    return ctypes.byref(x)


def test_property_full_baseline_size_c2():
    """BASELINE config C2 at full size (50 M points -> 10000 x 10000 @ 0.25 m) through size-independent
    properties: IDW of a constant is that constant in every cell, no cell is left empty at 8 points / m^2, the
    neighbour-count checksum over a 64-column band equals an independent torch evaluation."""
    import torch
    rows = cols = 10000
    res, n = 0.25, 50_000_000
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(2)
    xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
    xyz[:, 0] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * 1250
    xyz[:, 1] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * 1250
    xyz[:, 2] = 77.5
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res),
                           layer_names=("elevation",)).getMutable()
    gm.to_device(0, names=("elevation",))
    d = amb.Dsm(amb.DsmSettings(), gm)
    d.process_device(xyz.data_ptr(), n, gm)
    gm.sync()
    t = gm.timings()
    assert t["dsm_points_binned"] == n
    # warp-per-cell list: nothing at this density in f64 mode; in f32 mode only the cells with a pair inside the guard band
    assert t["dsm_cells_empty"] == 0 if PRECISION == "f64" else t["dsm_cells_empty"] < 1e-3 * rows * cols
    gm.download(("elevation",))
    e = gm["elevation"]
    assert not np.isnan(e).any() and (e == np.float32(77.5)).all()
    del gm
    # checksum on a band of columns (stripe context + debug counters keep the footprint small)
    band = (4992, 5056)
    gb = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res),
                           layer_names=("elevation",)).getMutable()
    gb.to_device(0, col_range=band, names=("elevation",))
    db = amb.Dsm(amb.DsmSettings(), gb)
    db.debug = True
    db.process_device(xyz.data_ptr(), n, gb)
    gb.sync()
    db._fetch_debug(gb)
    cnt, lvl = db.last_debug
    assert (lvl == 0).all()
    base = 0.5 * rows * res - 0.5 * res
    py = xyz[:, 1]
    near = (py < base - res * band[0] + 1.2) & (py > base - res * (band[1] - 1) - 1.2)
    px, py = xyz[near, 0], py[near]
    ci = torch.floor((base - px) / res + 0.5).to(torch.int64)
    cj = torch.floor((base - py) / res + 0.5).to(torch.int64)
    total = 0
    for di in range(-5, 6):
        for dj in range(-5, 6):
            i, j = ci + di, cj + dj
            inside = (i >= 0) & (i < rows) & (j >= band[0]) & (j < band[1])
            qx = base + res * (-(i.to(torch.float64)))
            qy = base + res * (-(j.to(torch.float64)))
            dx, dy = qx - px, qy - py
            total += int((((dx * dx + dy * dy) < 1.0) & inside).sum().item())
    assert int(cnt.astype(np.int64).sum()) == total
