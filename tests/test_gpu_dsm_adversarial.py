"""DSM and OrthoFromPcl decisions that sit EXACTLY on their boundaries: the strict `d2 < threshold` of the radius search
(nanoflann.hpp:156-158) at every retry level, window and bin edges, the map's apron, map-scale (UTM) coordinates, the
FP32 gather's guard band, and several points on one cell centre.

The scenes are sparse "probes": isolated cells with a few hand-placed points, spaced so that no probe's points can reach
another probe's cell at any retry level.  A tie is built from a cell centre as the reference computes it: the raw point
is walked over adjacent doubles until the reference's un-fused d2 of the SHIFTED point (dsm.cc:42-43) is exactly
thr_k, its predecessor or its successor (common.points_at_distance); every probe states the level and neighbour count
that follow from the strict `<` for the d2 it actually got.

Every DSM scene runs in both gather precisions and in every production variant:
  debug run        neighbour counts, levels and NaN mask equal to the oracle, heights within MAX_ULP;
  debug off        the production template (ROWS3 when a strip spans <= 3 bin rows)      -- bit-identical to the debug run
  chunked          pinned map with host mirrors: the column groups of amb_dsm_set_stream_chunks -- bit-identical
The case 1 / 2 / 5 scenes are also compared with the reference's own dsm.cc (common.reference_outputs)."""
import math

import numpy as np
import pytest

from common import (KINDS, UTM, UTM_SHIFT, Scene, Z, apron_scene, band_scene, bin_edge_scene, cell_of,
                    coincident_members, coincident_scene, dsm_thresholds_py, eps_f, expected_level, grid_base,
                    points_at_distance, probe_cells, reach_scene, reference_outputs, shifted_d2, tie_scene, ulp_diff)
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

PRECISIONS = ["f32", "f64"]
MAX_ULP = {"f64": 1, "f32": 4}


# ---- running ----------------------------------------------------------------------------------------------------------
def gpu_run(sc, precision, xyz=None, debug=False, chunked=False, col_range=None):
    xyz = sc.xyz if xyz is None else xyz
    s = amb.GridMapSettings(sc.pos[0], sc.pos[1], sc.rows * sc.res, sc.cols * sc.res, sc.res)
    gm = amb.AerialGridMap(s, pinned=chunked).getMutable()
    assert gm.getSize() == (sc.rows, sc.cols)
    if chunked:
        gm.to_device(0)
        gm.set_mirrors(("elevation",))
    elif col_range is not None:
        gm.context(0, col_range)
    d = amb.Dsm(amb.DsmSettings(interpolation_radius=sc.radius, center_easting=sc.ce, center_northing=sc.cn), gm)
    d.precision = precision
    d.debug = debug
    d.stream_chunks = 4 if chunked else 1
    d.process(xyz, gm)
    gm.sync()
    return gm["elevation"].copy(order="F"), d.last_debug, gm.timings()


def oracle_run(sc, xyz=None):
    xyz = sc.xyz if xyz is None else xyz
    g = po.make_geometry(sc.rows, sc.cols, sc.res, sc.pos[0], sc.pos[1])
    e = np.full((sc.rows, sc.cols), np.nan, np.float32, order="F")
    st, cnt, lvl, _ = po.dsm_process(g, e, xyz, radius=sc.radius, center_easting=sc.ce, center_northing=sc.cn,
                                     debug=True)
    assert st == 0
    return e, cnt, lvl


def check_all_variants(sc, precision):
    """Debug run against the oracle, then every production variant bit-identical to it.  Returns the oracle's output
    and the debug run's timings."""
    assert np.array_equal(np.asarray(amb.dsm_thresholds(sc.radius)), np.asarray(dsm_thresholds_py(sc.radius)))
    e, cnt, lvl = oracle_run(sc)
    for (i, j, level, count) in sc.probes:            # the oracle's decision is the strict `<` of the probe's d2
        assert (lvl[i, j], cnt[i, j] if level >= 0 else 0) == (level, count), (i, j)
    ge, (gc, gl), t = gpu_run(sc, precision, debug=True)
    assert np.array_equal(gl, lvl), "retry level differs in %d cells" % int((gl != lvl).sum())
    touched = lvl >= 0
    assert np.array_equal(gc[touched], cnt[touched]), "neighbour count differs"
    assert np.array_equal(np.isnan(ge), np.isnan(e))
    assert ulp_diff(ge, e).max() <= MAX_ULP[precision]
    bits = ge.view(np.uint32)
    prod, _, _ = gpu_run(sc, precision)
    assert np.array_equal(prod.view(np.uint32), bits), "production gather differs from the debug run"
    ch, _, _ = gpu_run(sc, precision, chunked=True)
    assert np.array_equal(ch.view(np.uint32), bits), "chunked evaluation differs from the debug run"
    return e, t


def check_reference(sc, oracle_elevation, suffix=""):
    """The reference's own dsm.cc on the scene: the same NaN mask, heights within one float32 ulp of the oracle (the
    GPU is held to the oracle above)."""
    g = po.make_geometry(sc.rows, sc.cols, sc.res, sc.pos[0], sc.pos[1])
    xyz = sc.xyz

    def refsrc():
        r = np.full((sc.rows, sc.cols), np.nan, np.float32, order="F")
        st, _ = po.refsrc_dsm_process(g, r, xyz, sc.radius, sc.ce, sc.cn)
        assert st == 0, po.refsrc_last_error()
        return {"elevation": r}
    ref = reference_outputs({"elevation": oracle_elevation}, refsrc, suffix=suffix)["elevation"]
    assert np.array_equal(np.isnan(ref), np.isnan(oracle_elevation))
    assert ulp_diff(ref, oracle_elevation).max() <= 1
    return ref


# ---- case 1: exact ties at every retry level --------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("radius", [1, 2, 3])
def test_ties_at_every_retry_level(precision, radius):
    sc = tie_scene(radius, 0.5)
    e, _ = check_all_variants(sc, precision)
    lv = [p[2] for p in sc.probes]
    assert -1 in lv and max(lv) == len(dsm_thresholds_py(radius)) - 1   # the last level and "give up" both occur
    check_reference(sc, e)


# ---- case 2: reach of the windows when sqrt(thr)/res is (nearly) a half-integer -------------------------------------
HALF = [(0.4, 1), (math.sqrt(dsm_thresholds_py(1)[2]) / 2.5, 1), (1.0 / (2.5 + 4e-10), 1),
        (math.sqrt(dsm_thresholds_py(1)[-1]) / 2.5, 1), (math.sqrt(2.0) / 3.5, 2)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("res,radius", HALF)
def test_window_reach_at_half_integer_widths(precision, res, radius):
    sc = reach_scene(radius, res)
    e, _ = check_all_variants(sc, precision)
    check_reference(sc, e)


# ---- case 3: points on bin edges, tile edges and stripe borders --------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("res", [0.5, 0.25])
def test_points_on_bin_and_tile_edges(precision, res):
    sc = bin_edge_scene(res)
    check_all_variants(sc, precision)
    full, _, _ = gpu_run(sc, precision)
    for c0, c1 in [(0, 32), (32, 64), (31, 45), (45, 72)]:          # stripe borders on and off the tile edges
        part, (pc, pl), _ = gpu_run(sc, precision, debug=True, col_range=(c0, c1))
        assert np.array_equal(part[:, c0:c1].view(np.uint32), full[:, c0:c1].view(np.uint32)), (c0, c1)


# ---- case 4: the map border and the bin grid's apron -----------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
def test_points_beyond_the_border_and_the_apron(precision):
    sc = apron_scene(0.5)
    check_all_variants(sc, precision)
    assert sorted(set(p[2] for p in sc.probes))[-1] == len(dsm_thresholds_py(1)) - 1
    # bin grid: rows [-Pa, rows + Pa) around the map; a point whose binning row is -Pa - 1 is dropped, the neighbouring
    # double (row -Pa) is binned.  Both are out of every cell's reach: the elevation must not change.
    thr = dsm_thresholds_py(1)
    P = int(math.floor(math.sqrt(thr[-1]) / sc.res + 0.5 + 1e-6))
    Pa = ((P + 15) // 16) * 16             # a sparse cloud: buckets of 16 cells
    bx, by, inv = grid_base(sc.rows, sc.cols, sc.res)
    x = bx + (Pa + 0.5) * sc.res           # row -Pa - 0.5: the edge between the last kept and the first dropped row
    xs = x + np.arange(-8, 9) * np.spacing(x)
    rows_of = [cell_of(bx, v, inv) for v in xs]
    kept = [v for v, r in zip(xs, rows_of) if r == -Pa]
    dropped = [v for v, r in zip(xs, rows_of) if r == -Pa - 1]
    assert kept and dropped
    x_in, x_out = max(kept), min(dropped)
    assert np.nextafter(x_in, np.inf) == x_out     # neighbouring doubles
    base_e, _, base_t = gpu_run(sc, precision)
    for xv, binned in ((x_out, 0), (x_in, 1)):
        xyz = np.vstack([sc.xyz, [[xv, sc.qy[10], 1000.0]]])
        e, _, t = gpu_run(sc, precision, xyz=xyz)
        assert np.array_equal(e.view(np.uint32), base_e.view(np.uint32))
        assert t["dsm_points_binned"] == base_t["dsm_points_binned"] + binned


# ---- case 5: map-scale (UTM) coordinates -------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("res", [0.1, 0.25, 1.0])
@pytest.mark.parametrize("where", ["map", "shift"])
def test_utm_scale_ties_reach_and_bin_edges(precision, res, where):
    kw = dict(pos=UTM) if where == "map" else dict(pos=UTM, ce=UTM_SHIFT[0], cn=UTM_SHIFT[1])
    thr = dsm_thresholds_py(1)
    # at these magnitudes one step of a coordinate moves d2 by ~1e-9: "lo"/"hi" are the nearest attainable d2
    sc = tie_scene(1, res, levels=[0, 1, len(thr) // 2, len(thr) - 1], require_exact=False, **kw)
    e, _ = check_all_variants(sc, precision)
    check_reference(sc, e, suffix="/ties")
    sc = reach_scene(1, res, **kw)
    e, _ = check_all_variants(sc, precision)
    check_reference(sc, e, suffix="/reach")
    sc = bin_edge_scene(res, rows=72, cols=72, **kw)
    check_all_variants(sc, precision)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_utm_exact_tie_on_an_axis(precision):
    # thr_0 = 1 m^2 is attainable exactly at UTM scale along the y axis: dx = 0 and qy -+ 1 are exact -> level 1
    sc = Scene(40, 48, 0.3, 1, UTM)      # 1 m is no multiple of a cell: the point is on no cell centre
    for (i, j), sj in (((10, 10), -1.0), ((30, 36), 1.0)):
        x, y = sc.qx[i], sc.qy[j] + sj
        assert float(shifted_d2(sc.qx[i], sc.qy[j], x, y)) == 1.0
        sc.add(x, y, Z(i))
        sc.expect(i, j, 1, 1)
    check_all_variants(sc, precision)


# ---- case 6: FP32 routing ---------------------------------------------------------------------------------------------
def band_cells(sc, eps, lvl, width, with_partner):
    """Level-0 cells with a (cell, point) pair within `width` of thr_0 — for the cell itself or (with_partner) the other
    cell of its column pair, with which the FP32 gather shares the band test."""
    xyz = sc.xyz
    near = np.zeros((sc.rows, sc.cols), bool)
    for j in range(sc.cols):
        d2 = shifted_d2(sc.qx[:, None], sc.qy[j], xyz[None, :, 0], xyz[None, :, 1])
        near[:, j] = (np.abs(d2 - 1.0) <= width).any(axis=1)
    if with_partner:
        partner = near[:, np.arange(sc.cols) ^ 1] if sc.cols % 2 == 0 else None
        near = near | partner
    return int((near & (lvl == 0)).sum())


@pytest.mark.parametrize("scene", ["band", "ties"])
def test_fp32_guard_band_sends_exactly_the_band_cells_to_the_exact_kernel(scene):
    sc, eps = band_scene() if scene == "band" else (tie_scene(1, 0.5), eps_f(0.5, 1))
    e32, _ = check_all_variants(sc, "f32")
    check_all_variants(sc, "f64")
    _, _, lvl = oracle_run(sc)
    _, _, t32 = gpu_run(sc, "f32")
    _, _, t64 = gpu_run(sc, "f64")
    # f64: the list holds the cells without a level-0 hit; f32 adds the level-0 cells with a pair inside the band
    extra = t32["dsm_cells_empty"] - t64["dsm_cells_empty"]
    assert t64["dsm_cells_empty"] == int((lvl != 0).sum())
    lo = band_cells(sc, eps, lvl, eps / 2, False)       # |d2 - thr| <= eps/2  =>  |d2_f - thr| <= eps: must go
    hi = band_cells(sc, eps, lvl, 2 * eps, True)        # |d2_f - thr| <= eps  =>  |d2 - thr| <= 1.5 eps
    assert lo >= 2 and lo <= extra <= hi, (lo, extra, hi)


def handover_scene(high, dense):
    """One tile row (32 x 96 cells @ 0.5 m), three tiles, each decided by one mechanism alone:
      tile 0  background points, and at cell (16, 14) a point 5000 m above them (high) or at their height;
      tile 1  background points only (control);
      tile 2  a cluster on 2 x 2 m around cell (16, 80): 8000 points (dense) or 2500.
    Every variant holds the same number of points (the rest far outside the bin grid, where the binning drops them),
    because the stage's capacity follows the cloud's average density: it is the same ~3.4-3.6 k points in all four."""
    sc = Scene(32, 96, 0.5, 1)
    rng = np.random.default_rng(61)
    for (c0, c1) in ((3, 29), (35, 61)):
        for t in range(300):
            i, j = rng.uniform(2, 30), rng.uniform(c0, c1)
            sc.add(sc.qx[0] - 0.5 * i, sc.qy[0] - 0.5 * j, Z(t))
    sc.add(sc.qx[16] + 0.1, sc.qy[14] - 0.2, 5100.0 if high else Z(7))
    xyz = sc.xyz
    sc.expect(16, 14, 0, int((shifted_d2(sc.qx[16], sc.qy[14], xyz[:, 0], xyz[:, 1]) < 1.0).sum()))
    n_cluster = 8000 if dense else 2500
    for t in range(n_cluster):
        sc.add(sc.qx[16] + rng.uniform(-1, 1), sc.qy[80] + rng.uniform(-1, 1), Z(t))
    for t in range(8000 - n_cluster):
        sc.add(5000.0 + t, 5000.0, 100.0)
    return sc


def listed_per_tile(sc, precision):
    # a stripe context per tile column (one tile each): the number of cells its gather hands to the exact kernel
    return [gpu_run(sc, precision, col_range=(32 * k, 32 * k + 32))[2]["dsm_cells_empty"] for k in range(3)]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_tiles_the_gather_hands_over_whole(precision):
    # a tile whose staged heights span more than zrange_limit (4096 m; FP32 gather only) and a tile whose window holds
    # more points than the stage (both gathers) are evaluated whole by the exact kernel: every one of their 1024 cells is
    # listed, and every decision is the oracle's
    sc = handover_scene(high=True, dense=True)
    check_all_variants(sc, precision)
    on = listed_per_tile(sc, precision)
    off = listed_per_tile(handover_scene(high=False, dense=False), precision)
    assert on[2] == 1024 and off[2] < 1024                   # the stage overflow alone decides tile 2
    assert off[0] < 1024 and on[1] < 1024 and off[1] == on[1]   # ... and nothing else hands a tile over
    assert on[0] == (1024 if precision == "f32" else off[0])   # the height range alone decides tile 0 (f32 only)


# ---- case 7: OrthoFromPcl ---------------------------------------------------------------------------------------------
def test_ortho_from_pcl_coincident_points_take_the_last_in_point_order():
    rows, cols, res, xyz, inten, cells = coincident_scene()
    qx, qy = synth.grid_positions(rows, cols, res)
    members = coincident_members(xyz, qx, qy, cells)
    assert [len(m) for m in members] == [2, 12, 30]
    for m in members:
        assert len(set(inten[m].tolist())) > 1 or len(m) == 1      # the choice matters
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=2)).process(xyz, inten, gm)
    g = po.make_geometry(rows, cols, res)
    o = np.full((rows, cols), 255.0, np.float32, order="F")
    assert po.ortho_from_pcl_process(g, o, xyz, inten, radius=2, num_threads=-1) == 0
    for (i, j), m in zip(cells, members):
        assert o[i, j] == np.float32(inten[m.max()])                   # the oracle: last zero-distance point
        assert gm["ortho"][i, j] == o[i, j], (i, j)                    # the GPU: the same point, bit for bit
    assert np.array_equal(gm["ortho"] == 255.0, o == 255.0)
    assert ulp_diff(gm["ortho"], o).max() <= 1

    def refsrc():
        r = np.full((rows, cols), 255.0, np.float32, order="F")
        assert po.refsrc_ortho_from_pcl_process(g, r, xyz, inten, 2, False) == 0
        return {"ortho": r}
    ref = reference_outputs({"ortho": o}, refsrc)["ortho"]
    # the reference keeps the last perfect match in ITS kd-tree's order: some member of the cluster
    for (i, j), m in zip(cells, members):
        assert ref[i, j] in set(np.float32(inten[m]).tolist())
    other = np.ones((rows, cols), bool)
    for (i, j) in cells:
        other[i, j] = False
    assert np.array_equal((ref == 255.0)[other], (o == 255.0)[other])
    assert ulp_diff(ref[other], gm["ortho"][other]).max() <= 1


def adaptive_scene():
    """Map 40 x 40 @ 1 m, r = 1, a handful of points: probes whose nearest point is at d2 == 10^k exactly (the ball of
    10^k is empty: the next level decides) and at one ulp below (level k decides)."""
    rows = cols = 40
    res = 1.0
    qx, qy = synth.grid_positions(rows, cols, res)
    pts = []
    probes = []
    # d2 = 1 + 9 = 10 and 36 + 64 = 100: exact in double.  Each probe also has a point at d2 = 50 or 200 on the other
    # side, which only the next level's ball holds.
    for (i, j), (dx, dy), far in (((5, 5), (1.0, 3.0), (-5.0, -5.0)), ((30, 8), (6.0, 8.0), (-10.0, 10.0))):
        pts += [(qx[i] - dx, qy[j] - dy), (qx[i] - far[0], qy[j] - far[1])]
        probes.append((i, j, dx * dx + dy * dy))
    c = points_at_distance(qx[20], qy[30], 10.0, 0.8)["lo"]
    pts += [(c[0], c[1]), (qx[20] + 5.0, qy[30] + 5.0)]
    probes.append((20, 30, c[2]))
    return rows, cols, res, np.array([[x, y, 0.0] for x, y in pts]), probes


def brute_adaptive(rows, cols, res, xyz, inten, radius):
    qx, qy = synth.grid_positions(rows, cols, res)
    out = np.empty((rows, cols), np.float32, order="F")
    for j in range(cols):
        for i in range(rows):
            d2 = shifted_d2(qx[i], qy[j], xyz[:, 0], xyz[:, 1])
            thr = float(radius)
            lam = 10
            while not (d2 < thr).any():
                thr = float(lam * radius)
                lam *= 10
            m = d2 < thr
            if (d2[m] == 0).any():
                out[i, j] = np.float32(inten[m][d2[m] == 0][-1])
            else:
                out[i, j] = np.float32(np.sum(inten[m] / d2[m]) / np.sum(1.0 / d2[m]))
    return out


def test_ortho_from_pcl_adaptive_ties_at_powers_of_ten():
    rows, cols, res, xyz, probes = adaptive_scene()
    inten = np.array([17, 130, 251, 3, 77, 199], np.int32)
    qx, qy = synth.grid_positions(rows, cols, res)
    for (i, j, d2) in probes:
        assert float(shifted_d2(qx[i], qy[j], xyz[:, 0], xyz[:, 1]).min()) == d2
    assert probes[0][2] == 10.0 and probes[1][2] == 100.0 and probes[2][2] == np.nextafter(10.0, 0.0)
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=1,
                                              use_adaptive_interpolation=True)).process(xyz, inten, gm)
    b = brute_adaptive(rows, cols, res, xyz, inten, 1)
    assert ulp_diff(gm["ortho"], b).max() <= 1
    # d2 == 10 (and == 100): that ball is empty, the next one also holds the point on the other side
    for (i, j, _), k in zip(probes[:2], (0, 2)):
        assert gm["ortho"][i, j] not in (np.float32(inten[k]), np.float32(inten[k + 1]))
    # one ulp below 10: the ball of 10 holds that point alone
    assert gm["ortho"][20, 30] == np.float32(inten[4])
    if po.have_ref():
        o = np.full((rows, cols), 255.0, np.float32, order="F")
        assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), o, xyz, inten, radius=1, adaptive=True,
                                         use_ref=True) == 0
        assert ulp_diff(gm["ortho"], o).max() <= 1


def test_ortho_from_pcl_adaptive_whole_grid_early_exit():
    # 8 x 8 cells, two points in the far corner of the bin grid's apron.  At 10^3 the window of every cell covers the
    # whole bin grid (reach 50 cells) while the ball is still empty: the level loop jumps to the first threshold above
    # the nearest point's d2 (10^4), where both points are neighbours.  What this shows is that the exit gives the
    # right value and raises no `unresolved` flag; without the exit the loop would reach the same level (the window of
    # 10^4 clamps to the same bin grid), so the test would not notice an exit that never fires.
    rows = cols = 8
    res = math.sqrt(1000.0) / 50.0
    bx, by, inv = grid_base(rows, cols, res)
    xyz = np.array([[bx - 47 * res, by - 47 * res, 0.0], [bx - 47 * res, by - 46 * res, 0.0]])
    inten = np.array([40, 200], np.int32)
    qx, qy = synth.grid_positions(rows, cols, res)
    d2 = shifted_d2(qx[:, None, None], qy[None, :, None], xyz[None, None, :, 0], xyz[None, None, :, 1]).min(axis=2)
    assert (d2 >= 1000.0).all() and (d2 < 10000.0).all()
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=1,
                                              use_adaptive_interpolation=True)).process(xyz, inten, gm)
    b = brute_adaptive(rows, cols, res, xyz, inten, 1)
    assert ulp_diff(gm["ortho"], b).max() <= 1
    assert ((gm["ortho"] > 40) & (gm["ortho"] < 200)).all()
