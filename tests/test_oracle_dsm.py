"""CPU tests of the DSM oracle (dsm.cc:36-52,113-184 restated): against brute force, scipy's kd-tree and — where
/root/reference exists — the reference's own nanoflann.hpp compiled verbatim (oracle/_ref)."""
import numpy as np
import pytest

from common import brute_dsm, ulp_diff
from aerial_mapper_b200 import synth
from oracle import pyoracle as po


def _run(rows, cols, res, xyz, **kw):
    g = po.make_geometry(rows, cols, res, kw.pop("pos_x", 0.0), kw.pop("pos_y", 0.0))
    e = kw.pop("elevation", None)
    if e is None:
        e = np.full((rows, cols), np.nan, np.float32, order="F")
    st, cnt, lvl, _ = po.dsm_process(g, e, xyz, debug=True, **kw)
    return st, e, cnt, lvl


def test_thresholds_follow_the_reference_recurrence():
    from oracle.pyoracle import lib  # noqa: F401  (forces the build)
    import ctypes as C
    import aerial_mapper_b200 as amb
    thr = amb.dsm_thresholds(1)
    assert len(thr) == 21 and thr[0] == 1.0
    lam = 1.0
    for k in range(21):
        assert thr[k] == lam * 1
        lam *= 1.1
    assert lam * 1 > 7.0 and thr[-1] <= 7.0
    assert amb.dsm_thresholds(7) == [7.0]      # 1.1*7 > 7 -> exactly one retry
    assert amb.dsm_thresholds(9) == [9.0]      # radius > 7: the loop body still runs once
    assert len(amb.dsm_thresholds(2)) == 14


@pytest.mark.parametrize("rows,cols,res,n,radius,seed", [(12, 9, 1.0, 150, 1, 1), (16, 10, 0.25, 60, 1, 2),
                                                         (9, 14, 0.5, 80, 2, 3), (7, 7, 2.0, 300, 1, 4)])
def test_oracle_matches_brute_force(rows, cols, res, n, radius, seed):
    xyz = synth.point_cloud(n, rows * res / 2 + 1.0, cols * res / 2 + 1.0, seed)
    st, e, cnt, lvl = _run(rows, cols, res, xyz, radius=radius, num_threads=-1)
    assert st == 0
    be, bc, bl = brute_dsm(rows, cols, res, xyz, radius)
    assert np.array_equal(bl, lvl)
    assert np.array_equal(np.where(bl >= 0, bc, 0), np.where(lvl >= 0, cnt, 0))
    assert np.array_equal(np.isnan(be), np.isnan(e))
    assert ulp_diff(be, e).max() <= 1  # summation order differs (numpy pairwise vs sequential)


def test_oracle_neighbour_counts_match_scipy_kdtree():
    from scipy.spatial import cKDTree
    rows, cols, res = 64, 48, 0.5
    xyz = synth.point_cloud(6000, 17.0, 13.0, seed=5)
    st, e, cnt, lvl = _run(rows, cols, res, xyz, num_threads=2)
    assert st == 0
    qx, qy = synth.grid_positions(rows, cols, res)
    tree = cKDTree(xyz[:, :2])
    Q = np.stack(np.meshgrid(qx, qy, indexing="ij"), -1).reshape(-1, 2)
    n1 = np.array(tree.query_ball_point(Q, 1.0, return_length=True)).reshape(rows, cols)
    primary = lvl == 0
    assert np.array_equal(n1[primary], cnt[primary])  # d2 < 1  <=>  dist < 1 away from exact ties
    assert (n1[~primary] == 0).all()


def test_oracle_equals_reference_nanoflann():
    if not po.have_ref():
        pytest.skip("oracle/_ref not built (no /root/reference on this box)")
    for rows, cols, res, n, holes, radius in [(256, 256, 1.0, 100000, 0, 1), (200, 120, 0.25, 9000, 3, 1),
                                              (90, 70, 0.5, 5000, 0, 3)]:
        xyz = synth.point_cloud(n, rows * res / 2, cols * res / 2, seed=7, holes=holes, hole_sides=(2.0, 8.0))
        st1, e1, c1, l1 = _run(rows, cols, res, xyz, radius=radius)
        st2, e2, c2, l2 = _run(rows, cols, res, xyz, radius=radius, use_ref=True)
        assert st1 == 0 and st2 == 0
        assert np.array_equal(c1, c2) and np.array_equal(l1, l2)
        d = ulp_diff(e1, e2)
        assert d.max() <= 1, "restatement vs nanoflann-order sums differ by more than one float ulp"
        assert (d != 0).mean() < 1e-4


def test_c1_statistics():
    # BASELINE.md §2 / SURVEY §8d config C1: ~4.8 neighbours per cell, ~0.85 % fallback cells, 0 NaN
    xyz = synth.point_cloud(100000, 128.0, 128.0, seed=1)
    st, e, cnt, lvl = _run(256, 256, 1.0, xyz)
    assert st == 0
    assert not np.isnan(e).any()
    assert 4.6 < cnt.mean() < 5.0
    assert 0.006 < (lvl > 0).mean() < 0.011


def test_threads_and_single_thread_twins_agree():
    xyz = synth.point_cloud(20000, 40.0, 30.0, seed=9, holes=2, hole_sides=(3.0, 10.0))
    outs = [_run(160, 120, 0.5, xyz, num_threads=t) for t in (-1, 1, 3, 8)]
    for st, e, cnt, lvl in outs[1:]:
        assert st == 0
        assert np.array_equal(e.view(np.uint32), outs[0][1].view(np.uint32))
        assert np.array_equal(cnt, outs[0][2]) and np.array_equal(lvl, outs[0][3])


def test_center_shift_swaps_northing_and_easting():
    # dsm.cc:42-43: x -= center_northing, y -= center_easting (sic).  The query centres are NOT shifted.
    xyz = synth.point_cloud(3000, 10.0, 8.0, seed=10)
    moved = xyz.copy()
    moved[:, 0] += 5.0   # undone by center_northing = 5
    moved[:, 1] -= 3.0   # undone by center_easting = -3
    st0, e0, c0, l0 = _run(20, 16, 1.0, xyz)
    st1, e1, c1, l1 = _run(20, 16, 1.0, moved, center_northing=5.0, center_easting=-3.0)
    assert st0 == 0 and st1 == 0
    assert np.array_equal(c0, c1) and np.array_equal(l0, l1)
    assert ulp_diff(e0, e1).max() <= 1


def test_empty_cloud_and_untouched_cells():
    g = po.make_geometry(8, 8, 1.0)
    e = np.full((8, 8), 7.5, np.float32, order="F")
    st, _, _, _ = po.dsm_process(g, e, np.zeros((0, 3)))
    assert st == -1 and (e == 7.5).all()          # dsm.cc:189-192: warn + return, layers untouched
    far = np.array([[100.0, 100.0, 5.0]])
    st, _, _, _ = po.dsm_process(g, e, far)
    assert st == 0 and (e == 7.5).all()           # no neighbour within any threshold: previous value kept


def test_second_process_overwrites_only_where_points_are():
    # incremental pipeline (main-ortho-backward-grid-incremental.cc:153): new tree from new points only
    a = synth.point_cloud(800, 5.0, 10.0, seed=11, center=(-5.0, 0.0))
    b = synth.point_cloud(800, 5.0, 10.0, seed=12, center=(5.0, 0.0))
    b[:, 2] += 50.0
    st, e, _, _ = _run(20, 20, 1.0, a)
    first = e.copy()
    st, e, cnt, lvl = _run(20, 20, 1.0, b, elevation=e)
    assert st == 0
    touched = lvl >= 0
    assert (e[touched] > 120).all()
    assert np.array_equal(e[~touched].view(np.uint32), first[~touched].view(np.uint32))
    assert touched.any() and (~touched).any()


def test_coincident_point_is_the_reference_abort():
    g = po.make_geometry(4, 4, 1.0)
    qx, qy = synth.grid_positions(4, 4, 1.0)
    xyz = np.array([[qx[1], qy[2], 3.0], [0.3, 0.2, 1.0]])
    e = np.full((4, 4), np.nan, np.float32, order="F")
    st, _, _, _ = po.dsm_process(g, e, xyz)
    assert st == -3  # CHECK(distances[i] > 0.0), dsm.cc:165


def test_cell_range_sample_equals_full_run():
    xyz = synth.point_cloud(5000, 20.0, 15.0, seed=13)
    st, full, _, _ = _run(80, 60, 0.5, xyz)
    g = po.make_geometry(80, 60, 0.5)
    part = np.full((80, 60), np.nan, np.float32, order="F")
    st, _, _, _ = po.dsm_process(g, part, xyz, cell_range=(80 * 10, 80 * 25))
    assert st == 0
    assert np.array_equal(part[:, 10:25].view(np.uint32), full[:, 10:25].view(np.uint32))
    assert np.isnan(part[:, :10]).all() and np.isnan(part[:, 25:]).all()


# ---- the probe scenes of tests/test_gpu_dsm_adversarial.py, on the oracle alone -----------------------------------------
def test_the_half_integer_scenes_reach_the_last_window_row():
    # the constructed points land in the last bin row half_widths() keeps (otherwise those scenes test nothing there)
    import math
    from common import last_window_row_hits, reach_scene
    assert last_window_row_hits(reach_scene(1, 0.4)) > 0
    assert last_window_row_hits(reach_scene(2, math.sqrt(2.0) / 3.5)) > 0


@pytest.mark.parametrize("radius", [1, 2, 3])
def test_probe_ties_decided_by_the_strict_threshold_like_brute_force(radius):
    # exact ties at every retry level: the oracle's levels, counts and heights equal the brute-force definition's, and
    # every probe gets the level and count the strict `<` implies for its d2
    from common import tie_scene
    sc = tie_scene(radius, 0.5)
    st, e, cnt, lvl = _run(sc.rows, sc.cols, sc.res, sc.xyz, radius=radius)
    assert st == 0
    be, bc, bl = brute_dsm(sc.rows, sc.cols, sc.res, sc.xyz, radius)
    assert np.array_equal(lvl, bl) and np.array_equal(cnt[bl >= 0], bc[bl >= 0])
    assert ulp_diff(e, be).max() <= 1
    for (i, j, level, count) in sc.probes:
        assert lvl[i, j] == level and (level < 0 or cnt[i, j] == count), (i, j)
