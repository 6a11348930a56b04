"""The restated oracle against the REFERENCE'S OWN translation units.

oracle/_ref/libamb_refsrc_{main,pcl}.so hold the reference's dsm.cc, ortho-backward-grid.cc, ortho-from-pcl.cc and
utils-common.cc (with nanoflann.hpp, dsm.h, ...) compiled verbatim from /root/reference against stand-in third-party
headers (oracle/refsrc_stubs/amb_refsrc_deps.h says exactly what is reference code and what is restated).  These
tests drive the reference's public API — dsm::Dsm::process, ortho::OrthoBackwardGrid::process,
ortho::OrthoFromPcl::process, single- and multi-threaded — on the same seeded inputs as the restatement and require:
  * every layer of the loop restated around the reference's nanoflann (same summation order): bit-identical;
  * the dependency-free bucket oracle (the one the GPU parity tests use): neighbour decisions identical, heights within
    one float32 ulp (summation order), everything else bit-identical.
The libraries are built where /root/reference exists and travel to the GPU box as prebuilt files."""
import numpy as np
import pytest

from common import fresh_layers, ulp_diff
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

pytestmark = pytest.mark.skipif(not po.have_refsrc(), reason="oracle/_ref/libamb_refsrc_*.so not built "
                                                             "(needs /root/reference)")

RADTAN = (-0.05, 0.01, 1e-4, 1e-4)
EQUI = (0.01, -0.002, 0.0005, -0.0001)


def _nan_layer(rows, cols):
    return np.full((rows, cols), np.nan, np.float32, order="F")


# ---- dsm.cc ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,res,n,holes,radius,ce,cn,pos", [
    (128, 96, 1.0, 30000, 0, 1, 0.0, 0.0, (0.0, 0.0)),
    (200, 120, 0.25, 9000, 3, 1, 0.0, 0.0, (0.0, 0.0)),          # holes -> retry levels up to "none"
    (90, 70, 0.5, 5000, 0, 3, 0.0, 0.0, (0.0, 0.0)),
    (64, 80, 0.5, 7000, 2, 2, 12.5, -7.25, (3.0, -2.0)),          # centre shift (sic: x-northing, y-easting) + offset map
])
@pytest.mark.parametrize("multi_thread", [True, False])
def test_dsm_restatement_equals_reference_dsm_cc(rows, cols, res, n, holes, radius, ce, cn, pos, multi_thread):
    xyz = synth.point_cloud(n, rows * res / 2, cols * res / 2, seed=11, holes=holes, hole_sides=(2.0, 8.0))
    xyz[:, 0] += cn + pos[0]
    xyz[:, 1] += ce + pos[1]
    g = po.make_geometry(rows, cols, res, pos[0], pos[1])
    e_src = _nan_layer(rows, cols)
    st, _ = po.refsrc_dsm_process(g, e_src, xyz, radius, ce, cn, multi_thread=multi_thread)
    assert st == 0, po.refsrc_last_error()
    # restated loop around the reference's nanoflann: same traversal order -> same bits
    e_nf = _nan_layer(rows, cols)
    st, _, lvl_nf, _ = po.dsm_process(g, e_nf, xyz, radius, ce, cn, num_threads=0 if multi_thread else -1,
                                      debug=True, use_ref=True)
    assert st == 0
    assert np.array_equal(e_src.view(np.uint32), e_nf.view(np.uint32))
    # dependency-free bucket restatement: same neighbour sets (hence same NaN pattern), sums within 1 ulp
    e_b = _nan_layer(rows, cols)
    st, _, lvl_b, _ = po.dsm_process(g, e_b, xyz, radius, ce, cn, num_threads=3, debug=True)
    assert st == 0
    assert np.array_equal(lvl_b, lvl_nf)
    assert np.array_equal(np.isnan(e_src), lvl_b < 0)
    d = ulp_diff(e_src, e_b)
    assert d.max() <= 1 and (d != 0).mean() < 1e-3
    if holes:
        assert (lvl_b > 0).any() and (lvl_b < 0).any()  # the case really exercises the retry loop and its give-up


def test_dsm_reference_keeps_cells_without_neighbours_and_previous_values():
    rows, cols, res = 40, 30, 1.0
    xyz = synth.point_cloud(300, 6.0, 5.0, seed=12)           # points only near the centre
    g = po.make_geometry(rows, cols, res)
    prior = np.asfortranarray(np.random.default_rng(0).uniform(0, 1, (rows, cols)).astype(np.float32))
    a, b = prior.copy(order="F"), prior.copy(order="F")
    assert po.refsrc_dsm_process(g, a, xyz)[0] == 0
    assert po.dsm_process(g, b, xyz, use_ref=True)[0] == 0
    assert np.array_equal(a, b)
    assert (a == prior).sum() > 100 and (a != prior).sum() > 100  # far cells keep the layer's previous value


def test_dsm_reference_empty_cloud_returns_without_touching_the_layer():
    g = po.make_geometry(8, 8, 1.0)
    e = _nan_layer(8, 8)
    assert po.refsrc_dsm_process(g, e, np.zeros((0, 3)))[0] == 0       # LOG(WARNING); return  (dsm.cc:189-192)
    assert np.isnan(e).all()
    assert po.dsm_process(g, _nan_layer(8, 8), np.zeros((0, 3)))[0] == -1  # the restatement reports AMB_ERR_EMPTY


def test_dsm_reference_check_fails_on_coincident_point():
    # CHECK(distances[i] > 0.0), dsm.cc:165: a point exactly on a cell centre aborts the reference; the stand-in
    # glog turns the abort into an exception on the calling thread (single-thread twin), the restatement into a status
    rows, cols, res = 6, 6, 1.0
    qx, qy = synth.grid_positions(rows, cols, res)
    xyz = np.array([[qx[2], qy[3], 5.0], [0.3, 0.2, 1.0]])
    g = po.make_geometry(rows, cols, res)
    st, _ = po.refsrc_dsm_process(g, _nan_layer(rows, cols), xyz, multi_thread=False)
    assert st == -6 and "distances[i] > 0.0" in po.refsrc_last_error()[0]     # AMB_ERR_CHECK_FAILED
    st, _, _, _ = po.dsm_process(g, _nan_layer(rows, cols), xyz, num_threads=-1)
    assert st != 0                                                            # AMB_ERR_COINCIDENT_POINT


def test_dsm_reference_sub_range_is_the_same_cells_of_the_full_run():
    rows, cols, res = 50, 40, 0.5
    xyz = synth.point_cloud(4000, 13.0, 10.5, seed=13)
    g = po.make_geometry(rows, cols, res)
    full, part = _nan_layer(rows, cols), _nan_layer(rows, cols)
    assert po.refsrc_dsm_process(g, full, xyz)[0] == 0
    k0, k1 = rows * 7 + 3, rows * 29 + 11
    assert po.refsrc_dsm_process(g, part, xyz, cell_range=(k0, k1))[0] == 0
    f, p = full.ravel(order="F"), part.ravel(order="F")
    assert np.array_equal(f[k0:k1], p[k0:k1], equal_nan=True)
    assert np.isnan(p[:k0]).all() and np.isnan(p[k1:]).all()


def _probe_scenes():
    import math
    import common as scenes
    utm = dict(pos=scenes.UTM, ce=scenes.UTM_SHIFT[0], cn=scenes.UTM_SHIFT[1])
    return {"ties_r1": lambda: scenes.tie_scene(1, 0.5),
            "ties_r2": lambda: scenes.tie_scene(2, 0.5),
            "ties_r3": lambda: scenes.tie_scene(3, 0.5),
            "reach_0.4": lambda: scenes.reach_scene(1, 0.4),
            "reach_half_2": lambda: scenes.reach_scene(2, math.sqrt(2.0) / 3.5),
            "edges": lambda: scenes.bin_edge_scene(0.25),
            "apron": lambda: scenes.apron_scene(0.5),
            "band": lambda: scenes.band_scene()[0],
            "utm_ties": lambda: scenes.tie_scene(1, 0.25, levels=[0, 1, 10, 20], require_exact=False, **utm),
            "utm_reach": lambda: scenes.reach_scene(1, 0.1, **utm)}


@pytest.mark.parametrize("scene", sorted(_probe_scenes()))
def test_probe_scene_decisions_equal_the_reference_nanoflann(scene):
    # the adversarial probe scenes of the GPU tests (exact ties at every retry level, half-integer window widths, bin
    # edges, the apron, UTM coordinates): the bucket oracle's neighbour sets against the reference's own kd-tree and dsm.cc
    sc = _probe_scenes()[scene]()
    g = po.make_geometry(sc.rows, sc.cols, sc.res, sc.pos[0], sc.pos[1])
    xyz = sc.xyz
    e_src = _nan_layer(sc.rows, sc.cols)
    st, _ = po.refsrc_dsm_process(g, e_src, xyz, sc.radius, sc.ce, sc.cn)
    assert st == 0, po.refsrc_last_error()
    e_nf, e_b = _nan_layer(sc.rows, sc.cols), _nan_layer(sc.rows, sc.cols)
    st, cnt_nf, lvl_nf, _ = po.dsm_process(g, e_nf, xyz, sc.radius, sc.ce, sc.cn, debug=True, use_ref=True)
    assert st == 0
    st, cnt_b, lvl_b, _ = po.dsm_process(g, e_b, xyz, sc.radius, sc.ce, sc.cn, num_threads=2, debug=True)
    assert st == 0
    assert np.array_equal(e_src.view(np.uint32), e_nf.view(np.uint32))
    assert np.array_equal(lvl_b, lvl_nf) and np.array_equal(cnt_b[lvl_b >= 0], cnt_nf[lvl_b >= 0])
    assert ulp_diff(e_src, e_b).max() <= 1
    for (i, j, level, count) in sc.probes:
        assert lvl_nf[i, j] == level and (level < 0 or cnt_nf[i, j] == count), (i, j)


def test_coincident_points_the_oracle_takes_the_last_the_reference_its_tree_order():
    # ortho-from-pcl.cc:90-96 keeps the LAST zero-distance point its loop visits, in the kd-tree's traversal order.  The
    # oracle (and the GPU) take the last in point order, i.e. the largest index: a documented divergence — the value is
    # always one of the cluster's intensities, but not necessarily the same one
    from common import coincident_members, coincident_scene
    rows, cols, res, xyz, inten, cells = coincident_scene()
    qx, qy = synth.grid_positions(rows, cols, res)
    members = coincident_members(xyz, qx, qy, cells)
    g = po.make_geometry(rows, cols, res)
    a = np.full((rows, cols), 255.0, np.float32, order="F")
    b, c = a.copy(order="F"), a.copy(order="F")
    assert po.refsrc_ortho_from_pcl_process(g, a, xyz, inten, 2, False) == 0, po.refsrc_last_error()
    assert po.ortho_from_pcl_process(g, b, xyz, inten, 2, False, use_ref=True) == 0
    assert po.ortho_from_pcl_process(g, c, xyz, inten, 2, False, num_threads=2) == 0
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    differ = 0
    for (i, j), m in zip(cells, members):
        assert a[i, j] in set(np.float32(inten[m]).tolist())
        assert c[i, j] == np.float32(inten[m.max()])
        differ += a[i, j] != c[i, j]
    assert differ >= 1                      # the divergence is real on this scene
    other = np.ones((rows, cols), bool)
    for (i, j) in cells:
        other[i, j] = False
    assert ulp_diff(a[other], c[other]).max() <= 1


# ---- ortho-backward-grid.cc ------------------------------------------------------------------------------------
def _scene(rows, cols, res, dist_type, dist, colored, seed, n_lines=2, per_line=3, agl=45.0, extrinsics=False):
    camd = synth.scaled_camera(0.05, dist_type=dist_type, dist=dist)
    if extrinsics:
        q = np.array([0.995, 0.05, -0.06, 0.04])
        camd["q_C_B"] = tuple(q / np.linalg.norm(q))
        camd["t_C_B"] = (0.1, -0.05, 0.02)
    poses = synth.lawnmower_poses(n_lines, per_line, rows * res / 2, cols * res / 2, agl=agl, seed=seed,
                                  jitter_pos=1.0)
    ch = 3 if colored else 1
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(poses))]
    elev = synth.analytic_elevation(rows, cols, res)
    return camd, poses, imgs, elev


@pytest.mark.parametrize("dist_type,dist,colored,extrinsics", [(1, RADTAN, False, False), (1, RADTAN, True, True),
                                                               (2, EQUI, False, True), (0, (0, 0, 0, 0), True, False)])
@pytest.mark.parametrize("multi_thread", [True, False])
def test_ortho_restatement_equals_reference_ortho_backward_grid_cc(dist_type, dist, colored, extrinsics,
                                                                  multi_thread):
    rows, cols, res = 70, 50, 0.5
    camd, poses, imgs, elev = _scene(rows, cols, res, dist_type, dist, colored, seed=41, extrinsics=extrinsics)
    elev[3:6, 4:9] = np.nan                       # cells the DSM left empty: never visible
    g, cam = po.make_geometry(rows, cols, res), po.make_camera(**camd)
    A = fresh_layers(rows, cols, elev)
    A["num_observations"] = np.zeros((rows, cols), np.float32, order="F")  # aerial-mapper-grid-map.cc:40-48
    st, _ = po.refsrc_ortho_process(g, A, cam, poses, imgs, colored=colored, multi_thread=multi_thread)
    assert st == 0, po.refsrc_last_error()
    B = fresh_layers(rows, cols, elev)
    st, _ = po.ortho_process(g, B, cam, poses, imgs, colored=colored, num_threads=0 if multi_thread else -1)
    assert st == 0
    for k in ("elevation", "elevation_angle", "observation_index", "ortho", "colored_ortho"):
        assert np.array_equal(A[k].view(np.uint32), B[k].view(np.uint32)), k
    assert (A["num_observations"] == 0).all()     # `+= itself` (ortho-backward-grid.cc:183): 0 stays 0
    seen = ~np.isnan(A["observation_index"])
    assert seen.mean() > 0.8 and len(np.unique(A["observation_index"][seen])) >= 3


def test_ortho_reference_state_lives_in_the_layers_across_calls():
    # incremental batches: the second call starts from the first call's elevation_angle (float32) — restated the same
    rows, cols, res = 48, 56, 0.5
    camd, poses, imgs, elev = _scene(rows, cols, res, 1, RADTAN, False, seed=43, n_lines=2, per_line=4)
    g, cam = po.make_geometry(rows, cols, res), po.make_camera(**camd)
    A, B = fresh_layers(rows, cols, elev), fresh_layers(rows, cols, elev)
    for lo, hi in ((0, 3), (3, 8)):
        assert po.refsrc_ortho_process(g, A, cam, poses[lo:hi], imgs[lo:hi])[0] == 0
        assert po.ortho_process(g, B, cam, poses[lo:hi], imgs[lo:hi])[0] == 0
        for k in ("elevation_angle", "observation_index", "ortho"):
            assert np.array_equal(A[k].view(np.uint32), B[k].view(np.uint32)), k


def test_ortho_reference_checks():
    g, cam = po.make_geometry(4, 4, 1.0), po.make_camera(8, 8, 4, 4, 4, 4)
    L = fresh_layers(4, 4, np.zeros((4, 4), np.float32))
    st, _ = po.refsrc_ortho_process(g, L, cam, np.zeros((0, 7)), [])
    assert st == -6 and "T_G_Bs.empty()" in po.refsrc_last_error()[0]  # CHECK(!T_G_Bs.empty()), :225


def test_ortho_reference_sub_range():
    rows, cols, res = 40, 36, 0.5
    camd, poses, imgs, elev = _scene(rows, cols, res, 1, RADTAN, False, seed=44)
    g, cam = po.make_geometry(rows, cols, res), po.make_camera(**camd)
    F, P = fresh_layers(rows, cols, elev), fresh_layers(rows, cols, elev)
    assert po.refsrc_ortho_process(g, F, cam, poses, imgs)[0] == 0
    k0, k1 = rows * 5 + 1, rows * 30 + 17
    assert po.refsrc_ortho_process(g, P, cam, poses, imgs, cell_range=(k0, k1))[0] == 0
    fresh = fresh_layers(rows, cols, elev)
    for k in ("elevation_angle", "observation_index", "ortho"):
        f, p, z = F[k].ravel(order="F"), P[k].ravel(order="F"), fresh[k].ravel(order="F")
        assert np.array_equal(f[k0:k1], p[k0:k1], equal_nan=True)
        assert np.array_equal(p[:k0], z[:k0], equal_nan=True) and np.array_equal(p[k1:], z[k1:], equal_nan=True)


# ---- ortho-from-pcl.cc -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("radius,holes,adaptive", [(2, 0, False), (1, 3, False), (1, 3, True)])
def test_ortho_from_pcl_restatement_equals_reference_cc(radius, holes, adaptive):
    rows, cols, res = 90, 60, 0.5
    xyz = synth.point_cloud(6000, rows * res / 2, cols * res / 2, seed=51, holes=holes, hole_sides=(3.0, 9.0))
    inten = np.random.default_rng(5).integers(0, 256, len(xyz)).astype(np.int32)
    qx, qy = synth.grid_positions(rows, cols, res)
    xyz[0, :2] = (qx[10], qy[20])                  # a perfect match: distance == 0 -> the cell takes that intensity
    g = po.make_geometry(rows, cols, res)
    a = np.full((rows, cols), 255.0, np.float32, order="F")
    b, c = a.copy(order="F"), a.copy(order="F")
    assert po.refsrc_ortho_from_pcl_process(g, a, xyz, inten, radius, adaptive) == 0, po.refsrc_last_error()
    assert po.ortho_from_pcl_process(g, b, xyz, inten, radius, adaptive, use_ref=True) == 0
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))   # restated loop, same nanoflann order: same bits
    if not adaptive:                                               # bucket restatement: fixed radius only
        assert po.ortho_from_pcl_process(g, c, xyz, inten, radius, False, num_threads=2) == 0
        assert np.array_equal(a == 255.0, c == 255.0)
        assert ulp_diff(a, c).max() <= 1
        if holes:
            assert (a == 255.0).any()              # no retry: hole cells keep the initial value
    else:
        assert not (a == 255.0).all() and np.isfinite(a).all()
    assert a[10, 20] == np.float32(inten[0])


# ---- the committed golden fixtures are what the reference's own code produces ------------------------------------
def test_golden_fixtures_are_bit_for_bit_what_the_reference_sources_produce():
    import os
    from common import GOLDEN
    z = np.load(os.path.join(GOLDEN, "dsm_96x80.npz"))
    rows, cols, res = int(z["rows"]), int(z["cols"]), float(z["res"])
    g = po.make_geometry(rows, cols, res)
    for mt in (True, False):
        e = _nan_layer(rows, cols)
        assert po.refsrc_dsm_process(g, e, z["xyz"], multi_thread=mt)[0] == 0
        assert np.array_equal(e.view(np.uint32), z["elevation"].view(np.uint32))
        assert np.array_equal(np.isnan(e), z["threshold_index"] < 0)
    for name, colored in (("ortho_gray_96x80.npz", False), ("ortho_color_96x80.npz", True)):
        z = np.load(os.path.join(GOLDEN, name))
        rows, cols, res = int(z["rows"]), int(z["cols"]), float(z["res"])
        camd = synth.scaled_camera(float(z["cam_scale"]), dist_type=1)
        ch = 3 if colored else 1
        imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(z["poses"]))]
        L = fresh_layers(rows, cols, z["elevation"])
        st, _ = po.refsrc_ortho_process(po.make_geometry(rows, cols, res), L, po.make_camera(**camd), z["poses"],
                                        imgs, colored=colored)
        assert st == 0
        assert np.array_equal(L["elevation_angle"].view(np.uint32), z["elevation_angle"].view(np.uint32))
        assert np.array_equal(L["observation_index"].view(np.uint32), z["observation_index"].view(np.uint32))
        assert np.array_equal(L["colored_ortho" if colored else "ortho"].view(np.uint32), z["out"])


# ---- randomised (hypothesis): any geometry / offset / camera — the restatement is the reference's code, bit for bit --
from hypothesis import given, settings, strategies as hst  # noqa: E402


@settings(max_examples=40, deadline=None)
@given(seed=hst.integers(0, 100_000), rows=hst.integers(3, 40), cols=hst.integers(3, 40),
       res=hst.sampled_from([0.1, 0.25, 0.4, 0.5, 1.0, 2.0]), radius=hst.integers(1, 9),
       pos_x=hst.floats(-500.0, 500.0), pos_y=hst.floats(-500.0, 500.0),
       ce=hst.floats(-50.0, 50.0), cn=hst.floats(-50.0, 50.0), density=hst.sampled_from([0.05, 0.5, 4.0]))
def test_random_dsm_cases_bit_identical_to_reference_dsm_cc(seed, rows, cols, res, radius, pos_x, pos_y, ce, cn,
                                                          density):
    n = max(1, int(density * rows * res * cols * res))
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(-rows * res / 2 - 2, rows * res / 2 + 2, n) + pos_x + cn,
                rng.uniform(-cols * res / 2 - 2, cols * res / 2 + 2, n) + pos_y + ce,
                rng.normal(100.0, 5.0, n)]
    g = po.make_geometry(rows, cols, res, pos_x, pos_y)
    a, b, c = _nan_layer(rows, cols), _nan_layer(rows, cols), _nan_layer(rows, cols)
    st, _ = po.refsrc_dsm_process(g, a, xyz, radius, ce, cn, multi_thread=bool(seed & 1))
    assert st == 0, po.refsrc_last_error()
    assert po.dsm_process(g, b, xyz, radius, ce, cn, num_threads=-1, use_ref=True)[0] == 0
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    st, _, lvl, _ = po.dsm_process(g, c, xyz, radius, ce, cn, num_threads=-1, debug=True)
    assert st == 0
    assert np.array_equal(np.isnan(a), lvl < 0) and ulp_diff(a, c).max() <= 1


@settings(max_examples=25, deadline=None)
@given(seed=hst.integers(0, 100_000), rows=hst.integers(4, 36), cols=hst.integers(4, 36),
       res=hst.sampled_from([0.25, 0.5, 1.0]), dist_type=hst.integers(0, 2), colored=hst.booleans(),
       agl=hst.floats(20.0, 120.0), tilt=hst.floats(0.0, 25.0), n_frames=hst.integers(1, 7))
def test_random_ortho_cases_bit_identical_to_reference_ortho_backward_grid_cc(seed, rows, cols, res, dist_type,
                                                                             colored, agl, tilt, n_frames):
    dist = {0: (0, 0, 0, 0), 1: RADTAN, 2: EQUI}[dist_type]
    camd = synth.scaled_camera(0.03, dist_type=dist_type, dist=dist)
    rng = np.random.default_rng(seed)
    q = np.r_[1.0, rng.normal(0, 0.05, 3)]
    camd["q_C_B"], camd["t_C_B"] = tuple(q / np.linalg.norm(q)), tuple(rng.normal(0, 0.1, 3))
    poses = synth.lawnmower_poses(1, n_frames, rows * res / 2, cols * res / 2, agl, seed=seed, jitter_pos=1.0,
                                  jitter_rp_deg=tilt)
    ch = 3 if colored else 1
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(n_frames)]
    elev = synth.analytic_elevation(rows, cols, res)
    elev[rng.integers(0, rows), rng.integers(0, cols)] = np.nan
    g, cam = po.make_geometry(rows, cols, res), po.make_camera(**camd)
    A, B = fresh_layers(rows, cols, elev), fresh_layers(rows, cols, elev)
    st, _ = po.refsrc_ortho_process(g, A, cam, poses, imgs, colored=colored, multi_thread=bool(seed & 1))
    assert st == 0, po.refsrc_last_error()
    assert po.ortho_process(g, B, cam, poses, imgs, colored=colored, num_threads=-1)[0] == 0
    for k in ("elevation_angle", "observation_index", "ortho", "colored_ortho"):
        assert np.array_equal(A[k].view(np.uint32), B[k].view(np.uint32)), k
