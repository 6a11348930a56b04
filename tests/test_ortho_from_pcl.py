""""Next" row N1 (SURVEY §8f): ortho::OrthoFromPcl::process (ortho-from-pcl.cc:20-113) — IDW of point intensities.
CPU: the oracle restatement against brute force and the reference's nanoflann (oracle/_ref).  GPU: the CUDA path
(the DSM kernels with z := intensity) against the oracle."""
import numpy as np
import pytest

from common import ulp_diff
from aerial_mapper_b200 import synth
from oracle import pyoracle as po


def make_cloud(n, half_x, half_y, seed):
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(-half_x, half_x, n), rng.uniform(-half_y, half_y, n), rng.uniform(0, 5, n)]
    inten = rng.integers(0, 256, n).astype(np.int32)
    return xyz, inten


def brute(rows, cols, res, xyz, inten, radius, init):
    qx, qy = synth.grid_positions(rows, cols, res)
    out = init.copy(order="F")
    for j in range(cols):
        dy2 = (qy[j] - xyz[:, 1]) ** 2
        for i in range(rows):
            d2 = (qx[i] - xyz[:, 0]) * (qx[i] - xyz[:, 0]) + dy2
            m = d2 < radius
            if m.any():
                if (d2[m] == 0).any():
                    out[i, j] = np.float32(inten[m][d2[m] == 0][-1])
                else:
                    out[i, j] = np.float32(np.sum(inten[m] / d2[m]) / np.sum(1.0 / d2[m]))
    return out


def test_oracle_matches_brute_force_and_keeps_untouched_cells():
    rows, cols, res = 14, 11, 1.0
    xyz, inten = make_cloud(40, 5.0, 4.0, 1)
    init = np.full((rows, cols), 255.0, np.float32, order="F")
    o = init.copy(order="F")
    assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), o, xyz, inten, radius=2) == 0
    b = brute(rows, cols, res, xyz, inten, 2, init)
    assert ulp_diff(o, b).max() <= 1
    assert (o == 255.0).any() and (o != 255.0).any()


def test_oracle_equals_reference_nanoflann_and_perfect_match():
    if not po.have_ref():
        pytest.skip("oracle/_ref not built (no /root/reference on this box)")
    rows, cols, res = 60, 50, 0.5
    xyz, inten = make_cloud(3000, 16.0, 13.0, 2)
    qx, qy = synth.grid_positions(rows, cols, res)
    xyz[7, :2] = (qx[20], qy[30])       # a point exactly on a cell centre: perfect match, value = its intensity
    g = po.make_geometry(rows, cols, res)
    a = np.full((rows, cols), 255.0, np.float32, order="F")
    b = a.copy(order="F")
    assert po.ortho_from_pcl_process(g, a, xyz, inten, radius=2, num_threads=4) == 0
    assert po.ortho_from_pcl_process(g, b, xyz, inten, radius=2, use_ref=True) == 0
    assert ulp_diff(a, b).max() <= 1
    assert a[20, 30] == np.float32(inten[7]) == b[20, 30]
    # adaptive interpolation (10^k radius growth) through the reference's tree: every cell gets a value
    c = np.full((rows, cols), 255.0, np.float32, order="F")
    sparse = xyz[:5]
    assert po.ortho_from_pcl_process(g, c, sparse, inten[:5], radius=1, adaptive=True, use_ref=True) == 0
    assert (c != 255.0).all()
    assert po.ortho_from_pcl_process(g, c, sparse, inten[:5], radius=1, adaptive=True) == -8   # portable: unsupported
    assert po.ortho_from_pcl_process(g, c, np.zeros((0, 3)), np.zeros(0, np.int32)) == -1     # CHECK(!empty)


def test_oracle_takes_the_last_coincident_point_in_point_order():
    # several points exactly on one cell centre: ortho-from-pcl.cc:90-96 keeps the last perfect match its loop visits;
    # the oracle's loop visits them in point order (one bucket, ascending index), so the largest index wins
    rows, cols, res = 12, 10, 1.0
    qx, qy = synth.grid_positions(rows, cols, res)
    xyz, inten = make_cloud(30, 4.0, 3.0, 8)
    for k in (3, 11, 17, 26):
        xyz[k, :2] = (qx[5], qy[4])
    inten[[3, 11, 17, 26]] = [9, 200, 31, 77]
    o = np.full((rows, cols), 255.0, np.float32, order="F")
    assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), o, xyz, inten, radius=2) == 0
    assert o[5, 4] == 77.0
    b = brute(rows, cols, res, xyz, inten, 2, np.full((rows, cols), 255.0, np.float32, order="F"))
    assert ulp_diff(o, b).max() <= 1


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,res,n,radius,seed", [(120, 90, 0.5, 20000, 2, 3), (64, 64, 1.0, 3000, 10, 4),
                                                         (200, 150, 0.25, 9000, 1, 5)])
def test_gpu_matches_oracle(rows, cols, res, n, radius, seed):
    import aerial_mapper_b200 as amb
    xyz, inten = make_cloud(n, rows * res / 2 + 1, cols * res / 2 + 1, seed)
    qx, qy = synth.grid_positions(rows, cols, res)
    xyz[11, :2] = (qx[rows // 3], qy[cols // 2])   # perfect match
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius)).process(xyz, inten, gm)
    o = np.full((rows, cols), 255.0, np.float32, order="F")
    assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), o, xyz, inten, radius=radius,
                                     num_threads=4) == 0
    assert np.array_equal(gm["ortho"] == 255.0, o == 255.0)       # same untouched cells
    assert ulp_diff(gm["ortho"], o).max() <= 1
    assert gm["ortho"][rows // 3, cols // 2] == np.float32(inten[11])
    assert np.isnan(gm["elevation"]).all()                         # only `ortho` is written
    with pytest.raises(amb.AmbError):
        amb.OrthoFromPcl(amb.OrthoFromPclSettings()).process(np.zeros((0, 3)), [], gm)


# ---- use_adaptive_interpolation (ortho-from-pcl.cc:63-72): csrc/pcl_adaptive_kernels.cu -------------------------------
def adaptive_case(rows, cols, res, n, seed, holes, hole_sides, radius):
    # every point inside the map (the adaptive pass refuses clouds the binning would truncate)
    xyz, inten = make_cloud(n, rows * res / 2 - 0.01, cols * res / 2 - 0.01, seed)
    rng = np.random.default_rng(seed + 1000)
    keep = np.ones(len(xyz), bool)
    for _ in range(holes):
        cx, cy = rng.uniform(-rows * res / 4, rows * res / 4), rng.uniform(-cols * res / 4, cols * res / 4)
        sx, sy = rng.uniform(*hole_sides, 2)
        keep &= ~((np.abs(xyz[:, 0] - cx) < sx / 2) & (np.abs(xyz[:, 1] - cy) < sy / 2))
    return xyz[keep], inten[keep]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,res,n,seed,holes,hole_sides,radius", [
    (120, 90, 0.5, 20000, 3, 3, (4.0, 9.0), 2),       # holes a few metres wide: level 10*r
    (200, 160, 0.25, 30000, 4, 2, (12.0, 20.0), 1),   # 100*r needed in the middle of the larger holes
    (64, 64, 1.0, 40, 5, 0, (1.0, 1.0), 1),           # nearly empty map: most cells need 100*r / 1000*r
    (48, 40, 0.5, 1, 6, 0, (1.0, 1.0), 2),            # a single point: every cell takes its intensity
])
def test_gpu_adaptive_interpolation_matches_the_reference_tree(rows, cols, res, n, seed, holes, hole_sides, radius):
    import aerial_mapper_b200 as amb
    if not po.have_ref():
        pytest.skip("oracle/_ref not present (adaptive mode needs the nanoflann back end)")
    xyz, inten = adaptive_case(rows, cols, res, n, seed, holes, hole_sides, radius)
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius,
                                              use_adaptive_interpolation=True)).process(xyz, inten, gm)
    o = np.full((rows, cols), 255.0, np.float32, order="F")
    assert po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), o, xyz, inten, radius=radius, adaptive=True,
                                     use_ref=True) == 0
    assert np.isfinite(gm["ortho"]).all()                      # adaptive: every cell gets a value
    assert ulp_diff(gm["ortho"], o).max() <= 1
    gm.sync()    # the adaptive pass's own counters must not read as a deferred CHECK failure (round-1 advisor finding)
    plain = np.full((rows, cols), 255.0, np.float32, order="F")
    po.ortho_from_pcl_process(po.make_geometry(rows, cols, res), plain, xyz, inten, radius=radius, num_threads=2)
    assert n < 100 or (plain == 255.0).any()                   # the case really has cells the adaptive pass filled
    if n == 1:
        assert (gm["ortho"] == np.float32(inten[0])).all()


@pytest.mark.gpu
def test_gpu_adaptive_interpolation_restrictions_restore_the_layer():
    import aerial_mapper_b200 as amb
    rows, cols, res = 40, 40, 1.0
    xyz, inten = make_cloud(500, 30.0, 30.0, 7)                # points up to 10 m outside the map: not all are binned
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    before = gm["ortho"].copy(order="F")
    with pytest.raises(amb.AmbError) as ei:
        amb.OrthoFromPcl(amb.OrthoFromPclSettings(use_adaptive_interpolation=True)).process(xyz, inten, gm)
    assert ei.value.status == -8                               # AMB_ERR_UNSUPPORTED
    gm.download()
    assert np.array_equal(gm["ortho"], before)                 # the layer got its content back
