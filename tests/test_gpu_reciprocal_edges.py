"""The DSM and OrthoFromPcl at the distances where the kernels' approximate reciprocals leave their normal domain.

The reference divides twice per neighbour, heights[i] / d2 and 1.0 / d2 (dsm.cc:166-167, ortho-from-pcl.cc:99-100);
the kernels multiply by fast_rcp(d2) (FP64) or rcp_f32(d2_f) (the FP32 gather, tile-local float coordinates).  A map at
(0, 0) with an odd number of rows and columns has its middle row and column at coordinate exactly 0.0, so a point at
(a, y_j) lies at d2 = a * a from the centre of cell (middle row, j), whatever small a is.  The clouds below put one such
point on every cell of the middle cross, with d2 spanning

  * the double subnormals [2^-1074, 2^-1022): where 1 / d2 overflows (below about 5.6e-309) while z / d2 may not, and
    where both stay finite;
  * the first normals above them;
  * the float32 band below 2^-126 (and its edge), where the FP32 gather's staged d2_f is subnormal;

each either alone in its cell's ball or among ordinary neighbours, with heights of both signs (intensities 0 and 255).
The DSM at FP64 and FP32 and OrthoFromPcl plain and adaptive, over the whole map and on a column stripe, must write what
the oracle writes: the same NaN mask, the same infinities, finite values within 1 float32 ulp (the FP32 DSM: or within
its documented 1e-4 relative bound).

The `gpu` tests also run on the emulated kernels (tests/emu) through the last test of this file."""
import itertools

import numpy as np
import pytest

from common import ulp_diff
from oracle import pyoracle as po

RADIUS = 1
# |offset| a of the edge point from its cell centre: d2 = a * a
OFFSETS = [
    2.0 ** -537,             # d2 = 2^-1074, the smallest subnormal
    2.0 ** -530,             # 2^-1060
    7e-155,                  # ~4.9e-309: 1 / d2 overflows
    2.0 ** -512,             # 2^-1024: 1 / d2 = 2^1024 overflows
    1.0e-154,                # ~1e-308: subnormal, 1 / d2 finite
    1.49e-154,               # just below 2^-1022
    2.0 ** -511,             # 2^-1022, the smallest normal
    1.5e-154,                # the first normals above it
    2.0 ** -70,              # float32 band: d2_f = 2^-140, subnormal
    2.0 ** -63.5,            # 2^-127
    2.0 ** -63,              # 2^-126, the smallest normal float
    3e-19,                   # 9e-38, just above it
]
HEIGHTS = [0.0, 1e-3, -1e-3, 0.75, -0.75, 123.5, -123.5]
INTENSITIES = [0, 255]


def edge_points(rows, cols, res, combos, mixed, seed):
    """One edge point per cell of the middle cross, (a, z) from `combos` in turn; `mixed`: three ordinary neighbours
    per such cell too, heights +-[1, 9)."""
    from aerial_mapper_b200 import synth
    qx, qy = synth.grid_positions(rows, cols, res)
    ci, cj = rows // 2, cols // 2
    assert qx[ci] == 0.0 and qy[cj] == 0.0
    cells = [(ci, j) for j in range(cols)] + [(i, cj) for i in range(rows) if i != ci]
    rng = np.random.default_rng(seed)
    pts = []
    for k, (i, j) in enumerate(cells[:len(combos)]):
        a, z = combos[k]
        # on the middle row the offset is along x, on the middle column along y (both signs)
        pts.append((qx[i] + (a if k % 2 else -a), qy[j], z) if i == ci else (qx[i], qy[j] + (a if k % 2 else -a), z))
        if mixed:
            for _ in range(3):
                r, t = rng.uniform(0.2, 0.9) * min(res, 1.0), rng.uniform(0, 2 * np.pi)
                pts.append((qx[i] + r * np.cos(t), qy[j] + r * np.sin(t), rng.choice([-1.0, 1.0]) * rng.uniform(1, 9)))
    return np.array(pts, np.float64)


def cloud_batches(rows, cols, res, values, mixed, seed):
    """Every (offset, value) combination, spread over as many clouds as the middle cross needs."""
    combos = list(itertools.product(OFFSETS, values))
    n_cells = rows + cols - 1
    for b in range(0, len(combos), n_cells):
        yield edge_points(rows, cols, res, combos[b:b + n_cells], mixed, seed + b)


def assert_matches(got, want, c0, c1, rel=None, what=""):
    g, w = got[:, c0:c1], want[:, c0:c1]
    nan_g, nan_w = np.isnan(g), np.isnan(w)
    assert np.array_equal(nan_g, nan_w), (what, np.argwhere(nan_g != nan_w)[:5].tolist())
    inf_w = np.isinf(w)
    assert np.array_equal(g[inf_w], w[inf_w]) and not np.isinf(g[~inf_w]).any(), what
    fin = np.isfinite(w)
    ok = ulp_diff(g[fin], w[fin]) <= 1
    if rel is not None:
        ok |= np.abs(g[fin].astype(np.float64) - w[fin]) <= rel * np.abs(w[fin].astype(np.float64))
    bad = np.argwhere(fin)[~ok]
    assert ok.all(), (what, [(tuple(ij), float(g[tuple(ij)]), float(w[tuple(ij)])) for ij in bad[:5]])


def adaptive_reference(n, res, xyz, inten, radius):
    """ortho-from-pcl.cc:58-106 with use_adaptive_interpolation, restated in numpy (the oracle restates the plain pass
    only): balls of radius, 10 radius, 100 radius, ... until one is non-empty, IEEE divisions per neighbour."""
    from aerial_mapper_b200 import synth
    qx, qy = synth.grid_positions(n, n, res)
    out = np.empty((n, n), np.float32, order="F")
    z = inten.astype(np.float64)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        for j in range(n):
            for i in range(n):
                dx, dy = qx[i] - xyz[:, 0], qy[j] - xyz[:, 1]
                d2 = dx * dx + dy * dy
                thr, lam = float(radius), 10
                while not (d2 < thr).any():
                    thr, lam = float(lam * radius), lam * 10
                m = d2 < thr
                assert (d2[m] > 0).all()   # (no perfect match in these clouds)
                out[i, j] = np.sum(z[m] / d2[m]) / np.sum(1.0 / d2[m])
    return out


MAPS = [(5, 1.0), (5, 0.5), (33, 1.0), (33, 0.5)]


def stripe_of(n):
    return (1, 4) if n == 5 else (5, 20)


def grid_map(n, res, col_range):
    import aerial_mapper_b200 as amb
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, n * res, n * res, res)).getMutable()
    if col_range is not None:
        gm.context(0, col_range)
    return gm


@pytest.mark.gpu
@pytest.mark.parametrize("stripe", [False, True], ids=["whole", "stripe"])
@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("mixed", [False, True], ids=["alone", "mixed"])
@pytest.mark.parametrize("n,res", MAPS)
def test_dsm_at_subnormal_distances_writes_what_the_oracle_writes(n, res, mixed, precision, stripe):
    import aerial_mapper_b200 as amb
    c0, c1 = stripe_of(n) if stripe else (0, n)
    g = po.make_geometry(n, n, res)
    for xyz in cloud_batches(n, n, res, HEIGHTS, mixed, seed=7 * n):
        want = np.full((n, n), np.nan, np.float32, order="F")
        st, _, _, _ = po.dsm_process(g, want, xyz, radius=RADIUS, num_threads=-1)
        assert st == 0
        gm = grid_map(n, res, (c0, c1) if stripe else None)
        dsm = amb.Dsm(amb.DsmSettings(interpolation_radius=RADIUS), gm)
        dsm.precision = precision
        dsm.process(xyz, gm)
        assert_matches(gm["elevation"], want, c0, c1, rel=1e-4 if precision == "f32" else None, what=precision)
        if po.have_ref():
            ref = np.full((n, n), np.nan, np.float32, order="F")
            assert po.dsm_process(g, ref, xyz, radius=RADIUS, use_ref=True)[0] == 0
            assert_matches(gm["elevation"], ref, c0, c1, rel=1e-4 if precision == "f32" else None, what="ref")


@pytest.mark.gpu
@pytest.mark.parametrize("stripe", [False, True], ids=["whole", "stripe"])
@pytest.mark.parametrize("adaptive", [False, True], ids=["plain", "adaptive"])
@pytest.mark.parametrize("mixed", [False, True], ids=["alone", "mixed"])
@pytest.mark.parametrize("n,res", MAPS)
def test_ortho_from_pcl_at_subnormal_distances_writes_what_the_oracle_writes(n, res, mixed, adaptive, stripe):
    import aerial_mapper_b200 as amb
    c0, c1 = stripe_of(n) if stripe else (0, n)
    g = po.make_geometry(n, n, res)
    for xyz in cloud_batches(n, n, res, INTENSITIES, mixed, seed=11 * n):
        inten = np.abs(xyz[:, 2]).astype(np.int32)   # 0 and 255 on the edge points, 1..8 on the others
        gm = grid_map(n, res, (c0, c1) if stripe else None)
        init = np.array(gm["ortho"], np.float32, order="F")   # what a cell keeps where nothing is written
        if adaptive:
            want = adaptive_reference(n, res, xyz, inten, RADIUS)
        else:
            want = init.copy(order="F")
            assert po.ortho_from_pcl_process(g, want, xyz, inten, radius=RADIUS, num_threads=-1) == 0
        amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=RADIUS,
                                                  use_adaptive_interpolation=adaptive)).process(xyz, inten, gm)
        assert_matches(gm["ortho"], want, c0, c1, what="adaptive" if adaptive else "plain")
        if po.have_ref():
            ref = init.copy(order="F")
            assert po.ortho_from_pcl_process(g, ref, xyz, inten, radius=RADIUS, adaptive=adaptive, use_ref=True) == 0
            assert_matches(gm["ortho"], ref, c0, c1, what="ref")


def test_the_gpu_tests_of_this_file_pass_on_the_emulated_kernels():
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_reciprocal_edges.py"])
    assert " passed" in tail and "failed" not in tail
