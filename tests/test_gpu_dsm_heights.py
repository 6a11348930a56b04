"""DSM heights of the FP32 gather against the oracle where FP32 height arithmetic goes wrong, in both gather precisions.

The decision tests (test_gpu_dsm_adversarial.py) keep every height near 100 m inside one metre, so that the FP32 gather's
height rounding stays out of the picture.  Here it is the subject.  Two error sources are not covered by the guard band:

  * weights near a cell centre: coordinates are staged as tile-local floats, so d2_f carries an absolute error of about
    2 |d| delta (delta ~ 5e-7 m) and the weight 1/d2 a relative error of about 2 delta / |d|;
  * heights far from the tile offset: heights are staged as float(z - z0), z0 the height of the tile's lowest-id point,
    so the rounding of the sums scales with the tile's height range, not with the cell's own height.

Bars, for every scene:
  f64   counts, levels and NaN mask equal to the oracle; heights <= 1 float32 ulp;
  f32   counts, levels and NaN mask equal to the oracle; |h_gpu - h_oracle| <= 1e-4 |h_oracle| (float64 arithmetic);
  both  the production template, the chunked evaluation and a ragged 3-stripe run bit-identical to the debug run or to
        the undivided map.
The near-centre (1e-4 m, ground near 0) and the 40 m tall-offset scenes are also compared with the reference's own dsm.cc."""
import numpy as np
import pytest

from common import UTM, UTM_SHIFT, Scene, ulp_diff
from aerial_mapper_b200 import synth
from test_gpu_dsm_adversarial import check_reference, gpu_run, oracle_run

pytestmark = pytest.mark.gpu

PRECISIONS = ["f32", "f64"]
TAU = 1e-4          # relative height bound of the FP32 gather (include/aerial_mapper_b200.h)


# ---- checking ---------------------------------------------------------------------------------------------------------
def check_heights(sc, precision):
    """Debug run against the oracle (decisions exact, heights within the precision's bound), then the production template,
    the chunked evaluation and three ragged stripes bit-identical.  Returns the oracle's elevation and the debug run's
    timings."""
    e, cnt, lvl = oracle_run(sc)
    ge, (gc, gl), t = gpu_run(sc, precision, debug=True)
    assert np.array_equal(gl, lvl), "retry level differs in %d cells" % int((gl != lvl).sum())
    touched = lvl >= 0
    assert np.array_equal(gc[touched], cnt[touched]), "neighbour count differs"
    assert np.array_equal(np.isnan(ge), np.isnan(e))
    ok = ~np.isnan(e)
    if precision == "f64":
        assert ulp_diff(ge, e).max() <= 1
    else:
        err = np.abs(ge[ok].astype(np.float64) - e[ok].astype(np.float64))
        lim = TAU * np.abs(e[ok].astype(np.float64))
        bad = err > lim
        worst = float((err / np.maximum(np.abs(e[ok].astype(np.float64)), 1e-300)).max()) if ok.any() else 0.0
        assert not bad.any(), "%d of %d cells beyond %g relative (worst %.3g)" % (int(bad.sum()), int(ok.sum()), TAU,
                                                                                 worst)
    bits = ge.view(np.uint32)
    prod, _, _ = gpu_run(sc, precision)
    assert np.array_equal(prod.view(np.uint32), bits), "production gather differs from the debug run"
    ch, _, _ = gpu_run(sc, precision, chunked=True)
    assert np.array_equal(ch.view(np.uint32), bits), "chunked evaluation differs from the debug run"
    c1, c2 = (sc.cols * 3) // 10 + 1, (sc.cols * 7) // 10 - 3          # ragged: off the 32-column tile edges
    for c0, c1_ in ((0, c1), (c1, c2), (c2, sc.cols)):
        part, _, _ = gpu_run(sc, precision, col_range=(c0, c1_))
        assert np.array_equal(part[:, c0:c1_].view(np.uint32), bits[:, c0:c1_]), ("stripe", c0, c1_)
    return e, t


# ---- scene builders ----------------------------------------------------------------------------------------------------
def carpet(sc, density, z_of, seed, margin=3.0):
    """Uniform random points over the map plus `margin` metres, height z_of(x, y, rng)."""
    rng = np.random.default_rng(seed)
    x0, x1 = sc.qx[-1] - margin, sc.qx[0] + margin
    y0, y1 = sc.qy[-1] - margin, sc.qy[0] + margin
    n = int(density * (x1 - x0) * (y1 - y0))
    x, y = rng.uniform(x0, x1, n), rng.uniform(y0, y1, n)
    z = z_of(x, y, rng)
    for p in zip(x, y, z):
        sc.add(*sc.raw(p[0], p[1]) + (p[2],))


# probe cells at tile-local corners and middles of a 3 x 3 tile map: |local| grows toward the tile's edges
NEAR_PROBES = [(32, 32), (63, 63), (32, 63), (63, 32), (48, 48), (0, 0), (16, 16), (80, 90), (90, 40)]


def near_centre_scene(d, ground, pos=(0.0, 0.0), ce=0.0, cn=0.0):
    """96 x 96 cells @ 0.25 m, r = 1, ground carpet (8 points/m^2) at `ground` +- 2 cm.  At each probe cell, points at
    d, 1.3 d (and 1.7 d) from the cell centre with contrasting heights ground + 20, + 0 (and - 7); the last probe holds a
    single point at d (height ground + 0.3) among the carpet."""
    sc = Scene(96, 96, 0.25, 1, pos, ce, cn)
    for t, (i, j) in enumerate(NEAR_PROBES):
        a = 0.4 + 1.1 * t
        if t == len(NEAR_PROBES) - 1:
            members = [(d, ground + 0.3)]
        elif t % 2:
            members = [(d, ground + 20.0), (1.3 * d, ground), (1.7 * d, ground - 7.0)]
        else:
            members = [(d, ground + 20.0), (1.3 * d, ground)]
        for u, (r, z) in enumerate(members):
            ang = a + 2.0 * u
            sc.add(*sc.raw(sc.qx[i] + r * np.cos(ang), sc.qy[j] + r * np.sin(ang)) + (z,))
    carpet(sc, 8.0, lambda x, y, rng: ground + rng.uniform(-0.02, 0.02, len(x)), seed=int(1e6 * d) % 997 + 5)
    return sc


def tall_scene(tall, ground):
    """128 x 128 cells @ 0.25 m, r = 1, ground carpet at `ground` +- 2 cm; one point `tall` metres high every 8 m of map,
    placed FIRST in the cloud (lowest ids): it is the height offset z0 of every tile whose window holds it."""
    sc = Scene(128, 128, 0.25, 1)
    for gx in np.arange(sc.qx[-1] + 2.0, sc.qx[0], 8.0):
        for gy in np.arange(sc.qy[-1] + 3.0, sc.qy[0], 8.0):
            sc.add(gx + 0.11, gy - 0.07, tall)
    carpet(sc, 8.0, lambda x, y, rng: ground + rng.uniform(-0.02, 0.02, len(x)), seed=17)
    return sc


# ---- near-centre clusters ----------------------------------------------------------------------------------------------
NEAR_D = [1e-3, 1e-4, 1e-5, 1e-6, 1e-9, 1e-12]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("ground", [0.0, 100.0])
@pytest.mark.parametrize("d", NEAR_D)
def test_points_near_a_cell_centre(precision, d, ground):
    sc = near_centre_scene(d, ground)
    e, _ = check_heights(sc, precision)
    for (i, j) in NEAR_PROBES:
        assert np.isfinite(e[i, j])
    if d == 1e-4 and ground == 0.0:
        ref = check_reference(sc, e)
        assert np.array_equal(np.isnan(ref), np.isnan(e))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("where", ["map", "shift"])
def test_points_near_a_cell_centre_at_utm_scale(precision, where):
    kw = dict(pos=UTM) if where == "map" else dict(pos=UTM, ce=UTM_SHIFT[0], cn=UTM_SHIFT[1])
    for d in (1e-3, 1e-4):
        check_heights(near_centre_scene(d, 0.0, **kw), precision)


# ---- tile offset far from the cell -------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("tall,ground", [(40.0, 0.05), (400.0, 0.05), (4000.0, 0.05), (4096.0, 0.05), (-390.0, -430.0)])
def test_tall_point_as_the_tile_height_offset(precision, tall, ground):
    sc = tall_scene(tall, ground)
    e, _ = check_heights(sc, precision)
    assert np.isfinite(e).all()
    if tall == 40.0:
        check_reference(sc, e)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_heights_of_both_signs_that_cancel(precision):
    # isolated probes whose ball holds +7, -7, +3, -3 m at nearly mirrored positions: |h| ~ 1e-3 .. 1e-2, so the relative
    # bound leaves the FP32 sums almost no room.  (Exactly mirrored heights would cancel to ~1e-16, where no summation
    # order, FP64 included, has a relative bound.)
    sc = Scene(96, 96, 0.25, 1)
    probes = [(20, 20), (20, 70), (70, 20), (70, 70)]
    for t, (i, j) in enumerate(probes):
        s = 1.0 + 1e-3 * (t + 1)
        for (dx, dy), z in zip(((0.3, 0.0), (-0.3 * s, 0.0), (0.0, 0.45), (0.0, -0.45 * s)), (7.0, -7.0, 3.0, -3.0)):
            sc.add(sc.qx[i] + dx, sc.qy[j] + dy, z)
    e, _ = check_heights(sc, precision)
    for (i, j) in probes:
        assert 1e-4 < abs(e[i, j]) < 0.1


# ---- many neighbours ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("mean", [0.0, 100.0])
def test_hundreds_of_neighbours_with_spread_heights(precision, mean):
    # r = 3 at 50 points/m^2: ~470 neighbours per cell, heights uniform in mean +- 50 m
    sc = Scene(64, 64, 0.1, 3)
    carpet(sc, 50.0, lambda x, y, rng: mean + rng.uniform(-50.0, 50.0, len(x)), seed=23)
    e, cnt, lvl = oracle_run(sc)
    assert np.median(cnt[lvl == 0]) > 300
    check_heights(sc, precision)


# ---- benign control ----------------------------------------------------------------------------------------------------
# Cells the f32 gather handed to the exact kernel on this input before the height rule existed (guard band only): the
# rule must not hand over a cell of ordinary terrain, not even one with a single point 1e-4 or 1e-5 m from its centre.
# (Closer than ~1e-5 m the staged distance's error is no longer small against the distance itself: such a cell goes to
# the exact kernel whatever its heights.)
BENIGN_LISTED_F32 = 30


def benign_scene():
    rows, cols, res = 128, 160, 0.25
    sc = Scene(rows, cols, res, 1)
    xyz = synth.point_cloud(int(8 * (rows * res + 6) * (cols * res + 6)), rows * res / 2 + 3.0, cols * res / 2 + 3.0,
                            seed=41)
    rng = np.random.default_rng(43)
    for t in range(60):        # single points 1e-4 and 1e-5 m from a cell centre, at the terrain's height
        i, j = int(rng.integers(0, rows)), int(rng.integers(0, cols))
        r, a = 10.0 ** -(4 + t % 2), rng.uniform(0, 2 * np.pi)
        x, y = sc.qx[i] + r * np.cos(a), sc.qy[j] + r * np.sin(a)
        sc.add(x, y, float(synth.terrain(x, y)) + rng.normal(0, 0.05))
    for p in xyz:
        sc.add(*p)
    return sc


@pytest.mark.parametrize("precision", PRECISIONS)
def test_benign_terrain_hands_over_no_more_cells(precision):
    sc = benign_scene()
    e, t = check_heights(sc, precision)
    _, _, lvl = oracle_run(sc)
    if precision == "f64":
        assert t["dsm_cells_empty"] == int((lvl != 0).sum())
    else:
        assert t["dsm_cells_empty"] == BENIGN_LISTED_F32
