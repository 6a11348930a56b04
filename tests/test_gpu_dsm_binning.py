"""The DSM's two-level binning (csrc/dsm_partition.inc: P1 dsm_partition_kernel, the scans, P2 dsm_fine_scatter_kernel)
checked bucket by bucket through amb_dsm_download_bins, against an independent numpy assignment of every point to its
bucket.

After every call: the bucket starts are monotone and end at the number of in-grid points, every bucket holds exactly the
ids the independent assignment puts there, every record is bit-exact (shifted x and y, z or the intensity, id word and
fine-bin code) and, in OrthoFromPcl mode, the canonical order sorts each bucket by id.

The number of coarse destinations S (a band of bucket columns per destination) follows the bytes per destination,
AMB_DSM_PART_WINDOW, which the library reads once per process: the cases that need S > 1 run in a child process that
sets it, and must reach the S they intend.  Their output layers must be bit-identical to the same scene binned with
S = 1, in both gather precisions (AMB_DSM_PRECISION, inherited by the children), for the DSM and adaptive OrthoFromPcl.
The S = 1 runs are compared with the oracle to the bars of test_gpu_dsm.py."""
import ctypes as C
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from common import ROOT, UTM, UTM_SHIFT, ulp_diff  # noqa: E402
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import synth  # noqa: E402

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
PRECISION = os.environ.get("AMB_DSM_PRECISION", "f32").lower()
REL = 1e-6
MAX_ULP = 1 if PRECISION == "f64" else 4
TILE = 2048          # points per partition tile (kPartTile)
MAX_COARSE = 256     # kMaxCoarse
TJ = TI = 32         # gather tile extents
LAYOUT = 10          # AMB_DSM_BINS_LAYOUT


# ---- the bins as the library left them ----------------------------------------------------------------------------
def download_bins(ctx):
    L = amb.lib()
    lay = np.zeros(LAYOUT, np.int32)
    amb.check(L.amb_dsm_download_bins(ctx, lay.ctypes.data, None, None, None), ctx)
    B, Pa, BR, BC, KR, KC, gj0, tile_j0, nb, S = (int(v) for v in lay)
    G = np.zeros(KR * KC + 1, np.uint32)
    rec = np.zeros((max(nb, 1), 4), np.float64)
    order = np.zeros(max(nb, 1), np.uint32)
    amb.check(L.amb_dsm_download_bins(ctx, lay.ctypes.data, G.ctypes.data, rec.ctypes.data, order.ctypes.data), ctx)
    return dict(B=B, Pa=Pa, BR=BR, BC=BC, KR=KR, KC=KC, gj0=gj0, tile_j0=tile_j0, n_binned=nb, S=S, G=G,
                rec=rec[:nb], order=order[:nb])


# ---- the independent assignment -------------------------------------------------------------------------------------
def fine_index(base, p, inv_res):
    """floor(fma(base - p, inv_res, 0.5)) per element, the FMA correctly rounded: evaluated un-fused first, and again
    with exact rationals wherever the un-fused argument lies within a few ulps of an integer."""
    d = base - np.asarray(p, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        prod = d * inv_res
        t = prod + 0.5
        f = np.floor(t)
        tol = 4.0 * (np.spacing(np.abs(prod)) + np.spacing(np.abs(t)))
        near = np.isfinite(t) & (np.abs(t - np.round(t)) <= tol)
    for k in np.flatnonzero(near):
        f[k] = math.floor(float(Fraction(float(d[k])) * Fraction(inv_res) + Fraction(1, 2)))
    return f


def fma_differs_from_unfused(base, p, inv_res):
    """True where floor(fma(base - p, inv_res, 0.5)) and floor((base - p) * inv_res + 0.5) disagree."""
    d = base - np.asarray(p, np.float64)
    return fine_index(base, p, inv_res) != np.floor(d * inv_res + 0.5)


def thresholds(radius, mode):
    if mode == "pcl":
        return [float(radius)]
    thr, lam = [], 1.0
    while True:     # dsm.cc:133-144
        thr.append(lam * radius)
        lam *= 1.1
        if lam * radius > 7.0:
            return thr


def round_up(a, b):
    return (a + b - 1) // b * b


def expected_layout(sc, n, whole_map=False):
    """B, Pa, BR, BC, KR, KC, gj0 and tile_j0 restated from the geometry (dsm_run's plan)."""
    rows, cols, res = sc["rows"], sc["cols"], sc["res"]
    thr = thresholds(sc["radius"], sc["mode"])
    W = int(math.floor(math.sqrt(float(sc["radius"])) / res + 0.5 + 1e-6))
    P = max(int(math.floor(math.sqrt(max(thr)) / res + 0.5 + 1e-6)), W)
    per_cell = sc["hint"] if sc.get("hint") else n / float(rows * cols)
    B = 1
    while B < 16 and per_cell * (2.0 * B) * (2.0 * B) <= 48.0:
        B *= 2
    c0, c1 = (0, cols) if whole_map or sc.get("col_range") is None else sc["col_range"]
    Pa = round_up(P, B)
    tile_j0, tile_j1 = c0 // TJ, (c1 - 1) // TJ
    gj0 = tile_j0 * TJ - Pa
    BR = round_up(round_up(rows, TI) + 2 * Pa, B)
    BC = round_up((tile_j1 + 1) * TJ + Pa - gj0, B)
    return dict(B=B, Pa=Pa, BR=BR, BC=BC, KR=BR // B, KC=BC // B, gj0=gj0, tile_j0=tile_j0)


def destinations(n, KC, window):
    """S as the partition derives it: ceil(32 n / window) bands, at most kMaxCoarse and KC, of whole bucket columns."""
    s = max(1, min(-(-(32 * n) // window), MAX_COARSE, KC))
    kj_per = -(-KC // s)
    return -(-KC // kj_per), kj_per


def check_bins(sc, bins, xyz, ids, z):
    """Every bin against the independent assignment of (xyz, ids, z): the exact input the binning was given."""
    B, KR, KC = bins["B"], bins["KR"], bins["KC"]
    shift = B.bit_length() - 1
    g = sc["geometry"]
    inv_res = 1.0 / g.resolution
    base_x = g.pos_x + (0.5 * g.length_x - 0.5 * g.resolution)
    base_y = g.pos_y + (0.5 * g.length_y - 0.5 * g.resolution)
    px = xyz[:, 0] - sc["cn"]
    py = xyz[:, 1] - sc["ce"]
    fi = fine_index(base_x, px, inv_res) + bins["Pa"]
    fj = fine_index(base_y, py, inv_res) - bins["gj0"]
    with np.errstate(invalid="ignore"):
        inside = (fi >= 0) & (fi < bins["BR"]) & (fj >= 0) & (fj < bins["BC"])
    bi, bj = fi[inside].astype(np.int64), fj[inside].astype(np.int64)
    eb = (bi >> shift) + (bj >> shift) * KR
    eid = ids[inside].astype(np.uint64) & np.uint64(0xffffffff)
    assert len(np.unique(eid)) == len(eid), "the scene's ids must be unique"

    G = bins["G"].astype(np.int64)
    nb = bins["n_binned"]
    assert G[0] == 0 and (np.diff(G) >= 0).all(), "bucket starts not monotone"
    assert nb == int(inside.sum()), "binned %d points, %d lie in the bin grid" % (nb, int(inside.sum()))
    assert G[-1] == nb, "bucket starts end at %d, %d points binned" % (G[-1], nb)
    counts = np.bincount(eb, minlength=KR * KC)
    bad = np.flatnonzero(counts != np.diff(G))
    assert len(bad) == 0, "%d buckets hold the wrong number of records, first %s: %d instead of %d" % (
        len(bad), bad[0], np.diff(G)[bad[0]], counts[bad[0]])

    rec = bins["rec"]
    word = rec[:, 3].copy().view(np.uint64)
    rid = word & np.uint64(0xffffffff)
    rb = np.repeat(np.arange(KR * KC), np.diff(G))
    o_r = np.lexsort((rid, rb))
    o_e = np.lexsort((eid, eb))
    assert np.array_equal(rid[o_r], eid[o_e]), "a bucket holds other ids than the assignment puts there"
    bits = lambda a: np.ascontiguousarray(a, np.float64).view(np.uint64)  # noqa: E731
    assert np.array_equal(bits(rec[o_r, 0]), bits(px[inside][o_e])), "x - center_northing not bit-exact"
    assert np.array_equal(bits(rec[o_r, 1]), bits(py[inside][o_e])), "y - center_easting not bit-exact"
    assert np.array_equal(bits(rec[o_r, 2]), bits(z[inside][o_e])), "height / intensity not bit-exact"
    code = ((bi.astype(np.uint64) << np.uint64(4)) | (bj.astype(np.uint64) & np.uint64(15)))
    assert np.array_equal(word[o_r] >> np.uint64(32), code[o_e]), "fine-bin code differs"
    if sc["mode"] == "pcl":   # OrthoFromPcl orders every bucket by id
        order = bins["order"].astype(np.int64)
        assert np.array_equal(np.sort(order), np.arange(nb)), "order is not a permutation of the records"
        assert np.array_equal(rb[order], rb), "order leaves a bucket"
        assert np.array_equal(rid[order], rid[o_r]), "order does not sort a bucket by id"
    return int(inside.sum())


# ---- scenes ---------------------------------------------------------------------------------------------------------
def scene(rows, cols, res, xyz, radius=1, pos=(0.0, 0.0), ce=0.0, cn=0.0, ids=None, inten=None, mode="dsm",
          adaptive=False, col_range=None, hint=16.0):
    """hint: amb_dsm_set_density_hint.  More than 12 points per cell gives 1-cell buckets (B = 1): many bucket columns
    from a small cloud, and every fine bin its own bucket."""
    xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
    if mode == "pcl" and inten is None:
        inten = np.random.default_rng(len(xyz)).integers(0, 256, len(xyz)).astype(np.int32)
    return dict(rows=rows, cols=cols, res=res, xyz=xyz, radius=radius, pos=pos, ce=ce, cn=cn, ids=ids, inten=inten,
                mode=mode, adaptive=adaptive, col_range=col_range, hint=hint)


# the main geometry: res 0.16 m, radius 1 -> reach 16 cells = Pa; B = 1: BC = 8 * 32 + 2 * 16 = 288 bucket columns
A = dict(rows=40, cols=250, res=0.16)


def uniform(n, seed, rows=A["rows"], cols=A["cols"], res=A["res"], margin=1.0, holes=0, hole_sides=(0.5, 1.5)):
    return synth.point_cloud(n, rows * res / 2 + margin, cols * res / 2 + margin, seed, holes=holes,
                             hole_sides=hole_sides)


def y_of_bin(bj, gj0, res, cols, jitter, rng, pos_y=0.0):
    """Shifted y of points in bin column bj (global column gj0 + bj), up to `jitter` cells off the centre."""
    base_y = pos_y + (0.5 * cols * res - 0.5 * res)
    return base_y - res * (np.asarray(bj, np.float64) + gj0) + rng.uniform(-jitter, jitter, np.shape(bj)) * res


def columns_scene(which, n=6000, seed=3):
    """Points confined to bin columns: of the first or the last of S = 7 destinations (kj_per = 42 on the main
    geometry), or point k in destination k mod 7."""
    rng = np.random.default_rng(seed)
    rows, cols, res = A["rows"], A["cols"], A["res"]
    gj0, KC, kj = -16, 288, 42
    if which == "first":
        bj = rng.integers(0, kj, n)
    elif which == "last":
        bj = rng.integers(6 * kj, KC, n)
    else:   # destination k mod 7, the last one ragged (36 columns)
        d = np.arange(n) % 7
        bj = d * kj + rng.integers(0, np.where(d == 6, KC - 6 * kj, kj))
    y = y_of_bin(bj, gj0, res, cols, 0.45, rng)
    x = rng.uniform(-rows * res / 2 - 1.0, rows * res / 2 + 1.0, n)
    return scene(rows, cols, res, np.c_[x, y, synth.terrain(x, y)])


def edge_scene(seed=4):
    """Points on the outermost bin rows and columns of the grid (kept) and one bin beyond them (dropped)."""
    rng = np.random.default_rng(seed)
    rows, cols, res = A["rows"], A["cols"], A["res"]
    Pa, gj0, BR, BC = 16, -16, 96, 288
    base_x = 0.5 * rows * res - 0.5 * res
    pts = []
    for bi in (-1, 0, BR - 1, BR):
        for bj in rng.integers(0, BC, 40):
            pts.append((bi, bj))
    for bj in (-1, 0, BC - 1, BC):
        for bi in rng.integers(0, BR, 40):
            pts.append((bi, bj))
    bi, bj = np.array(pts).T
    x = base_x - res * (bi - Pa) + rng.uniform(-0.45, 0.45, len(bi)) * res
    y = y_of_bin(bj, gj0, res, cols, 0.45, rng)
    inner = uniform(3000, seed)
    xyz = np.r_[np.c_[x, y, 50.0 + rng.uniform(-1, 1, len(x))], inner]
    return scene(rows, cols, res, xyz[rng.permutation(len(xyz))])


def tie_scene(res, utm):
    """Shifted coordinates exactly on fine-bin edges (fma(base - p, 1/res, 0.5) an integer), one ulp either side, and
    every coordinate near an edge where the fused and the un-fused expression floor differently.  P2 recomputes the
    column from the stored y: these are where P1 and P2 could disagree.

    With 0.5 exact, fused and un-fused can only floor differently where base - p and the argument lie in different
    binades: the edges of index 0 (argument near 0 and near 1).  The local variant places the map so that those edges
    lie near p = 0, where doubles are dense enough to land there, and scans them finely."""
    rows, cols = 24, 64
    if utm:
        pos, ce, cn = UTM, UTM_SHIFT[0], UTM_SHIFT[1]
    else:
        pos, ce, cn = (-0.5 * rows * res, -0.5 * cols * res), 2.0 ** -20, -(2.0 ** -21)
    g = amb.AerialGridMap(amb.GridMapSettings(pos[0], pos[1], rows * res, cols * res, res)).getMutable().geometry
    inv = 1.0 / g.resolution
    base_x = g.pos_x + (0.5 * g.length_x - 0.5 * g.resolution)
    base_y = g.pos_y + (0.5 * g.length_y - 0.5 * g.resolution)
    rng = np.random.default_rng(int(res * 1000) + utm)

    def near_edges(base, shift, n_edges, lo, hi):
        out, differ = [], 0
        for k in sorted(set(range(lo, hi, max(1, (hi - lo) // n_edges))) | {0, 1}):
            p0 = base - (k - 0.5) * res
            raw0 = p0 + shift
            span = 48 if (utm or k not in (0, 1)) else 3000
            # steps of one ulp of the coarsest of raw, p and base - p: finer steps would not move base - p
            raw = raw0 + np.arange(-span, span + 1) * np.spacing(max(abs(raw0), abs(p0), abs(base - p0)))
            p = raw - shift
            exact = np.array([Fraction(float(base - q)) * Fraction(inv) + Fraction(1, 2) for q in p])
            tie = np.array([e.denominator == 1 for e in exact])
            dif = fma_differs_from_unfused(base, p, inv)
            keep = dif | tie | np.r_[tie[1:], False] | np.r_[False, tie[:-1]]
            keep[span] = True     # the nominal edge
            differ += int(dif.sum())
            out.append(raw[keep])
        return np.concatenate(out), differ

    ys, ydiff = near_edges(base_y, ce, 24, -10, cols + 10)
    xs, xdiff = near_edges(base_x, cn, 12, -10, rows + 10)
    n_y, n_x = len(ys), len(xs)
    x_for_y = rng.uniform(base_x - rows * res, base_x, n_y) + cn
    y_for_x = rng.uniform(base_y - cols * res, base_y, n_x) + ce
    bg = synth.point_cloud(2500, rows * res / 2 + 0.5, cols * res / 2 + 0.5, 9, center=(pos[0] + cn, pos[1] + ce))
    x, y = np.r_[x_for_y, xs], np.r_[ys, y_for_x]
    xyz = np.r_[np.c_[x, y, synth.terrain(x, y) + rng.normal(0.0, 0.05, len(x))], bg]
    sc = scene(rows, cols, res, xyz[rng.permutation(len(xyz))], pos=pos, ce=ce, cn=cn)
    sc["fma_differs"] = ydiff
    return sc


def ids_of(n):
    """Caller ids that are not positions, ascending (the canonical order stays the array order), 3 .. 2^32 - 1."""
    ids = np.uint64(3) + np.arange(n, dtype=np.uint64) * np.uint64((2 ** 32 - 4) // max(n - 1, 1))
    ids[-1] = 2 ** 32 - 1
    return ids


def make_scene(name):
    rows, cols, res = A["rows"], A["cols"], A["res"]
    if name == "uniform":
        return scene(rows, cols, res, uniform(6000, 1, holes=3))
    if name.startswith("n="):        # partition-tile edges
        n = int(name[2:])
        return scene(rows, cols, res, uniform(n, n % 1000 + 5))
    if name == "one_bucket":
        rng = np.random.default_rng(6)
        base_x, base_y = 0.5 * rows * res - 0.5 * res, 0.5 * cols * res - 0.5 * res
        x = base_x - res * 17 + rng.uniform(-0.4, 0.4, 5000) * res
        y = base_y - res * 100 + rng.uniform(-0.4, 0.4, 5000) * res
        return scene(rows, cols, res, np.c_[x, y, rng.uniform(0, 3, 5000)])
    if name in ("first", "last", "mod"):
        return columns_scene(name)
    if name == "descending_column":   # column j grows as y falls: ascending y
        xyz = uniform(7000, 7)
        return scene(rows, cols, res, xyz[np.argsort(xyz[:, 1], kind="stable")])
    if name == "tile_outside":        # tiles 0 and 2 in the grid, tile 1 wholly beyond the apron (binned: 0)
        xyz = uniform(3 * TILE, 8)
        xyz[TILE:2 * TILE, 0] += 1e4
        return scene(rows, cols, res, xyz)
    if name == "non_finite":
        xyz = uniform(6000, 10)
        for k, v in enumerate((np.nan, np.inf, -np.inf, 1e300, -1e300)):
            xyz[100 + 7 * k::211, 0] = v
            xyz[150 + 11 * k::223, 1] = v
        return scene(rows, cols, res, xyz)
    if name == "edges":
        return edge_scene()
    if name.startswith("ties"):       # ties_<res>_<utm|local>
        _, r, where = name.split("_")
        return tie_scene(float(r), where == "utm")
    if name == "ids":
        xyz = uniform(5000, 11)
        return scene(rows, cols, res, xyz, ids=ids_of(len(xyz)))
    if name == "intensity":
        return scene(rows, cols, res, uniform(5000, 12), radius=2, mode="pcl")
    if name == "adaptive":
        return scene(rows, cols, res, uniform(6000, 13, margin=0.5, holes=4, hole_sides=(3.0, 5.0)), mode="pcl",
                     adaptive=True)
    if name == "stripe":              # gj0 = 32 - 16 != -Pa
        return scene(rows, cols, res, uniform(6000, 14), col_range=(45, 170))
    if name == "adaptive_stripe":     # the whole-map re-binning of a stripe
        return scene(rows, cols, res, uniform(6000, 15, margin=0.5, holes=4, hole_sides=(3.0, 5.0)), mode="pcl",
                     adaptive=True, col_range=(45, 170))
    # exactly kMaxCoarse destinations: KC = 224 + 32 = 256 (kj_per = 1) or 480 + 32 = 512 (kj_per = 2)
    if name == "kc256":
        return scene(24, 224, res, uniform(5000, 16, rows=24, cols=224))
    if name == "kc512":
        return scene(16, 480, res, uniform(5000, 17, rows=16, cols=480))
    if name == "kc42":                # KC = 32 + 2 * 5 = 42 clamps a requested S of 256
        return scene(40, 20, 0.5, uniform(3000, 18, rows=40, cols=20, res=0.5))
    raise KeyError(name)


# ---- running a scene ------------------------------------------------------------------------------------------------
def device_array(a):
    """(owner, device pointer) of a copy of `a` on the device; the emulation's device memory is host memory."""
    a = np.ascontiguousarray(a)
    if EMULATED:
        return a, a.ctypes.data
    import torch
    t = torch.from_numpy(a).to("cuda:0")
    return t, t.data_ptr()


def grid_map(sc):
    rows, cols, res, pos = sc["rows"], sc["cols"], sc["res"], sc["pos"]
    gm = amb.AerialGridMap(amb.GridMapSettings(pos[0], pos[1], rows * res, cols * res, res)).getMutable()
    gm.to_device(0, col_range=sc["col_range"], names=("ortho" if sc["mode"] == "pcl" else "elevation",))
    return gm


def run_scene(sc, gm=None):
    """One call on `gm` (a fresh map by default); checks the bins it leaves.  Returns (layer slab, debug, bins)."""
    gm = gm or grid_map(sc)
    sc["geometry"] = gm.geometry
    ctx = gm.context()
    if sc["hint"]:
        amb.check(amb.lib().amb_dsm_set_density_hint(ctx, float(sc["hint"])), ctx)
    xyz, n = sc["xyz"], len(sc["xyz"])
    ids = sc["ids"]
    keep = [device_array(xyz)]
    d_ids = None
    if ids is not None:
        keep.append(device_array(ids.view(np.int64)))
        d_ids = keep[-1][1]
    dbg = None
    if sc["mode"] == "pcl":
        keep.append(device_array(sc["inten"]))
        amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=sc["radius"],
                                                  use_adaptive_interpolation=sc["adaptive"])).process_device(
            keep[0][1], keep[-1][1], n, gm, d_ids=d_ids)
        layer, z = "ortho", sc["inten"].astype(np.float64)
    else:
        d = amb.Dsm(amb.DsmSettings(interpolation_radius=sc["radius"], center_easting=sc["ce"],
                                    center_northing=sc["cn"]), gm)
        d.debug = True
        d.process_device(keep[0][1], n, gm, d_ids=d_ids)
        layer, z = "elevation", xyz[:, 2]
    gm.sync()
    if sc["mode"] == "dsm":
        d._fetch_debug(gm)
        dbg = d.last_debug
    gm.download((layer,))
    bins = download_bins(ctx)
    whole = sc["adaptive"] and sc["col_range"] is not None
    exp = expected_layout(sc, n, whole_map=whole)
    got = {k: bins[k] for k in exp}
    assert got == exp, (got, exp)
    check_bins(sc, bins, xyz, np.arange(n, dtype=np.uint64) if ids is None else ids, z)
    c0, c1 = gm._col_range
    return gm[layer][:, c0:c1].copy(), dbg, bins


def window_for(n, S):
    """Bytes per destination for which the partition asks for S destinations: ceil(32 n / window) = S."""
    w = -(-(32 * n) // S)
    while -(-(32 * n) // w) > S:
        w += 1
    assert -(-(32 * n) // w) == S
    return w


def run_in_child(name, window, tmp_path):
    """Run scene `name` (or the reuse sequence) in a process whose partition uses `window` bytes per destination."""
    out = str(tmp_path / ("%s_%d.npz" % (name.replace("=", ""), window)))
    env = dict(os.environ, AMB_DSM_PART_WINDOW=str(window))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), name, out], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    z = np.load(out)
    return [int(s) for s in z["S"]], [z["layer%d" % k] for k in range(len(z["S"]))]


def child_main(name, out):
    if name == "reuse":
        results = reuse_sequence()
    else:
        layer, _, bins = run_scene(make_scene(name))
        results = [(layer, bins["S"])]
    np.savez(out, S=np.array([s for _, s in results]), **{"layer%d" % k: l for k, (l, _) in enumerate(results)})


# ---- end-to-end: the oracle ----------------------------------------------------------------------------------------
def check_against_oracle(sc, layer, dbg):
    from oracle import pyoracle as po
    rows, cols, res, pos = sc["rows"], sc["cols"], sc["res"], sc["pos"]
    g = po.make_geometry(rows, cols, res, pos[0], pos[1])
    c0, c1 = sc["col_range"] or (0, cols)
    if sc["mode"] == "pcl":
        o = np.full((rows, cols), 255.0, np.float32, order="F")
        assert po.ortho_from_pcl_process(g, o, sc["xyz"], sc["inten"], radius=sc["radius"]) == 0
        o = o[:, c0:c1]
        filled = o != 255.0
        assert ulp_diff(layer[filled], o[filled]).max() <= 1
        if not sc["adaptive"]:
            assert np.array_equal(filled, layer != 255.0)
            return
        # adaptive: the cells the primary ball leaves empty take the 10^k r balls (the reference's own loop, where built)
        assert np.isfinite(layer).all() and (layer != 255.0).all() and (~filled).any()
        if po.have_ref():
            ref = np.full((rows, cols), 255.0, np.float32, order="F")
            assert po.ortho_from_pcl_process(g, ref, sc["xyz"], sc["inten"], radius=sc["radius"], adaptive=True,
                                             use_ref=True) == 0
            assert ulp_diff(layer, ref[:, c0:c1]).max() <= 1
        return
    e = np.full((rows, cols), np.nan, np.float32, order="F")
    st, cnt, lvl, _ = po.dsm_process(g, e, sc["xyz"], radius=sc["radius"], center_easting=sc["ce"],
                                     center_northing=sc["cn"], debug=True)
    assert st == 0
    e, cnt, lvl = e[:, c0:c1], cnt[:, c0:c1], lvl[:, c0:c1]
    gc, gl = dbg
    assert np.array_equal(gl, lvl), "retry-threshold index differs in %d cells" % int((gl != lvl).sum())
    touched = lvl >= 0
    assert np.array_equal(gc[touched], cnt[touched]), "neighbour count differs"
    assert np.array_equal(np.isnan(layer), np.isnan(e))
    ok = ~np.isnan(e)
    assert np.allclose(layer[ok], e[ok], rtol=REL, atol=0.0)
    assert ulp_diff(layer, e).max() <= MAX_ULP


def bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


# ---- 1. destination counts: S = 1, 2, 7, 256 and a clamped S; skewed clouds at S = 7 -------------------------------
WINDOW_CASES = [
    # scene, S the window asks for, S the partition must reach
    ("uniform", 2, 2),
    ("uniform", 7, 7),            # kj_per = 42: the last destination has 36 columns
    ("uniform", 256, 144),        # 256 requested of 288 columns: kj_per = 2
    ("kc256", 256, 256),          # S = kMaxCoarse with kj_per = 1: only lane 31 writes offs[S]
    ("kc512", 256, 256),          # S = kMaxCoarse with kj_per = 2
    ("kc42", 256, 42),            # clamped by KC
    ("first", 7, 7),
    ("last", 7, 7),
    ("mod", 7, 7),
    ("one_bucket", 7, 7),
    ("descending_column", 7, 7),
    ("tile_outside", 7, 7),
    ("non_finite", 7, 7),
    ("edges", 7, 7),
    ("ties_0.1_local", 7, 7),
    ("ids", 7, 7),
    ("intensity", 7, 7),
    ("adaptive", 7, 7),
    ("adaptive", 256, 134),       # OrthoFromPcl, radius 1: Pa = 6, 268 columns, kj_per = 2
    ("stripe", 7, 7),
    ("adaptive_stripe", 7, 7),
]


@pytest.mark.parametrize("name,s_req,s_exp", WINDOW_CASES)
def test_destination_count_changes_no_bin_and_no_output_bit(name, s_req, s_exp, tmp_path):
    sc = make_scene(name)
    layer, dbg, bins = run_scene(sc)                      # this process: the default window, one destination
    assert bins["S"] == 1
    check_against_oracle(sc, layer, dbg)
    n = len(sc["xyz"])
    exp = expected_layout(sc, n, whole_map=sc["adaptive"] and sc["col_range"] is not None)
    assert destinations(n, exp["KC"], window_for(n, s_req))[0] == s_exp
    S, layers = run_in_child(name, window_for(n, s_req), tmp_path)
    assert S == [s_exp], "the partition used %s destinations, the case needs %d" % (S, s_exp)
    assert bits_equal(layers[0], layer), "the output depends on the number of destinations"


# ---- 2. partition-tile edges and skewed clouds (one destination) ---------------------------------------------------
TILE_EDGES = [1, 2047, 2048, 2049, 4 * 2048 - 1, 32 * 2048 + 1]


@pytest.mark.parametrize("n", TILE_EDGES)
def test_partition_tile_edges(n):
    sc = make_scene("n=%d" % n)
    layer, dbg, bins = run_scene(sc)
    check_against_oracle(sc, layer, dbg)


SKEWED = ["one_bucket", "first", "last", "mod", "descending_column", "tile_outside", "non_finite", "edges", "ids",
          "intensity", "adaptive", "stripe", "adaptive_stripe"]


@pytest.mark.parametrize("name", SKEWED)
def test_skewed_clouds_and_sources(name):
    sc = make_scene(name)
    layer, dbg, bins = run_scene(sc)
    check_against_oracle(sc, layer, dbg)
    if name == "tile_outside":
        assert bins["n_binned"] <= 2 * TILE
    if name == "one_bucket":
        assert np.count_nonzero(np.diff(bins["G"].astype(np.int64))) == 1
    if name in ("first", "last", "mod"):    # the bucket columns the cloud fills: those of 1 or of all 7 destinations
        used = np.flatnonzero(np.diff(bins["G"].astype(np.int64)).reshape(bins["KC"], bins["KR"]).sum(axis=1))
        dest = np.unique(used // 42)
        assert list(dest) == {"first": [0], "last": [6], "mod": list(range(7))}[name]
    if name == "ids":
        assert (bins["rec"][:, 3].copy().view(np.uint64) & np.uint64(0xffffffff)).max() == 2 ** 32 - 1


@pytest.mark.parametrize("res", [0.25, 0.1, 0.3])
@pytest.mark.parametrize("where", ["utm", "local"])
def test_fine_bin_ties(res, where):
    sc = make_scene("ties_%s_%s" % (res, where))
    if res != 0.25 and where == "local":
        assert sc["fma_differs"] > 0      # the scene holds columns where an un-fused evaluation floors differently
    layer, dbg, bins = run_scene(sc)
    check_against_oracle(sc, layer, dbg)


@pytest.mark.skipif(EMULATED, reason="1.2 M points: minutes on the emulated kernels")
def test_blocks_that_loop_over_several_tiles():
    # more than 4 * num_sms * 2048 points (1.08 M on an H100): a P1 block takes several tiles, with no barrier at the
    # end of a tile
    sc = scene(120, 250, 0.16, uniform(1_200_000, 19, rows=120), hint=None)
    layer, dbg, bins = run_scene(sc)
    assert bins["n_binned"] > 1_100_000
    check_against_oracle(sc, layer, dbg)


# ---- 3. a sharded cloud with border halos, one device -------------------------------------------------------------
def test_sharded_stripes_with_halo_slots():
    import torch
    from aerial_mapper_b200 import sharding
    # three stripe contexts, each binning [all ranks' halo slots (its own and the unused ones NaN) | its own points] as
    # test_gpu_dsm.py simulates the all-gather; no count is a whole number of tiles
    rows, cols, res, world = A["rows"], A["cols"], A["res"], 3
    xyz_np = uniform(15001, 21, holes=2)
    full, _, _ = run_scene(scene(rows, cols, res, xyz_np, hint=None))
    dev = torch.device("cpu" if EMULATED else "cuda:0")
    device_sync = (lambda: None) if EMULATED else torch.cuda.synchronize
    xyz = torch.from_numpy(xyz_np).to(dev)
    ids = torch.arange(xyz.shape[0], dtype=torch.int64, device=dev) * 5 + 7   # not positions, same order
    ranks = []
    for r in range(world):
        c0, c1 = sharding.stripe_range(cols, r, world)
        sc = scene(rows, cols, res, np.zeros((0, 3)), col_range=(c0, c1), hint=len(xyz_np) / float(rows * cols))
        gm = grid_map(sc)
        y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
        m = sharding.owner_mask(xyz[:, 1], y_lo, y_hi, r, world)
        hx = sharding.HaloExchange(torch, world, r, 8000, xyz[m], ids[m], dev)
        hx.extract(gm.context(), y_lo, y_hi, amb.lib().amb_dsm_halo_reach(C.byref(gm.geometry), 1))
        ranks.append((sc, gm, hx))
    device_sync()
    for _, gm, _ in ranks:
        gm.sync()
    gathered = torch.stack([hx.send for _, _, hx in ranks])
    device_sync()
    for sc, gm, hx in ranks:
        hx.gathered.copy_(gathered)
        device_sync()
        assert (hx.counts() <= hx.cap).all() and (hx.counts() > 0).all()
        hx.assemble()
        device_sync()
        assert hx.n_local % TILE != 0 and hx.n_total % TILE != 0
        sc["xyz"] = hx.big_xyz.cpu().numpy()
        sc["ids"] = hx.big_ids.cpu().numpy().view(np.uint64)
        layer, _, bins = run_scene(sc, gm)
        assert bins["n_binned"] > hx.n_local                # the halos are binned too
        c0, c1 = sc["col_range"]
        assert bits_equal(layer, full[:, c0:c1])


# ---- 4. context reuse ----------------------------------------------------------------------------------------------
REUSE_WINDOW = 40 * TILE * 32 // 8      # 40 tiles -> S = 8


def reuse_sequence():
    """One context: a 40-tile call with S = 8, a 1-tile call with S = 1, then a 10-tile one; the buffers only grow, so
    the later calls run over stale records and a stale offset table of another stride."""
    out = []
    gm = None
    for n, seed in ((40 * TILE, 31), (TILE, 32), (10 * TILE + 5, 33)):
        sc = scene(A["rows"], A["cols"], A["res"], uniform(n, seed), hint=None)
        gm = gm or grid_map(sc)
        layer, _, bins = run_scene(sc, gm)
        out.append((layer, bins["S"]))
    return out


def test_context_reuse_with_shrinking_calls(tmp_path):
    S, layers = run_in_child("reuse", REUSE_WINDOW, tmp_path)
    assert S == [8, 1, 3]
    for (n, seed), got in zip(((40 * TILE, 31), (TILE, 32), (10 * TILE + 5, 33)), layers):
        sc = scene(A["rows"], A["cols"], A["res"], uniform(n, seed), hint=None)
        fresh, dbg, _ = run_scene(sc)
        assert bits_equal(got, fresh)
        check_against_oracle(sc, fresh, dbg)


def test_download_bins_before_any_binning_is_an_error():
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 8.0, 8.0, 1.0)).getMutable()
    lay = np.zeros(LAYOUT, np.int32)
    assert amb.lib().amb_dsm_download_bins(gm.context(), lay.ctypes.data, None, None, None) == amb._lib.AMB_ERR_INVALID_ARGUMENT


if __name__ == "__main__":      # child process of run_in_child (AMB_DSM_PART_WINDOW set)
    sys.path.insert(0, ROOT)
    import conftest  # noqa: F401  (AMB_TEST_EMU=1: the emulated library, as in the parent)
    child_main(sys.argv[1], sys.argv[2])
