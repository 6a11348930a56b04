"""Shared helpers of the test suite."""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from aerial_mapper_b200 import synth  # noqa: E402  (pure numpy: scene and input generators)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def ulp_diff(a, b):
    """Distance in float32 units-in-the-last-place between two float32 arrays (NaN==NaN counts as 0)."""
    a = np.ascontiguousarray(a, dtype=np.float32).ravel()
    b = np.ascontiguousarray(b, dtype=np.float32).ravel()
    both_nan = np.isnan(a) & np.isnan(b)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[both_nan] = 0
    return d


REFERENCE_OUTPUTS = os.path.join(GOLDEN, "reference_outputs.json")


def _bits(a):
    a = np.asarray(a)
    return np.ascontiguousarray(a.reshape(-1, order="F")).view(np.uint32 if a.itemsize == 4 else np.uint64)


def _digest(a):
    import hashlib
    return hashlib.sha256(_bits(a).tobytes()).hexdigest()


def _current_case():
    # "tests/test_x.py::test_y[params] (call)" -> "test_x.py::test_y[params]" (the same from any working directory)
    node = os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0]
    return os.path.basename(node)


def reference_outputs(oracle, refsrc=None, suffix=""):
    """What the reference's own sources (aerial_mapper's dsm.cc, ortho-backward-grid.cc, ...) output for the current test
    case: a dict name -> array, like `oracle`, which holds the same case evaluated by the in-repo oracle (oracle/).

    Where the reference build exists (oracle/_ref) `refsrc()` computes the outputs.  Elsewhere they are restored from
    tests/golden/reference_outputs.json: the record of the reference's run lists the few elements in which its output
    differs from the oracle's (summation order) and the SHA-256 of every output array, and a restored array is accepted
    only if its digest matches — so the comparison is always against the reference's own output, bit for bit.
    AMB_RECORD_REFERENCE=<file>: add the records of the cases run to <file> (a copy of reference_outputs.json)."""
    import json
    key = _current_case() + suffix
    record_to = os.environ.get("AMB_RECORD_REFERENCE")
    src = record_to if record_to and os.path.exists(record_to) else REFERENCE_OUTPUTS
    records = {}
    if os.path.exists(src):
        with open(src) as f:
            records = json.load(f)
    if refsrc is not None and _have_refsrc():
        ref = refsrc()
        rec = {}
        for name, a in ref.items():
            diff = np.nonzero(_bits(a) != _bits(oracle[name]))[0]
            rec[name] = {"sha256": _digest(a), "index": diff.tolist(), "bits": _bits(a)[diff].tolist()}
        if record_to:
            records[key] = rec
            with open(record_to, "w") as f:
                json.dump(records, f, indent=0, sort_keys=True)
        elif key in records:
            assert records[key] == rec, "%s: the reference's output differs from its record" % key
        return ref
    assert key in records, "no recorded reference output for %s (tests/golden/reference_outputs.json)" % key
    out = {}
    for name, r in records[key].items():
        a = np.array(oracle[name], copy=True, order="F")
        flat = _bits(a).copy()
        flat[np.asarray(r["index"], np.int64)] = np.asarray(r["bits"], flat.dtype)
        a = flat.view(a.dtype).reshape(a.shape, order="F")
        assert _digest(a) == r["sha256"], "%s/%s: the oracle no longer reproduces the reference's record" % (key, name)
        out[name] = np.asfortranarray(a)
    return out


def _have_refsrc():
    from oracle import pyoracle as po
    return po.have_refsrc()


def fresh_layers(rows, cols, elevation=None):
    """AerialGridMap::initialize values (aerial-mapper-grid-map.cc:40-48) as float32 F-order arrays."""
    L = {"elevation": np.full((rows, cols), np.nan, np.float32, order="F"),
         "elevation_angle": np.zeros((rows, cols), np.float32, order="F"),
         "observation_index": np.full((rows, cols), np.nan, np.float32, order="F"),
         "ortho": np.full((rows, cols), 255.0, np.float32, order="F"),
         "colored_ortho": np.full((rows, cols), np.nan, np.float32, order="F")}
    if elevation is not None:
        L["elevation"][...] = elevation
    return L


def dsm_thresholds_py(radius):
    """The retry thresholds of dsm.cc:133-144 (lambda *= 1.1 accumulated in double, stop once lambda * r > 7),
    evaluated independently of the library."""
    thr, lam = [], 1.0
    while True:
        thr.append(lam * radius)
        lam *= 1.1
        if lam * radius > 7.0:
            return thr


def fma(a, b, c):
    """Correctly rounded a * b + c (what the device's fma computes), via exact rationals."""
    from fractions import Fraction
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def shifted_d2(qx, qy, x, y, ce=0.0, cn=0.0):
    """The reference's squared distance from cell centre (qx, qy) to raw point (x, y): the point is shifted first
    (dsm.cc:42-43: x - center_northing, y - center_easting), then 0 + dx*dx + dy*dy un-fused (nanoflann L2_Adaptor).
    numpy element-wise double arithmetic rounds every operation like the reference."""
    px = np.asarray(x, np.float64) - cn
    py = np.asarray(y, np.float64) - ce
    dx = qx - px
    dy = qy - py
    return dx * dx + dy * dy


def points_at_distance(qx, qy, thr, angle, ce=0.0, cn=0.0, xs=2048, span=24):
    """Raw points (x, y) around cell centre (qx, qy) whose shifted_d2 is just below, exactly at and just above `thr`.

    Starts from the point at distance sqrt(thr) in direction `angle`, walks x over adjacent doubles and, for each x,
    y over the doubles next to the solution of d2 == thr.  Returns {"lo": .., "eq": .., "hi": ..}, each (x, y, d2) or
    None: "eq" has d2 == thr; "lo" the largest d2 < thr found, "hi" the smallest d2 > thr found.  Near the origin these
    are thr's neighbouring doubles; at map-scale coordinates (steps of ~1e-9 m) they are the nearest attainable."""
    r = np.sqrt(thr)
    x0 = (qx - r * np.cos(angle)) + cn
    y0 = (qy - r * np.sin(angle)) + ce
    # steps of at least one ulp of 1.0: near a zero coordinate a step of its own ulp would not move d2 at all
    sx, sy = np.spacing(max(abs(x0), 1.0)), np.spacing(max(abs(y0), 1.0))
    X = x0 + np.arange(-xs, xs + 1) * sx
    dx = qx - (X - cn)
    rem = np.maximum(thr - dx * dx, 0.0)
    sign = 1.0 if np.sin(angle) >= 0 else -1.0
    Yc = (qy - sign * np.sqrt(rem)) + ce
    Y = Yc[:, None] + np.arange(-span, span + 1)[None, :] * sy
    Y = np.concatenate([Y, np.full((len(X), 1), qy + ce)], axis=1)     # dy = 0: the axis directions
    XX = np.broadcast_to(X[:, None], Y.shape)
    D = shifted_d2(qx, qy, XX, Y, ce, cn)
    out = {}
    eq = np.argwhere(D == thr)
    out["eq"] = (XX[tuple(eq[0])], Y[tuple(eq[0])], thr) if len(eq) else None
    below = np.where(D < thr, D, -np.inf)
    k = np.unravel_index(np.argmax(below), D.shape)
    out["lo"] = (XX[k], Y[k], D[k]) if np.isfinite(below[k]) else None
    above = np.where(D > thr, D, np.inf)
    k = np.unravel_index(np.argmin(above), D.shape)
    out["hi"] = (XX[k], Y[k], D[k]) if np.isfinite(above[k]) else None
    return out


def grid_base(rows, cols, res, pos=(0.0, 0.0)):
    """Centre of cell (0, 0) and 1/res as the library's plan computes them (grid_map getPosition)."""
    return (pos[0] + (0.5 * (rows * res) - 0.5 * res), pos[1] + (0.5 * (cols * res) - 0.5 * res), 1.0 / res)


def cell_of(base, p, inv_res):
    """Cell index whose centre is nearest to shifted coordinate p, by the binning's floor(fma(base - p, 1/res, 0.5))."""
    import math
    return int(math.floor(fma(base - p, inv_res, 0.5)))


def brute_dsm(rows, cols, res, xyz, radius=1, ce=0.0, cn=0.0, pos=(0.0, 0.0)):
    """Independent O(cells x points) numpy evaluation of the DSM definition (tiny inputs only).
    numpy element-wise double arithmetic is un-fused, i.e. rounds like the reference's."""
    from aerial_mapper_b200 import synth
    qx, qy = synth.grid_positions(rows, cols, res, pos[0], pos[1])
    px = xyz[:, 0] - cn
    py = xyz[:, 1] - ce
    pz = xyz[:, 2]
    thr = []
    lam = 1.0
    while True:
        thr.append(lam * radius)
        lam *= 1.1
        if lam * radius > 7.0:
            break
    elev = np.full((rows, cols), np.nan, np.float32, order="F")
    cnt = np.zeros((rows, cols), np.int32, order="F")
    lvl = np.full((rows, cols), -1, np.int8, order="F")
    for j in range(cols):
        dy2 = (qy[j] - py) * (qy[j] - py)
        for i in range(rows):
            dx = qx[i] - px
            d2 = dx * dx + dy2
            for k, t in enumerate(thr):
                m = d2 < t
                if m.any():
                    w = 1.0 / d2[m]
                    num = np.sum(pz[m] / d2[m])
                    elev[i, j] = np.float32(num / np.sum(w))
                    cnt[i, j] = int(m.sum())
                    lvl[i, j] = k
                    break
    return elev, cnt, lvl


# ---- probe scenes of the DSM / OrthoFromPcl decision tests (tests/test_gpu_dsm_adversarial.py) -------------------
KINDS = ("lo", "eq", "hi")
UTM = (4.6e5 + 123.0, 5.2e6 + 457.0)          # a map position in UTM metres (easting, northing)
UTM_SHIFT = (3.1e5 + 77.25, 4.9e6 + 31.5)      # center_easting, center_northing of the same magnitude


def Z(t):
    # heights: distinct per point (a wrong neighbour set moves a cell by ~0.1 m) within one metre, so that the FP32
    # gather's height rounding (relative to the tile's height range; not the subject here) stays inside MAX_ULP
    return 100.0 + ((0.37 * t) % 1.0)


class Scene(object):
    def __init__(self, rows, cols, res, radius=1, pos=(0.0, 0.0), ce=0.0, cn=0.0):
        self.rows, self.cols, self.res, self.radius = rows, cols, res, radius
        self.pos, self.ce, self.cn = pos, ce, cn
        self.qx, self.qy = synth.grid_positions(rows, cols, res, pos[0], pos[1])
        self.pts = []
        self.probes = []     # (i, j, level, count) the strict `<` implies

    def add(self, x, y, z):
        self.pts.append((x, y, z))

    @property
    def xyz(self):
        return np.array(self.pts, np.float64).reshape(-1, 3)

    def expect(self, i, j, level, count):
        self.probes.append((i, j, level, count))

    def raw(self, px, py):
        # raw point of shifted coordinates (px, py); callers re-evaluate d2 on what the shift gives back
        return px + self.cn, py + self.ce


def probe_spacing(res):
    # more than 2 * sqrt(7) m (two largest balls) plus a cell between probe centres
    return int(math.ceil((2.0 * math.sqrt(7.0) + res + 0.05) / res))


def probe_cells(n, res, min_cols=0):
    S = probe_spacing(res)
    per = int(math.ceil(math.sqrt(n)))
    cols = max(per * S, min_cols)
    rows = int(math.ceil(n / float(per))) * S
    return rows, cols, [(S // 2 + S * (t // per), S // 2 + S * (t % per)) for t in range(n)]


def expected_level(d2, thr):
    for k, t in enumerate(thr):
        if d2 < t:
            return k
    return -1


def tie_scene(radius, res, levels=None, pos=(0.0, 0.0), ce=0.0, cn=0.0, require_exact=True):
    """Case 1: for each retry level k a probe whose only point is at d2 = thr_k^-, thr_k, thr_k^+, and one probe with
    three points at thr_0^-, thr_0, thr_0^+ (exactly one neighbour)."""
    thr = dsm_thresholds_py(radius)
    levels = list(range(len(thr))) if levels is None else levels
    n = 3 * len(levels) + 1
    rows, cols, cells = probe_cells(n, res, min_cols=40)
    sc = Scene(rows, cols, res, radius, pos, ce, cn)
    t = 0
    for k in levels:
        for kind in KINDS:
            i, j = cells[t]
            want = thr[k] if kind == "eq" else np.nextafter(thr[k], -np.inf if kind == "lo" else np.inf)
            for attempt in range(8):         # a different direction (and bin geometry) for every probe
                c = points_at_distance(sc.qx[i], sc.qy[j], thr[k], 0.37 + 0.61 * t + 0.29 * attempt, ce, cn)[kind]
                if c is not None and (c[2] == want or not require_exact):
                    break
            if c is None and not require_exact:      # map scale: an exact tie is rarely attainable
                t += 1
                continue
            assert c is not None and (c[2] == want or not require_exact), (k, kind)
            sc.add(c[0], c[1], Z(t))
            d2 = float(shifted_d2(sc.qx[i], sc.qy[j], c[0], c[1], ce, cn))
            lvl = expected_level(d2, thr)
            sc.expect(i, j, lvl, 1 if lvl >= 0 else 0)
            t += 1
    i, j = cells[t]
    for u, kind in enumerate(KINDS):
        c = points_at_distance(sc.qx[i], sc.qy[j], thr[0], 1.1 + 2.0 * u, ce, cn)[kind]
        if c is None and not require_exact:
            continue
        assert c is not None and (kind == "eq") == (c[2] == thr[0]) and (kind == "lo") == (c[2] < thr[0])
        sc.add(c[0], c[1], Z(100 + u))
    sc.expect(i, j, 0, 1)
    return sc


def reach_scene(radius, res, pos=(0.0, 0.0), ce=0.0, cn=0.0):
    """Case 2: points just inside the primary ball and the largest retry ball, in 24 directions (the axis directions
    put them in the last bin row / column the windows keep), around isolated probe cells."""
    thr = dsm_thresholds_py(radius)
    rows, cols, cells = probe_cells(2, res, min_cols=40)
    sc = Scene(rows, cols, res, radius, pos, ce, cn)
    for (i, j), k in zip(cells, (0, len(thr) - 1)):
        for a in range(24):
            c = points_at_distance(sc.qx[i], sc.qy[j], thr[k], a * math.pi / 12, ce, cn)["lo"]
            sc.add(c[0], c[1], Z(a))
        sc.expect(i, j, k, 24)
    return sc


def last_window_row_hits(sc):
    """Points of the scene inside the primary ball of a probe cell AND binned W cells away from it along j or i —
    the last bin row half_widths() keeps."""
    W = int(math.floor(math.sqrt(sc.radius) / sc.res + 0.5 + 1e-6))
    bx, by, inv = grid_base(sc.rows, sc.cols, sc.res, sc.pos)
    n = 0
    for (i, j, _, _) in sc.probes:
        for (x, y, _) in sc.pts:
            d2 = float(shifted_d2(sc.qx[i], sc.qy[j], x, y, sc.ce, sc.cn))
            if d2 < sc.radius:
                ci, cj = cell_of(bx, x - sc.cn, inv), cell_of(by, y - sc.ce, inv)
                n += abs(cj - j) == W or abs(ci - i) == W
    return n


def bin_edge_scene(res, pos=(0.0, 0.0), ce=0.0, cn=0.0, rows=72, cols=72):
    """Case 3: points whose binning coordinate (base - p)/res + 0.5 is an integer on both axes (cell corners), and the
    neighbouring doubles, at tile edges (cells 31/32, 63/64) and elsewhere; plus a sparse background."""
    sc = Scene(rows, cols, res, 1, pos, ce, cn)
    bx, by, inv = grid_base(rows, cols, res, pos)
    rng = np.random.default_rng(31)
    corners = [(31, 31), (31, 63), (63, 31), (10, 45), (44, 17), (63, 63), (5, 5)]
    placed = 0
    for (i, j) in corners:
        # corner between cells (i, j), (i + 1, j), (i, j + 1), (i + 1, j + 1): centre minus half a cell on both axes
        px0, py0 = sc.qx[i] - 0.5 * res, sc.qy[j] - 0.5 * res
        for di in (-1, 0, 1):
            for dj in (-1, 0, 1):
                px = px0 + di * np.spacing(abs(px0))
                py = py0 + dj * np.spacing(abs(py0))
                x, y = sc.raw(px, py)
                sc.add(x, y, Z(rng.integers(0, 1000)))
                placed += (fma_is_integer(bx, x - cn, inv) and fma_is_integer(by, y - ce, inv))
    if res * 4 == int(res * 4):
        assert placed >= 1       # a dyadic resolution: some points lie exactly on a bin edge on both axes
    n_bg = int(rows * cols * res * res * 0.8)
    bg = np.c_[rng.uniform(sc.qx[-1], sc.qx[0], n_bg) + cn, rng.uniform(sc.qy[-1], sc.qy[0], n_bg) + ce,
               rng.uniform(100.0, 101.0, n_bg)]
    for p in bg:
        sc.add(*p)
    return sc


def fma_is_integer(base, p, inv_res):
    v = fma(base - p, inv_res, 0.5)
    return v == math.floor(v)


def apron_scene(res, radius=1):
    """Case 4: no point inside the map; points just inside sqrt(thr_k) beyond the outer cells (edge cells resolve only
    at retry level k), and one point just beyond / just inside the bin grid's apron."""
    thr = dsm_thresholds_py(radius)
    rows, cols = 40, 48
    sc = Scene(rows, cols, res, radius)
    edge = [(0, 5), (rows - 1, 20), (12, 0), (25, cols - 1), (0, 0), (rows - 1, cols - 1)]
    dirs = [(-1, 0), (1, 0), (0, -1), (0, 1), (-1, -1), (1, 1)]
    ks = [len(thr) - 1, len(thr) // 2, 3, len(thr) - 2, 1, len(thr) - 1]
    for (i, j), (si, sj), k in zip(edge, dirs, ks):
        # outward from the map: +x is towards smaller i (qx decreases with i)
        angle = math.atan2(sj, si)
        c = points_at_distance(sc.qx[i], sc.qy[j], thr[k], angle)["lo"]
        sc.add(c[0], c[1], Z(k))
        sc.expect(i, j, expected_level(c[2], thr), 1)
    return sc


def eps_f(res, radius):
    """The FP32 gather's guard band (dsm_run): bound on |d2_f32 - d2| with a safety factor 2."""
    W = int(math.floor(math.sqrt(radius) / res + 0.5 + 1e-6))
    u = 2.0 ** -24
    M = (16 + W + 2) * res
    t = radius * 1.01
    bound = 2.0 * math.sqrt(2.0 * t) * (2.0 * u * M + u * math.sqrt(t)) + 3.0 * u * t
    return float(np.float32(2.0 * bound))


def band_scene(res=0.5):
    """Level-0 probes, each with one point well inside the ball and one at d2 = thr_0 -+ delta, delta from 1/64 to 32
    guard bands, plus exact ties: which cells the FP32 gather must hand to the exact kernel is known."""
    eps = eps_f(res, 1)
    deltas = [eps / 64, eps / 8, eps / 4, 4 * eps, 8 * eps, 32 * eps]
    targets = [1.0 - d for d in deltas] + [1.0 + d for d in deltas]
    rows, cols, cells = probe_cells(len(targets) + 3, res, min_cols=40)
    sc = Scene(rows, cols, res, 1)
    for t, (i, j) in enumerate(cells):
        angle = 0.3 + 0.7 * t
        sc.add(sc.qx[i] - 0.3, sc.qy[j] + 0.2, Z(2 * t))              # d2 = 0.13: a level-0 hit in every probe
        if t < len(targets):
            c = points_at_distance(sc.qx[i], sc.qy[j], targets[t], angle)["eq" if t % 2 else "lo"]
        else:
            c = points_at_distance(sc.qx[i], sc.qy[j], 1.0, angle)[KINDS[t - len(targets)]]
        sc.add(c[0], c[1], Z(2 * t + 1))
        sc.expect(i, j, 0, 2 if c[2] < 1.0 else 1)
    return sc, eps



def coincident_scene(sizes=(2, 12, 30), seed=71):
    rows, cols, res = 64, 72, 0.5
    qx, qy = synth.grid_positions(rows, cols, res)
    rng = np.random.default_rng(seed)
    n_bg = 3000
    bg = np.c_[rng.uniform(-15, 15, n_bg), rng.uniform(-17, 17, n_bg), np.zeros(n_bg)]
    cells = [(10, 12), (33, 40), (50, 61), (20, 55)][:len(sizes)]
    parts = [bg]
    for (i, j), k in zip(cells, sizes):
        parts.append(np.tile([qx[i], qy[j], 0.0], (k, 1)))
    xyz = np.vstack(parts)
    perm = rng.permutation(len(xyz))          # cluster members get scattered ids
    xyz = xyz[perm]
    inten = rng.integers(0, 256, len(xyz)).astype(np.int32)
    for m in coincident_members(xyz, qx, qy, cells):
        inten[m] = rng.choice(256, len(m), replace=False)      # distinct intensities inside a cluster
    return rows, cols, res, xyz, inten, cells


def coincident_members(xyz, qx, qy, cells):
    return [np.nonzero((xyz[:, 0] == qx[i]) & (xyz[:, 1] == qy[j]))[0] for (i, j) in cells]
