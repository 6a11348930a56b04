"""The DSM's fine scatter runs band by band (a band = one coarse destination of the binning, a range of bucket columns) on
its own stream, and the gather of the tile columns over band d starts once band d is scattered (csrc/dsm_kernels.cu,
dsm_run).  Nothing but stream events orders the two, so:

* CPU: amb::dsm_scatter_band, which says which band a tile column's gather (reach W) and fill (reach P) wait for,
  against a brute-force list of every bucket start G and every bucket record those reads touch, and of the band whose
  scatter writes each of them last (after the scatter G[b] is bucket b - 1's cursor).  The function comes from the
  emulated library (tests/emu), called through a small C entry point the test compiles against it.
* GPU: one map binned into 1, 2, 7 and >= 100 bands (AMB_DSM_PART_WINDOW, which the library reads once per process: one
  child process per count and map): whole, in three column stripes given their border halos, and evaluated in column
  chunks with a host mirror.  Every layer equals the 1-band run bit for bit, and so does the number of cells the
  warp-per-cell kernel evaluated.
* GPU: two DSM calls in a row on one context, then OrthoFromPcl on the same context, enqueued back to back and binned
  into many bands: the results equal those of the same calls synchronised one by one, so every call finds the previous
  call's scatter finished.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from common import ROOT  # noqa: E402

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
TI = TJ = 32          # gather tile extents
MAX_COARSE = 256      # kMaxCoarse


# ---- CPU: the tile column -> band mapping -------------------------------------------------------------------------
def round_up(a, b):
    return (a + b - 1) // b * b


def bin_grid(rows, tile_j0, tile_j1, B, W, P, s_req):
    """The bin grid and bands dsm_run derives for a stripe of tile columns [tile_j0, tile_j1]."""
    Pa = round_up(P, B)
    gj0 = tile_j0 * TJ - Pa
    BR = round_up(round_up(rows, TI) + 2 * Pa, B)
    BC = round_up((tile_j1 + 1) * TJ + Pa - gj0, B)
    KR, KC = BR // B, BC // B
    S = max(1, min(s_req, MAX_COARSE, KC))
    kj_per = -(-KC // S)
    return dict(rows=rows, B=B, shift=B.bit_length() - 1, W=W, P=P, Pa=Pa, gj0=gj0, BR=BR, BC=BC, KR=KR, KC=KC,
                kj_per=kj_per, S=-(-KC // kj_per))


def writer_band(g, kind, p):
    """The band whose scatter writes G entry g (the cursor of bucket g - 1) or the records of bucket g last."""
    b = g - 1 if kind == "G" else g
    return -1 if b < 0 else (b // p["KR"]) // p["kj_per"]


def reads(p, tile, reach):
    """(G entries, buckets) the tile column's gather (reach W) or fill (reach P) reads, as contiguous index ranges."""
    KR, sh, Pa, BR, BC = p["KR"], p["shift"], p["Pa"], p["BR"], p["BC"]
    out = set()
    if reach == p["W"]:     # gather_tile / gather_tables: one window per tile, G at both ends of each bucket row
        W = p["W"]
        wj0 = tile * TJ - p["gj0"] - W
        kbj0, kbj1 = wj0 >> sh, min(wj0 + TJ + 2 * W - 1, BC - 1) >> sh
        for i0 in range(0, p["rows"], TI):
            wi0 = i0 + Pa - W
            kbi0, kbi1 = wi0 >> sh, min(wi0 + TI + 2 * W - 1, BR - 1) >> sh
            for kj in range(kbj0, kbj1 + 1):
                out.add(("G", kj * KR + kbi0, kj * KR + kbi0))
                out.add(("G", kj * KR + kbi1 + 1, kj * KR + kbi1 + 1))
                out.add(("rec", kj * KR + kbi0, kj * KR + kbi1))
        return out
    # the fill: bucket_window of every cell (dsm_mark_buckets_kernel, dsm_cell_kernel), and the ordering of each
    # flagged bucket b (dsm_bucket_order_kernel: G[b], G[b + 1] and its records)
    for i in range(p["rows"]):
        for j in range(tile * TJ, tile * TJ + TJ):
            bi, bj = i + Pa, j - p["gj0"]
            kbi0, kbi1 = max(bi - reach, 0) >> sh, min(bi + reach, BR - 1) >> sh
            kbj0, kbj1 = max(bj - reach, 0) >> sh, min(bj + reach, BC - 1) >> sh
            for kj in range(kbj0, kbj1 + 1):
                out.add(("G", kj * KR + kbi0, kj * KR + kbi1 + 1))
                out.add(("rec", kj * KR + kbi0, kj * KR + kbi1))
    return out


def needed_band(p, tile, reach):
    need = -1
    for kind, lo, hi in reads(p, tile, reach):
        for g in range(lo, hi + 1):
            need = max(need, writer_band(g, kind, p))
    return need


# amb::dsm_scatter_band as the product sources define it, from the emulated library (the CUDA sources compiled as plain
# C++, tests/emu/README.md), behind a C entry point that this test compiles next to it
PROBE = r"""
#include <cstring>
#include "amb_context.h"
#include "dsm_plan.h"
extern "C" int scatter_band(int bucket_shift, int BC, int gj0, int kj_per, int tile, int reach) {
  amb::dsmk::DsmPlan plan;
  std::memset(&plan, 0, sizeof(plan));
  plan.Bshift = bucket_shift;
  plan.B = 1 << bucket_shift;
  plan.BC = BC;
  plan.gj0 = gj0;
  return amb::dsm_scatter_band(plan, kj_per, tile, reach);
}
"""


@pytest.fixture(scope="module")
def scatter_band(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    emu = build_emu.build()
    d = tmp_path_factory.mktemp("band_probe")
    src, lib = str(d / "probe.cc"), str(d / "libband_probe.so")
    with open(src, "w") as f:
        f.write(PROBE)
    subprocess.check_call(["g++", "-std=c++17", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "tests", "emu", "include"),
                           "-I" + build_emu.CSRC, "-I" + os.path.join(ROOT, "include"), src, emu,
                           "-Wl,-rpath," + os.path.dirname(emu), "-o", lib])
    L = C.CDLL(lib)
    L.scatter_band.restype = C.c_int
    L.scatter_band.argtypes = [C.c_int] * 6
    return L.scatter_band


GRIDS = [  # rows, tile_j0, tile_j1, W, P
    # (the top tile row's window starts in bucket row 0, whose G entry is the previous column's last cursor, when
    # Pa - W < B: here for B >= 8 and for every B respectively)
    (40, 0, 9, 2, 5),      # a whole map
    (64, 3, 14, 4, 4),     # a stripe (tile_j0 > 0), P = W
    (33, 0, 5, 1, 9),      # P much larger than W: the fill reaches further bands than the gather
    (70, 2, 8, 8, 12),
]


@pytest.mark.parametrize("B", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("grid", GRIDS)
def test_tile_column_band_matches_the_reads(B, grid, scatter_band):
    rows, tj0, tj1, W, P = grid
    for s_req in (1, 2, 7, 256):
        p = bin_grid(rows, tj0, tj1, B, W, P, s_req)
        prev = {W: 0, P: 0}
        for tile in range(tj0, tj1 + 1):
            for reach in (W, P):
                got = scatter_band(p["shift"], p["BC"], p["gj0"], p["kj_per"], tile, reach)
                assert got == needed_band(p, tile, reach), (p, tile, reach)
                assert prev[reach] <= got < p["S"]          # one launch per run of tile columns, in band order
                prev[reach] = got
        # the fill of the last tile column waits for the last band: the join before the fill of an unchunked call
        last = scatter_band(p["shift"], p["BC"], p["gj0"], p["kj_per"], tj1, P)
        assert last == p["S"] - 1, p


# ---- GPU: bit-identical for every band count ----------------------------------------------------------------------
ROWS, COLS, RES, RADIUS = 64, 1200, 0.5, 1
STRIPES = 3
# one point per cell on average: 4-cell buckets, and 108 bucket columns in a 400-column stripe (up to 108 bands there,
# 154 on the whole map), so that the fill's reach P = 5 cells spans more than one band
N_POINTS = ROWS * COLS
HOLES = ((10, 200, 30, 260), (40, 395, 60, 410), (0, 790, 20, 815))   # rows, cols of empty rectangles: the retry path


def cloud(seed, n=N_POINTS):
    """Uniform points over the map, none in the HOLES (cell rectangles), heights a smooth surface plus noise."""
    rng = np.random.default_rng(seed)
    hx, hy = ROWS * RES / 2, COLS * RES / 2
    x = rng.uniform(-hx, hx, 2 * n)
    y = rng.uniform(-hy, hy, 2 * n)
    # cell (i, j) of a point: i = (hx - x) / res, j = (hy - y) / res (grid_map: index 0 at the max corner)
    i, j = (hx - x) / RES, (hy - y) / RES
    keep = np.ones(2 * n, bool)
    for i0, j0, i1, j1 in HOLES:
        keep &= ~((i >= i0) & (i < i1) & (j >= j0) & (j < j1))
    x, y = x[keep][:n], y[keep][:n]
    z = 100.0 + 3.0 * np.sin(0.05 * x) * np.cos(0.02 * y) + rng.normal(0.0, 0.05, n)
    return np.c_[x, y, z]


def window_for(n, S):
    """Bytes per band for which the binning asks for S bands: ceil(32 n / window) = S."""
    w = -(-(32 * n) // S)
    while -(-(32 * n) // w) > S:
        w += 1
    return w


def settings():
    import aerial_mapper_b200 as amb
    return amb.GridMapSettings(0.0, 0.0, ROWS * RES, COLS * RES, RES)


def stripe_input(gm, xyz, ids, c0, c1):
    """A stripe's own points and its border halos: every point within the halo reach of the stripe's y-interval."""
    import aerial_mapper_b200 as amb
    from aerial_mapper_b200 import sharding
    y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
    reach = amb.lib().amb_dsm_halo_reach(C.byref(gm.geometry), RADIUS)
    m = (xyz[:, 1] > y_lo - reach) & (xyz[:, 1] <= y_hi + reach)
    return np.ascontiguousarray(xyz[m]), np.ascontiguousarray(ids[m])


def run_case(case, s_req):
    """Elevation slab, bands and warp-per-cell cell count of `case` ("whole", "chunked" or "stripe<r>").  s_req > 1: the
    window is set for that many bands before the library's first binning in this process."""
    import aerial_mapper_b200 as amb
    from aerial_mapper_b200 import sharding
    xyz = cloud(7)
    ids = np.arange(len(xyz), dtype=np.uint64) * np.uint64(3) + np.uint64(11)
    col_range = None
    if case.startswith("stripe"):
        col_range = sharding.stripe_range(COLS, int(case[6:]), STRIPES)
    gm = amb.AerialGridMap(settings(), pinned=case == "chunked").getMutable()
    gm.to_device(0, col_range=col_range, names=("elevation",))
    ctx = gm.context()
    amb.check(amb.lib().amb_dsm_set_density_hint(ctx, len(xyz) / float(ROWS * COLS)), ctx)
    d = amb.Dsm(amb.DsmSettings(interpolation_radius=RADIUS), gm)
    d.stream_chunks = 1
    pts, pid = xyz, ids
    if col_range is not None:
        pts, pid = stripe_input(gm, xyz, ids, *col_range)
    if s_req > 1:
        os.environ["AMB_DSM_PART_WINDOW"] = str(window_for(len(pts), s_req))
    if case == "chunked":
        gm.set_mirrors(("elevation",))
        d.stream_chunks = 4
    d.process_sharded(pts, pid, gm, 0)
    gm.sync()
    layout = np.zeros(10, np.int32)
    amb.check(amb.lib().amb_dsm_download_bins(ctx, layout.ctypes.data, None, None, None), ctx)
    if case != "chunked":
        gm.download(("elevation",))
    c0, c1 = gm._col_range
    return gm["elevation"][:, c0:c1].copy(order="F"), int(layout[9]), int(gm.timings()["dsm_cells_empty"])


def run_sequence(sync_between):
    """Two DSM calls and an OrthoFromPcl call on one context, from device inputs: enqueued back to back with one sync at
    the end, or each synchronised before the next is enqueued."""
    import aerial_mapper_b200 as amb
    a, b = cloud(21), cloud(22, n=N_POINTS - 5000)
    inten = np.random.default_rng(23).integers(0, 255, len(b)).astype(np.int32)
    if EMULATED:    # the emulation's device memory is host memory
        dev = [a, b, inten]
        ptr = [v.ctypes.data for v in dev]
    else:
        import torch
        dev = [torch.from_numpy(v).to("cuda:0") for v in (a, b, inten)]
        ptr = [t.data_ptr() for t in dev]
    gm = amb.AerialGridMap(settings()).getMutable()
    gm.to_device(0, names=("elevation", "ortho"))
    d = amb.Dsm(amb.DsmSettings(interpolation_radius=RADIUS), gm)
    d.stream_chunks = 1
    o = amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=RADIUS))
    for call in (lambda: d.process_device(ptr[0], len(a), gm),
                 lambda: d.process_device(ptr[1], len(b), gm),
                 lambda: o.process_device(ptr[1], ptr[2], len(b), gm)):
        call()
        if sync_between:
            gm.sync()
    gm.sync()
    layout = np.zeros(10, np.int32)
    amb.check(amb.lib().amb_dsm_download_bins(gm.context(), layout.ctypes.data, None, None, None), gm.context())
    gm.download(("elevation", "ortho"))
    return gm["elevation"].copy(order="F"), gm["ortho"].copy(order="F"), int(layout[9])


def in_child(tmp_path, *args):
    out = str(tmp_path / ("_".join(args) + ".npz"))
    env = {k: v for k, v in os.environ.items() if k != "AMB_DSM_PART_WINDOW"}
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out] + list(args), cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    return np.load(out)


def bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


CASES = ["whole", "chunked"] + ["stripe%d" % r for r in range(STRIPES)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_every_band_count_gives_the_one_band_result(case, tmp_path):
    ref, s1, cells = run_case(case, 1)
    assert s1 == 1
    assert cells > 0                       # the holes reach the warp-per-cell kernel
    if case.startswith("stripe"):          # a stripe with its halos is the whole map's slab
        from aerial_mapper_b200 import sharding
        c0, c1 = sharding.stripe_range(COLS, int(case[6:]), STRIPES)
        whole, _, _ = run_case("whole", 1)
        assert bits_equal(ref, whole[:, c0:c1])
    for s_req in (2, 7, 256):
        z = in_child(tmp_path, "case", case, str(s_req))
        S = int(z["S"])
        assert S == s_req if s_req < 100 else S >= 100, (case, s_req, S)
        assert bits_equal(z["layer"], ref), "%s: %d bands change the elevation" % (case, S)
        assert int(z["cells"]) == cells, "%s: %d bands change the cells evaluated one by one" % (case, S)


@pytest.mark.gpu
def test_calls_in_a_row_on_one_context_find_the_scatter_done(tmp_path):
    z = in_child(tmp_path, "sequence", "256")
    assert int(z["S"]) >= 100
    elev, ortho, S = run_sequence(sync_between=True)
    assert S == 1
    assert bits_equal(z["elevation"], elev)
    assert bits_equal(z["ortho"], ortho)


if __name__ == "__main__":      # child process: out.npz, then "case" <case> <bands> or "sequence" <bands>
    sys.path.insert(0, ROOT)
    import conftest  # noqa: F401  (AMB_TEST_EMU=1: the emulated library, as in the parent)
    out, what, bands = sys.argv[1], sys.argv[2], int(sys.argv[-1])
    if what == "case":
        layer, S, cells = run_case(sys.argv[3], bands)
        np.savez(out, layer=layer, S=S, cells=cells)
    else:
        os.environ["AMB_DSM_PART_WINDOW"] = str(window_for(N_POINTS - 5000, bands))
        elev, ortho, S = run_sequence(sync_between=False)
        np.savez(out, elevation=elev, ortho=ortho, S=S)
