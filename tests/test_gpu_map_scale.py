"""Every map kernel at the map sizes the ABI admits: slabs past 2^31 cells, rows at the DSM's fine-bin limit, and the
largest slab below 2^32.

amb_create accepts a slab of up to 2^32 - 2 cells and dsm_run up to 2^27 - 1 rows, so cell lists, pixel indices and
cell offsets must hold indices up to there.  Method: a BIG context (the whole map) against a STRIPE context over a few
of its columns (amb_create(geom, dev, c0, c1)).  Stripes give the same bits as the undivided map (tiles align to global
columns; test_ortho_from_pcl_stripes.py, test_gpu_raster_*.py), and a stripe's indices are small, so a difference in a
window can only come from index width.  Both are compared on the device through amb_layer_device_ptr (multi-GB layers
never cross PCIe), and the window is also checked against the CPU oracle (pyoracle, int64 cell ranges) or the numpy
restatements of test_gpu_raster_export.py / test_gpu_raster_import.py.

Windows: the first two columns, the columns around cell index 2^31, around 2^32 - 2^20 where the map reaches it, and the
last two (a ragged last tile).  Shapes (resolution 5 cm):
    S1  46341 x 46341      2^31 + 4633 cells: cell 2^31 is (41708, 46340); ragged 32-cell tiles on both axes
    S2  (2^27 - 1) x 17    the DSM's row limit: fine bin rows past 2^27 after the apron; columns 16+ start past 2^31
    S3  65535 x 65536      2^32 - 65536 cells, the largest slab amb_create accepts (~17 GB per float32 layer)

Each case reads torch.cuda.mem_get_info() first and skips, naming the numbers, when the free device memory is short of
its estimate + 4 GiB; every context and buffer is freed before the next case.  Run with -s to see the time per case."""
import ctypes as C
import gc
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from common import ulp_diff  # noqa: E402
import test_gpu_raster_export as rexp  # noqa: E402
import test_gpu_raster_import as rimp  # noqa: E402

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(EMULATED, reason="the emulated kernels cannot hold maps of 2^31 cells and more")]

GiB = float(1 << 30)
RES = 0.05
S1, S2, S3 = (46341, 46341), ((1 << 27) - 1, 17), (65535, 65536)
SHAPES = {"S1": S1, "S2": S2, "S3": S3}
I31, I32M = 1 << 31, (1 << 32) - (1 << 20)
SHIFT = (3.1e5 + 77.25, 4.9e6 + 31.5)      # DSM centre shift on S1 (center_easting, center_northing): UTM-size raw points
F32, F64 = _lib.DSM_F32, _lib.DSM_F64
LAYER = _lib.LAYER_ID


# ---- contexts and device views --------------------------------------------------------------------------------------
def L():
    return _lib.lib()


def geometry(shape):
    rows, cols = shape
    return amb.Geometry(rows, cols, RES, rows * RES, cols * RES, 0.0, 0.0)


class _Cai(object):
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def device_view(ptr, n, dtype):
    """A torch CUDA tensor over n elements of device memory the library owns (no copy)."""
    import torch
    typestr = {torch.float32: "<f4", torch.int32: "<i4", torch.uint8: "|u1"}[dtype]
    return torch.as_tensor(_Cai(ptr, n, typestr), device="cuda")


class Ctx(object):
    def __init__(self, shape, c0=0, c1=None):
        self.g = geometry(shape)
        self.rows = shape[0]
        self.c0, self.c1 = c0, shape[1] if c1 is None else c1
        self.h = C.c_void_p()
        amb.check(L().amb_create(C.byref(self.g), 0, self.c0, self.c1, C.byref(self.h)))
        self.cells = self.rows * (self.c1 - self.c0)

    def check(self, st):
        amb.check(st, self.h)

    def sync(self):
        self.check(L().amb_sync(self.h))

    def ptr(self, layer):
        p = C.c_void_p()
        self.check(L().amb_layer_device_ptr(self.h, LAYER[layer], C.byref(p)))
        self.sync()      # a slab allocated here is born with its initial value, written on the context's stream
        return p.value

    def view(self, layer, dtype=None):
        import torch
        return device_view(self.ptr(layer), self.cells, dtype or torch.float32)

    def cols_of(self, layer, c0, c1):
        """Device view of global columns [c0, c1) of a layer (as int32 bits)."""
        import torch
        v = self.view(layer, torch.int32)
        return v[(c0 - self.c0) * self.rows:(c1 - self.c0) * self.rows]

    def close(self):
        if self.h:
            L().amb_destroy(self.h)
            self.h = None


@pytest.fixture
def res(request):
    """Contexts and device buffers of one case, all released at its end; prints the case's wall time."""
    import torch

    class R(object):
        ctxs = []

        def ctx(self, shape, c0=0, c1=None):
            c = Ctx(shape, c0, c1)
            self.ctxs.append(c)
            return c

    r = R()
    r.ctxs = []
    t0 = time.time()
    yield r
    for c in r.ctxs:
        c.close()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    print("\n[map scale] %s: %.1f s" % (request.node.name, time.time() - t0))


def need_device(gib, what):
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < (gib + 4.0) * GiB:
        pytest.skip("%s needs ~%.1f GiB of device memory + 4 GiB headroom; %.1f of %.1f GiB free"
                    % (what, gib, free / GiB, total / GiB))


def host_available_gib():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / float(1 << 20)
    return 0.0


def layer_gib(shape, bpc=4):
    return shape[0] * shape[1] * bpc / GiB


# ---- windows --------------------------------------------------------------------------------------------------------
def windows(shape):
    rows, cols = shape
    w = [(0, 2)]
    for idx in (I31, I32M):
        if rows * cols > idx:
            j = idx // rows
            w.append((max(j - 1, 0), min(j + 2, cols)))
    w.append((cols - 2, cols))
    w.sort()
    out = [list(w[0])]
    for a, b in w[1:]:
        if a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return [tuple(x) for x in out]


def assert_windows_reach(shape, wins):
    rows, cols = shape
    last = max(c1 for _, c1 in wins) * rows - 1
    assert last >= I31, "no compared cell has an index >= 2^31"
    if rows * cols > I32M:
        assert any(c0 * rows <= I32M < c1 * rows for c0, c1 in wins), "no compared cell near 2^32 - 2^20"


def oracle_ranges(shape, c0, c1, span=3000):
    """Cell ranges [lo, hi) of window [c0, c1) the oracle evaluates: the whole window, or on S2 (134 M cells per
    column) both ends of every column and the cells around 2^31."""
    rows = shape[0]
    lo, hi = c0 * rows, c1 * rows
    if hi - lo <= 300000:
        return [(lo, hi)]
    r = []
    for c in range(c0, c1):
        r += [(c * rows, c * rows + span), ((c + 1) * rows - span, (c + 1) * rows)]
    if lo <= I31 < hi:
        r.append((I31 - span, I31 + span))
    r.sort()
    out = [list(r[0])]
    for a, b in r[1:]:
        if a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return [tuple(x) for x in out]


def first_difference(a, b):
    import torch
    d = torch.nonzero(a != b)
    return "%d cells differ, first at window offsets %s" % (d.numel(), d[:4].flatten().tolist())


def assert_same_bits(big, stripe, what):
    import torch
    assert big.shape == stripe.shape
    assert torch.equal(big, stripe), "%s: %s" % (what, first_difference(big, stripe))


# ---- scenes -----------------------------------------------------------------------------------------------------------
def cell_centres(shape, i, j):
    rows, cols = shape
    bx = 0.5 * rows * RES - 0.5 * RES
    by = 0.5 * cols * RES - 0.5 * RES
    return bx - RES * np.asarray(i, np.float64), by - RES * np.asarray(j, np.float64)


def rect_points(rng, shape, i0, i1, j0, j1, density):
    """Uniform points over the cells [i0, i1) x [j0, j1) (may reach past the map by whole cells)."""
    n = int((i1 - i0) * (j1 - j0) * density)
    x_hi, y_hi = cell_centres(shape, i0 - 0.5, j0 - 0.5)
    x_lo, y_lo = cell_centres(shape, i1 - 0.5, j1 - 0.5)
    return np.c_[rng.uniform(x_lo, x_hi, n), rng.uniform(y_lo, y_hi, n)]


def scene(shape, seed, density=0.002):
    """Uniform background (`density` points per cell: a few million) plus, over every window: a sparse patch (gather path), a dense patch (tiles
    past the stage capacity go to the warp-per-cell kernel whole) and a hole (empty primary balls: the hand-over list and
    the retry levels), in rows at both ends of the columns and around cell 2^31.  Returns xy [n, 2] in map coordinates,
    heights z (terrain-like, within one metre: the FP32 gather's rounding stays within its ulp bar) and intensities."""
    rows, cols = shape
    rng = np.random.default_rng(seed)
    parts = [rect_points(rng, shape, 0, rows, 0, cols, density)]
    holes = []
    for c0, c1 in windows(shape):
        j0, j1 = max(c0 - 40, 0), min(c1 + 40, cols)
        row_bands = {0, rows - 600}
        for idx in (I31, I32M):
            if c0 * rows <= idx < c1 * rows:
                row_bands.add(min(max(idx % rows - 300, 0), rows - 600))
        for b in sorted(row_bands):
            parts.append(rect_points(rng, shape, b, b + 200, j0, j1, 0.06))
            parts.append(rect_points(rng, shape, b + 200, b + 400, j0, j1, 0.6))
            parts.append(rect_points(rng, shape, b + 400, b + 600, j0, j1, 0.06))
            holes.append((b + 60, b + 140, j0, j1))               # ~4 m across: retry levels up to the last
            holes.append((b + 450, b + 520, c0, c1))
    xy = np.vstack(parts)
    keep = np.ones(len(xy), bool)
    for i0, i1, j0, j1 in holes:
        x_hi, y_hi = cell_centres(shape, i0 - 0.5, j0 - 0.5)
        x_lo, y_lo = cell_centres(shape, i1 - 0.5, j1 - 0.5)
        keep &= ~((xy[:, 0] > x_lo) & (xy[:, 0] < x_hi) & (xy[:, 1] > y_lo) & (xy[:, 1] < y_hi))
    xy = xy[keep]
    z = 100.0 + 0.25 * np.sin(xy[:, 0] / 13.0) + 0.2 * np.cos(xy[:, 1] / 7.0) + rng.uniform(0.0, 0.3, len(xy))
    inten = rng.integers(0, 256, len(xy)).astype(np.int32)
    return xy, z, inten


def cell_rows_of(shape, x):
    bx = 0.5 * shape[0] * RES - 0.5 * RES
    return np.floor((bx - x) / RES + 0.5).astype(np.int64)


# ---- the oracle over cell ranges of a full-size (untouched, hence unallocated) host map ---------------------------------
def oracle_dsm(shape, xyz, ce, cn, ranges, debug):
    rows, cols = shape
    total = rows * cols
    g = po.make_geometry(rows, cols, RES)
    elev = np.empty(total, np.float32)      # only the pages of the ranges are ever touched
    cnt = np.empty(total, np.int32) if debug else None
    lvl = np.empty(total, np.int8) if debug else None
    out = []
    for lo, hi in ranges:
        elev[lo:hi] = np.nan
        if debug:
            cnt[lo:hi] = -1
            lvl[lo:hi] = -1
        st = po.lib().ambo_dsm_process(C.byref(g), elev.ctypes.data_as(C.c_void_p), xyz.ctypes.data_as(C.c_void_p),
                                       len(xyz), 1, ce, cn, 0, lo, hi, po._ptr(cnt), po._ptr(lvl), None)
        assert st == 0, st
        out.append((lo, hi, elev[lo:hi].copy(), cnt[lo:hi].copy() if debug else None,
                    lvl[lo:hi].copy() if debug else None))
    return out


def oracle_pcl(shape, xyz, inten, ranges, radius):
    rows, cols = shape
    g = po.make_geometry(rows, cols, RES)
    ortho = np.empty(rows * cols, np.float32)
    out = []
    for lo, hi in ranges:
        ortho[lo:hi] = 255.0
        st = po.lib().ambo_ortho_from_pcl_process(C.byref(g), ortho.ctypes.data_as(C.c_void_p),
                                                  xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p),
                                                  len(xyz), radius, 0, 0, lo, hi, None)
        assert st == 0, st
        out.append((lo, hi, ortho[lo:hi].copy()))
    return out


def download(view, lo, hi):
    return view[lo:hi].cpu().numpy()


# ---- 1. DSM -------------------------------------------------------------------------------------------------------------
_SCENES = {}


def dsm_scene(name):
    if name not in _SCENES:
        shape = SHAPES[name]
        xy, z, inten = scene(shape, seed={"S1": 1, "S2": 2, "S3": 3}[name])
        _SCENES.clear()
        _SCENES[name] = (xy, z, inten, {})
    return _SCENES[name]


def dsm_cloud(name):
    xy, z, inten, cache = dsm_scene(name)
    ce, cn = SHIFT if name == "S1" else (0.0, 0.0)
    xyz = np.ascontiguousarray(np.c_[xy[:, 0] + cn, xy[:, 1] + ce, z])
    return xyz, ce, cn, cache


def run_dsm(ctx, xyz, ce, cn, precision, debug):
    ctx.check(L().amb_dsm_set_precision(ctx.h, precision))
    ctx.check(L().amb_dsm_enable_debug(ctx.h, 1 if debug else 0))
    ctx.check(L().amb_dsm_process(ctx.h, xyz.ctypes.data_as(C.c_void_p), len(xyz), 1, ce, cn))
    ctx.sync()


def handed_over(ctx):
    """Cells the last DSM run handed to the warp-per-cell kernel (empty primary ball, dense tile, FP32 band or bound)."""
    t = _lib.Timings()
    ctx.check(L().amb_get_timings(ctx.h, C.byref(t)))
    return int(t.dsm_cells_empty)


def complement(cols, wins):
    out, c = [], 0
    for c0, c1 in wins:
        if c0 > c:
            out.append((c, c0))
        c = c1
    return out + ([(c, cols)] if c < cols else [])


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("name", ["S1", "S2", "S3"])
def test_dsm_big_context_equals_stripes_and_oracle(name, precision, res):
    import torch
    shape = SHAPES[name]
    rows, cols = shape
    prec = F32 if precision == "f32" else F64
    need_device(2 * layer_gib(shape) + 1.0, "DSM on %s" % name)   # elevation + hand-over list, bins
    xyz, ce, cn, cache = dsm_cloud(name)
    wins = windows(shape)
    assert_windows_reach(shape, wins)

    big = res.ctx(shape)
    # the big context's neighbour counts and levels too, where the host can take the whole slab's (~5 B per cell)
    big_debug = host_available_gib() > 3.0 * layer_gib(shape, 5) and \
        torch.cuda.mem_get_info()[0] > (3 * layer_gib(shape) + layer_gib(shape, 5) + 4.0) * GiB
    run_dsm(big, xyz, ce, cn, prec, big_debug)
    big_handed = handed_over(big)
    big_cnt = big_lvl = None
    if big_debug:
        big_cnt = np.empty(big.cells, np.int32)
        big_lvl = np.empty(big.cells, np.int8)
        big.check(L().amb_dsm_download_debug(big.h, big_cnt.ctypes.data_as(C.c_void_p),
                                             big_lvl.ctypes.data_as(C.c_void_p)))
    if name == "S2":
        # points whose fine bin row i + Pa (after the apron) lies past 2^27; the last window holds their rows
        layout = (C.c_int32 * 10)()
        big.check(L().amb_dsm_download_bins(big.h, layout, None, None, None))
        Pa = layout[1]
        i = cell_rows_of(shape, xyz[:, 0] - cn)
        assert (i >= (1 << 27) - 2 * Pa).any() and (i + Pa >= (1 << 27)).any(), Pa
        assert wins[-1][1] == cols and oracle_ranges(shape, *wins[-1])[-1][1] == rows * cols
    max_ulp = 4 if prec == F32 else 1
    handed = 0
    for c0, c1 in wins:
        st = res.ctx(shape, c0, c1)
        run_dsm(st, xyz, ce, cn, prec, True)
        assert handed_over(st) > 0, (name, c0, c1)
        handed += handed_over(st)
        assert_same_bits(big.cols_of("elevation", c0, c1), st.view("elevation", torch.int32),
                         "%s elevation, columns [%d, %d)" % (name, c0, c1))
        s_cnt = np.empty(st.cells, np.int32)
        s_lvl = np.empty(st.cells, np.int8)
        st.check(L().amb_dsm_download_debug(st.h, s_cnt.ctypes.data_as(C.c_void_p), s_lvl.ctypes.data_as(C.c_void_p)))
        if big_debug:
            lo, hi = c0 * rows, c1 * rows
            assert np.array_equal(big_cnt[lo:hi], s_cnt) and np.array_equal(big_lvl[lo:hi], s_lvl), (name, c0, c1)
        # the window against the oracle (cached per scene: the same for both precisions)
        key = (c0, c1)
        if key not in cache:
            cache[key] = oracle_dsm(shape, xyz, ce, cn, oracle_ranges(shape, c0, c1), True)
        s_elev = st.view("elevation")
        levels = set()
        for lo, hi, e, cnt, lvl in cache[key]:
            a, b = lo - c0 * rows, hi - c0 * rows
            got = download(s_elev, a, b)
            assert np.array_equal(np.isnan(got), np.isnan(e)), (name, lo, hi)
            assert ulp_diff(got, e).max() <= max_ulp, (name, lo, hi, int(ulp_diff(got, e).max()))
            assert np.array_equal(s_cnt[a:b], cnt), (name, lo, hi)
            assert np.array_equal(s_lvl[a:b], lvl), (name, lo, hi)
            levels |= set(np.unique(lvl).tolist())
        assert {0, 1, 2}.issubset(levels), (name, c0, c1, sorted(levels))   # the retry levels occur in the window
    # Which cells go to the warp-per-cell kernel is decided per cell and per tile (tiles align to global columns), so
    # stripes that partition the map hand over as many cells as the big run; the library reports the count per context
    # (amb_timings.dsm_cells_empty).  The windows' stripes are checked above; the rest of the map runs after the big
    # context is gone, one stripe at a time.
    big.close()
    for a, b in complement(cols, wins):
        rest = res.ctx(shape, a, b)
        run_dsm(rest, xyz, ce, cn, prec, False)
        handed += handed_over(rest)
        rest.close()
    assert handed == big_handed, (name, handed, big_handed)


# ---- 2. OrthoFromPcl --------------------------------------------------------------------------------------------------
def run_pcl(ctx, xyz, inten, adaptive):
    ctx.check(L().amb_ortho_from_pcl_process(ctx.h, xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p),
                                             len(xyz), 2, 1 if adaptive else 0))
    ctx.sync()


@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("name", ["S1", "S2"])
def test_ortho_from_pcl_big_context_equals_stripes(name, adaptive, res):
    import torch
    shape = SHAPES[name]
    rows, cols = shape
    # ortho + hand-over list (+ the adaptive pass's saved copy of the layer)
    need_device((3 if adaptive else 2) * layer_gib(shape) + 1.0, "OrthoFromPcl on %s" % name)
    xy, z, inten, cache = dsm_scene(name)
    xyz = np.ascontiguousarray(np.c_[xy, np.zeros(len(xy))])
    wins = windows(shape)
    assert_windows_reach(shape, wins)
    big = res.ctx(shape)
    run_pcl(big, xyz, inten, adaptive)
    for c0, c1 in wins:
        st = res.ctx(shape, c0, c1)
        run_pcl(st, xyz, inten, adaptive)
        assert_same_bits(big.cols_of("ortho", c0, c1), st.view("ortho", torch.int32),
                         "%s ortho, columns [%d, %d)" % (name, c0, c1))
        s_ortho = st.view("ortho")
        if adaptive:
            # the holes over the window left cells to the adaptive pass: every cell got a value, some not from the
            # primary ball (those the plain oracle leaves at 255 with no neighbour)
            assert not torch.isnan(s_ortho).any()
            continue
        key = ("pcl", c0, c1)
        if key not in cache:
            cache[key] = oracle_pcl(shape, xyz, inten, oracle_ranges(shape, c0, c1), 2)
        for lo, hi, o in cache[key]:
            got = download(s_ortho, lo - c0 * rows, hi - c0 * rows)
            assert ulp_diff(got, o).max() <= 1, (name, lo, hi)
    if adaptive:
        # the adaptive list held cells at indices >= 2^31: cells of the holes over the last columns differ from what the
        # plain pass leaves there (255)
        st = res.ctx(shape, wins[-1][0], wins[-1][1])
        run_pcl(st, xyz, inten, False)
        plain = st.view("ortho")
        adapt = big.cols_of("ortho", wins[-1][0], wins[-1][1]).view(torch.float32)
        changed = torch.nonzero(plain != adapt).flatten() + wins[-1][0] * rows
        assert changed.numel() > 0 and int(changed.max()) >= I31


# ---- 3. orthomosaic ----------------------------------------------------------------------------------------------------
# cells the frames look at: both ends of the first columns, and cell 2^31 and the rows after it in the last column
ORTHO_TARGETS = ((300, 0), (23000, 1), (S1[0] - 300, 0), (I31 % S1[0], S1[1] - 1), (S1[0] - 300, S1[1] - 1))


def ortho_frames(colored):
    """C3 frames (a quarter of the raster, the same field of view), three per target, 60 m above the terrain: footprints
    of ~80 x 60 m over every window."""
    from aerial_mapper_b200 import synth
    camd = synth.scaled_camera(0.25)
    poses = []
    for k, (i, j) in enumerate(ORTHO_TARGETS):
        x, y = cell_centres(S1, i, j)
        poses.append(synth.lawnmower_poses(1, 3, 12.0, 8.0, agl=60.0, seed=40 + k, center=(float(x), float(y))))
    poses = np.vstack(poses)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], 3 if colored else 1) for k in range(len(poses))]
    return camd, poses, imgs


def fill_elevation(view, first_cell, rows, chunk=1 << 25):
    """A terraced DEM around the frames' mean terrain (100 m), exact in float32: the same bits on the host."""
    import torch
    n = view.numel()
    for a in range(0, n, chunk):
        idx = torch.arange(first_cell + a, first_cell + min(a + chunk, n), dtype=torch.int64, device="cuda")
        view[a:a + idx.numel()] = elevation_of(idx % rows, idx // rows).to(torch.float32)
    torch.cuda.synchronize()


def elevation_of(i, j):
    return 100.0 + ((i // 64 + j // 64) % 16) * 0.5


def reset_ortho_layers(ctx, out):
    import torch
    ctx.view("elevation_angle").fill_(0.0)
    ctx.view("observation_index").fill_(float("nan"))
    ctx.view(out).fill_(float("nan") if out == "colored_ortho" else 255.0)
    torch.cuda.synchronize()


def run_ortho(ctx, cam, poses, imgs, d_imgs, colored, dominance):
    n = len(poses)
    ch = 3 if colored else 1
    row_step = imgs[0].shape[1] * ch
    ctx.check(L().amb_ortho_set_dominance_cull(ctx.h, 1 if dominance else 0))
    T = np.ascontiguousarray(poses)
    if d_imgs is None:
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        ctx.check(L().amb_ortho_process(ctx.h, C.byref(cam), T.ctypes.data_as(C.c_void_p), C.cast(ptrs, C.c_void_p), n,
                                        ch, row_step, 1 if colored else 0))
    else:
        ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in d_imgs])
        ctx.check(L().amb_ortho_process_device(ctx.h, C.byref(cam), T.ctypes.data_as(C.c_void_p),
                                               C.cast(ptrs, C.c_void_p), n, ch, row_step, 1 if colored else 0))
    ctx.sync()


def oracle_ortho(camd, poses, imgs, colored, ranges):
    rows, cols = S1
    g = po.make_geometry(rows, cols, RES)
    out = "colored_ortho" if colored else "ortho"
    layers = {k: np.empty((rows, cols), np.float32, order="F")      # only the pages of the ranges are touched
              for k in ("elevation", "elevation_angle", "observation_index", out)}
    flat = {k: a.reshape(-1, order="F") for k, a in layers.items()}
    res = []
    for lo, hi in ranges:
        idx = np.arange(lo, hi, dtype=np.int64)
        flat["elevation"][lo:hi] = elevation_of(idx % rows, idx // rows).astype(np.float32)
        flat["elevation_angle"][lo:hi] = 0.0
        flat["observation_index"][lo:hi] = np.nan
        flat[out][lo:hi] = np.nan if colored else 255.0
        st, _ = po.ortho_process(g, layers, po.make_camera(**camd), poses, imgs, colored=colored, cell_range=(lo, hi))
        assert st == 0, st
        res.append((lo, hi, {k: flat[k][lo:hi].copy() for k in ("elevation_angle", "observation_index", out)}))
    return res


@pytest.mark.parametrize("colored", [False, True])
def test_orthomosaic_big_context_equals_stripes_and_oracle(colored, res):
    """Resident and host frames (the host path adds the slab-sized `ortho_pix` buffer and ortho_texel_kernel), dominance
    cull on and off: every layer the orthomosaic writes, bit for bit between the big and the stripe contexts, and against
    the oracle (elevation_angle within 1 ulp)."""
    import torch
    shape = S1
    rows, cols = shape
    out = "colored_ortho" if colored else "ortho"
    need_device(5 * layer_gib(shape) + 1.0, "the orthomosaic on S1")   # four layers + the host path's pixel buffer
    wins = windows(shape)
    assert_windows_reach(shape, wins)
    camd, poses, imgs = ortho_frames(colored)
    cam = amb.NCamera(**camd).camera
    d_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    big = res.ctx(shape)
    fill_elevation(big.view("elevation"), 0, rows)
    stripes = []
    for c0, c1 in wins:
        st = res.ctx(shape, c0, c1)
        fill_elevation(st.view("elevation"), c0 * rows, rows)
        stripes.append(st)
    oracle = {w: oracle_ortho(camd, poses, imgs, colored, [(w[0] * rows, w[1] * rows)]) for w in wins}
    names = ("elevation_angle", "observation_index", out)
    for frames in ("resident", "host"):
        for dominance in (True, False):
            what = "%s frames, dominance cull %s" % (frames, "on" if dominance else "off")
            for ctx in [big] + stripes:
                reset_ortho_layers(ctx, out)
                run_ortho(ctx, cam, poses, imgs, d_imgs if frames == "resident" else None, colored, dominance)
            for (c0, c1), st in zip(wins, stripes):
                for name in names:
                    assert_same_bits(big.cols_of(name, c0, c1), st.view(name, torch.int32),
                                     "%s, %s, columns [%d, %d)" % (what, name, c0, c1))
                seen_past_2_31 = 0
                for lo, hi, want in oracle[(c0, c1)]:
                    a, b = lo - c0 * rows, hi - c0 * rows
                    got = {name: download(st.view(name), a, b) for name in names}
                    assert np.array_equal(got["observation_index"], want["observation_index"], equal_nan=True), what
                    assert np.array_equal(got[out].view(np.uint32), want[out].view(np.uint32)), what
                    assert ulp_diff(got["elevation_angle"], want["elevation_angle"]).max() <= 1, what
                    seen = ~np.isnan(got["observation_index"])
                    assert seen.sum() > 1000, (what, c0, c1)
                    seen_past_2_31 += int(seen[max(I31 - lo, 0):].sum()) if hi > I31 else 0
                if c1 * rows > I31:
                    assert seen_past_2_31 > 1000, what   # the frames cover cells at indices >= 2^31


# ---- 4. raster export --------------------------------------------------------------------------------------------------
def fill_pattern(view, first_cell, chunk=1 << 25):
    """Layer bits as a function of the GLOBAL cell index (the same in a big and a stripe context): mostly values in
    [-200, 824) on a 1/64 grid (gray ties and saturation), every 8th cell raw hashed bits (NaN payloads, denormals,
    infinities, packed colours)."""
    import torch
    bits = view.view(torch.int32)
    n = bits.numel()
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        idx = torch.arange(first_cell + a, first_cell + b, dtype=torch.int64, device="cuda")
        h = ((idx & 0xFFFFFFFF) * 1540483477 + (idx >> 32) * 97 + 12345) & 0xFFFFFFFF   # products < 2^63
        h = h ^ (h >> 15)
        h = (h * 668265261) & 0xFFFFFFFF
        h = h ^ (h >> 13)
        val = ((h >> 12) & 0xFFFF).to(torch.float32) / 64.0 - 200.0
        raw = torch.where(h >= (1 << 31), h - (1 << 32), h).to(torch.int32)
        bits[a:b] = torch.where((h & 7) == 0, raw, val.view(torch.int32))
    torch.cuda.synchronize()


def export_device(ctx, layer, fmt, dst_ptr):
    ctx.check(L().amb_export_raster_device(ctx.h, LAYER[layer], _lib.RASTER_FORMAT[fmt], C.c_void_p(dst_ptr)))
    ctx.sync()


@pytest.mark.parametrize("name", ["S1", "S3"])
def test_raster_export_windows_equal_stripes_and_restatement(name, res):
    import torch
    shape = SHAPES[name]
    rows, cols = shape
    need_device(2 * layer_gib(shape) + 0.5, "raster export on %s" % name)     # layer + F32 image
    wins = windows(shape)
    assert_windows_reach(shape, wins)
    big = res.ctx(shape)
    fill_pattern(big.view("ortho"), 0)
    img = torch.empty(big.cells * 4 + 32, dtype=torch.uint8, device="cuda")
    for fmt in rexp.FORMATS:
        bpp = _lib.RASTER_BPP[_lib.RASTER_FORMAT[fmt]]
        end = 1 + big.cells * bpp
        img[:16].fill_(rexp.CANARY)
        img[end:end + 16].fill_(rexp.CANARY)
        export_device(big, "ortho", fmt, img.data_ptr() + 1)      # an odd destination: the unaligned head and tail
        for c0, c1 in wins:
            st = res.ctx(shape, c0, c1)
            fill_pattern(st.view("ortho"), c0 * rows)
            band = torch.empty(st.cells * bpp, dtype=torch.uint8, device="cuda")
            export_device(st, "ortho", fmt, band.data_ptr())
            got = img[1 + c0 * rows * bpp:1 + c1 * rows * bpp]
            assert_same_bits(got, band, "%s %s image rows [%d, %d)" % (name, fmt, c0, c1))
            layer = st.view("ortho").cpu().numpy().reshape((rows, c1 - c0), order="F")
            want = rexp.restate(layer, fmt)
            assert rexp.same(rexp.as_fmt(got.cpu().numpy(), fmt, (c1 - c0, rows)), want), (name, fmt, c0, c1)
            st.close()
            del band
        assert int(img[0]) == rexp.CANARY and bool((img[end:end + 16] == rexp.CANARY).all()), fmt
    del img


# ---- 5. raster import --------------------------------------------------------------------------------------------------
def import_device(ctx, layer, band_ptr, width, height, stride, gt, method):
    ctx.check(L().amb_import_raster_device(ctx.h, LAYER[layer], C.c_void_p(band_ptr), width, height, stride,
                                           (C.c_double * 6)(*gt), 0, 0.0, _lib.RESAMPLE[method]))
    ctx.sync()


def import_host(ctx, layer, band, gt, method):
    ctx.check(L().amb_import_raster(ctx.h, LAYER[layer], band.ctypes.data_as(C.c_void_p), band.shape[1], band.shape[0],
                                    band.strides[0], (C.c_double * 6)(*gt), 0, 0.0, _lib.RESAMPLE[method]))
    ctx.sync()


def geotransform(ctx):
    gt = (C.c_double * 6)()
    amb.check(L().amb_raster_geotransform(C.byref(ctx.g), gt))
    return tuple(gt)


@pytest.mark.parametrize("method", ["nearest", "bilinear"])
@pytest.mark.parametrize("name", ["S1", "S3"])
def test_raster_import_of_the_export_gives_the_layer_back(name, method, res):
    import torch
    shape = SHAPES[name]
    rows, cols = shape
    need_device(3 * layer_gib(shape) + 0.5, "raster import on %s" % name)     # layer, its F32 image, target layer
    wins = windows(shape)
    assert_windows_reach(shape, wins)
    big = res.ctx(shape)
    fill_pattern(big.view("elevation"), 0)
    img = torch.empty(big.cells, dtype=torch.float32, device="cuda")
    export_device(big, "elevation", "f32", img.data_ptr())
    target = big.view("delta")
    target.fill_(rimp.SENTINEL)
    torch.cuda.synchronize()
    import_device(big, "delta", img.data_ptr(), rows, cols, rows * 4, geotransform(big), method)
    del img
    src_bits, dst_bits = big.view("elevation", torch.int32), big.view("delta", torch.int32)
    sentinel = int(np.float32(rimp.SENTINEL).view(np.int32))
    for c0, c1 in wins:
        lo, hi = c0 * rows, c1 * rows
        s, d = src_bits[lo:hi], dst_bits[lo:hi]
        nan = (s & 0x7FFFFFFF) > 0x7F800000                          # no-data: the cell keeps its value
        want = torch.where(nan, torch.full_like(s, sentinel), s)
        assert_same_bits(d, want, "%s %s columns [%d, %d)" % (name, method, c0, c1))
        assert bool(nan.any()) and bool((~nan).any())


@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_resampled_import_into_s1_equals_stripes_and_restatement(method, res):
    import torch
    shape = S1
    rows, cols = shape
    need_device(layer_gib(shape) + 0.5, "resampled import on S1")
    wins = windows(shape)
    assert_windows_reach(shape, wins)
    # a DEM at 0.37 m covering the map and a little more, north-up, offset from the map's grid
    dres = 0.37
    w, h = int(rows * RES / dres) + 3, int(cols * RES / dres) + 3
    band = rimp.dem(h, w, seed=7, nan_frac=0.01)
    big = res.ctx(shape)
    gt0 = geotransform(big)
    gt = (gt0[0] - 0.211, dres, 0.0, gt0[3] + 0.163, 0.0, -dres)
    big.view("elevation").fill_(rimp.SENTINEL)
    torch.cuda.synchronize()
    import_host(big, "elevation", band, gt, method)
    for c0, c1 in wins:
        st = res.ctx(shape, c0, c1)
        st.view("elevation").fill_(rimp.SENTINEL)
        torch.cuda.synchronize()
        import_host(st, "elevation", band, gt, method)
        assert_same_bits(big.cols_of("elevation", c0, c1), st.view("elevation", torch.int32),
                         "S1 %s columns [%d, %d)" % (method, c0, c1))
        before = np.full((rows, c1 - c0), rimp.SENTINEL, np.float32, order="F")
        want = rimp.restate(before, big.g, band, gt, method, col_range=(c0, c1))
        got = st.view("elevation").cpu().numpy().reshape((rows, c1 - c0), order="F")
        assert rimp.same(got, want), (method, c0, c1)
        assert (got != rimp.SENTINEL).mean() > 0.9


# ---- 6. JPEG -----------------------------------------------------------------------------------------------------------
def test_jpeg_of_an_s1_gray_layer_equals_opencv(res):
    import test_gpu_jpeg_encode as tj
    shape = S1
    rows, cols = shape
    need_device(3 * layer_gib(shape) + 2.0, "JPEG of S1")     # layer, GRAY8 band, the encoder's buffers
    if host_available_gib() < 4 * layer_gib(shape, 1) + 2.0:
        pytest.skip("JPEG of S1 needs ~%.1f GiB of host memory; %.1f GiB available"
                    % (4 * layer_gib(shape, 1) + 2.0, host_available_gib()))
    big = res.ctx(shape)
    fill_pattern(big.view("ortho"), 0)
    img = np.empty((cols, rows), np.uint8)                    # the GRAY8 export: 2^31 + 4633 pixels
    big.check(L().amb_export_raster(big.h, LAYER["ortho"], _lib.RASTER_GRAY8, img.ctypes.data_as(C.c_void_p)))
    cap = L().amb_jpeg_max_size(rows, cols, 1, 95, 0, 0)
    out = np.empty(cap, np.uint8)
    size = C.c_size_t(0)
    big.check(L().amb_export_jpeg(big.h, LAYER["ortho"], _lib.RASTER_GRAY8, 95, 0, 0, out.ctypes.data_as(C.c_void_p),
                                  cap, C.byref(size)))
    got = out[:size.value].tobytes()
    del out
    want = tj.cv2_jpeg(img, 95)
    assert len(got) == len(want) and got == want, tj.first_difference(got, want)
    assert 8 * len(got) > (1 << 32)      # the entropy-coded stream's bit offsets pass 2^32


# ---- 7. the ABI's size limits --------------------------------------------------------------------------------------------
def create_status(rows, cols, c0=0, c1=None):
    g = amb.Geometry(rows, cols, 1.0, float(rows), float(cols), 0.0, 0.0)
    h = C.c_void_p()
    st = L().amb_create(C.byref(g), 0, c0, cols if c1 is None else c1, C.byref(h))
    if st == _lib.AMB_OK:
        L().amb_destroy(h)
    return st


def test_amb_create_admits_slabs_below_2_pow_32_minus_1_cells():
    assert 65537 * 65535 == (1 << 32) - 1 and 2 * ((1 << 31) - 1) == (1 << 32) - 2
    assert create_status(65537, 65535) == _lib.AMB_ERR_UNSUPPORTED
    assert create_status((1 << 31) - 1, 2) == _lib.AMB_OK                      # 2^32 - 2 cells (layers are lazy)
    assert create_status(65536, 65536) == _lib.AMB_ERR_UNSUPPORTED
    assert create_status(65536, 65536, 0, 65535) == _lib.AMB_OK                # a stripe of the same map fits
    assert create_status(65536, 65536, 1, 65536) == _lib.AMB_OK


def test_dsm_and_ortho_from_pcl_refuse_2_pow_27_rows(res):
    need_device(1.0, "the DSM row limit")
    xyz = np.array([[0.3, 0.2, 100.0], [1.7, -0.4, 101.0]])
    inten = np.array([10, 20], np.int32)
    ctx = res.ctx((1 << 27, 1))
    assert L().amb_dsm_process(ctx.h, xyz.ctypes.data_as(C.c_void_p), 2, 1, 0.0, 0.0) == _lib.AMB_ERR_UNSUPPORTED
    assert L().amb_ortho_from_pcl_process(ctx.h, xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p), 2,
                                          2, 0) == _lib.AMB_ERR_UNSUPPORTED
