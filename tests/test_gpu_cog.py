"""Cloud-Optimized GeoTIFF tiles on the device (amb_cog_tiles_device, amb_export_cog_tiles, csrc/raster_pyramid.cu;
convention in include/aerial_mapper_b200.h): every tile must inflate with zlib, with nothing after its stream and within
its bound, to the numpy restatement of tests/test_cog_cpu.py (the pyramid, zero padding, the predictor), and the files
GridMap.to_cog writes must read back with level 0 equal to to_raster and every overview equal to the restatement.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels, so the kernel logic is checked on
every CPU run too (the 10000 x 10000 case and the torch wrapper need a GPU)."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, io  # noqa: E402
from test_cog_cpu import (BPP, FORMATS, QNAN, bound, check_cog_structure, content, layout, predicted_tiles,  # noqa: E402
                          pyramid, read_level, same_bits)
from test_gpu_geotiff_deflate import CANARY, EMULATED, Dev, mapping_run  # noqa: E402

gpu = pytest.mark.gpu


def cog_dev(d, h, w, fmt, tile, out=None, capacity=None, counts=None):
    L = _lib.lib()
    f = _lib.RASTER_FORMAT[fmt]
    cap = L.amb_cog_max_size(w, h, f, tile)
    buf = np.empty(max(cap, 1), np.uint8) if out is None else out
    n_tiles = sum(-(-a // tile) * -(-b // tile) for a, b in layout(w, h, tile)[1])
    counts = np.zeros(n_tiles, np.uint32) if counts is None else counts
    size = C.c_size_t(0)
    st = L.amb_cog_tiles_device(api._jpeg_context(0), d.ptr, w, h, d.pitch, f, tile, buf.ctypes.data,
                                cap if capacity is None else capacity, C.byref(size), counts.ctypes.data)
    return st, buf, size.value, counts


def check_tiles(img, fmt, tile, data, counts):
    """Every tile inflates to its restated predicted bytes, with nothing after it, within the bound."""
    want = predicted_tiles(img, fmt, tile)
    assert len(counts) == len(want) and int(np.sum(counts, dtype=np.int64)) == len(data)
    at = 0
    for k, n in enumerate(counts):
        t = data[at:at + int(n)]
        at += int(n)
        z = zlib.decompressobj()
        got = z.decompress(t)
        assert z.eof and z.unused_data == b"" and got == want[k], (fmt, tile, img.shape, k, len(got))
        assert len(t) <= bound(tile * tile * BPP[fmt]) and t[:2] == b"\x78\x01"


def cog(img, fmt, tile, pitch=None, off=0):
    h, w = img.shape[:2]
    st, buf, n, counts = cog_dev(Dev(img, pitch, off), h, w, fmt, tile)
    amb.check(st, api._jpeg_context(0))
    data = buf[:n].tobytes()
    check_tiles(img, fmt, tile, data, counts)
    return data, counts


def decoded_levels(data, counts, w, h, fmt, tile):
    """The levels the device's tiles hold (inflated, predictor undone, padding dropped), level 0 first."""
    levels = layout(w, h, tile)[1]
    item, spp = (4, 1) if fmt == "f32" else (1, 3 if fmt == "bgr8" else 1)
    dtype = np.float32 if fmt == "f32" else np.uint8
    out, at, k = [], 0, 0
    for lw, lh in levels[::-1]:
        a = np.zeros((lh, lw, spp), dtype)
        for ty in range(-(-lh // tile)):
            for tx in range(-(-lw // tile)):
                raw = zlib.decompress(data[at:at + int(counts[k])])
                at += int(counts[k])
                k += 1
                t = io._undo_predictor(raw, 3 if fmt == "f32" else 2, dtype, tile, tile, spp)
                part = a[ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile]
                part[...] = t[:part.shape[0], :part.shape[1]]
        if fmt == "bgr8":
            a = a[:, :, ::-1]            # stored as R, G, B
        out.append(a if spp == 3 else a[:, :, 0])
    return out[::-1]


# ---- formats x tile sides x sizes -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("tile", [16, 32, 512])
def test_every_format_tile_side_and_size(fmt, tile):
    sizes = [(1, 1), (1, 37), (37, 1), (17, 33), (tile, tile), (tile + 1, 2 * tile + 1)]
    if tile < 512 or not EMULATED:   # odd sizes with partial 2 x 2 windows at several levels
        sizes += [(2 * tile + 3, 4 * tile + 5), (5 * tile - 1, 3 * tile + 7)]
    for k, (h, w) in enumerate(sizes):
        cog(content(fmt, h, w, seed=k + tile), fmt, tile)


@gpu
def test_10000_by_10000_dem():
    if EMULATED:
        return   # minutes on the emulated kernels; every path it takes is covered by the smaller cases
    from test_gpu_geotiff_deflate import content as deflate_content
    img = deflate_content("smooth", "f32", 10000, 10000, seed=3)
    cog(img, "f32", 512)


# ---- edge content -----------------------------------------------------------------------------------------------------------
@gpu
def test_f32_edge_values():
    rng = np.random.default_rng(4)
    inf = np.float32(np.inf)
    payloads = np.array([0x7FA00001, 0xFFC00123, 0x7F800001, 0xFFFFFFFF, 0x7FC00000], np.uint32).view(np.float32)
    pool = np.concatenate([payloads, [inf, -inf, np.float32(-0.0), np.float32(0.0), np.float32(1.5),
                                      np.float32(-2.25), np.float32(3.4e38), np.float32(1e-45)]]).astype(np.float32)
    for h, w in ((35, 67), (64, 64), (33, 17)):
        img = pool[rng.integers(0, len(pool), (h, w))]
        data, counts = cog(img, "f32", 16)
        lv = decoded_levels(data, counts, w, h, "f32", 16)
        for a in lv[1:]:   # every NaN of an overview is the quiet NaN 0x7FC00000
            assert (a.view(np.uint32)[np.isnan(a)] == 0x7FC00000).all()
    # all-NaN windows and single survivors, -0 alone and with +0
    img = np.full((40, 40), np.nan, np.float32)
    img[0, 0] = -0.0
    img[2, 3] = 7.25
    img[5, 5] = -0.0
    img[4, 4] = 0.0
    img[10, 10], img[10, 11] = inf, -inf
    data, counts = cog(img, "f32", 16)
    lv1 = decoded_levels(data, counts, 40, 40, "f32", 16)[1]
    assert lv1[0, 0].view(np.uint32) == 0x80000000 and lv1[1, 1] == 7.25 and lv1[2, 2].view(np.uint32) == 0
    assert lv1[5, 5].view(np.uint32) == 0x7FC00000 and lv1[3, 3].view(np.uint32) == 0x7FC00000


@gpu
def test_8bit_half_way_sums_and_the_mask_f32_invariant():
    rng = np.random.default_rng(6)
    for fmt in ("gray8", "bgr8"):
        shape = (61, 93, 3) if fmt == "bgr8" else (61, 93)
        for lo, hi in ((254, 256), (0, 4), (0, 256)):   # small ranges: sums that end in .5 and .25 / .75 of n
            img = rng.integers(lo, hi, shape).astype(np.uint8)
            cog(img, fmt, 16)
        cog(np.full(shape, 255, np.uint8), fmt, 16)
    for h, w in ((70, 45), (129, 33)):
        dem = content("f32", h, w, seed=h)
        dem[rng.random((h, w)) < 0.6] = np.nan
        mask = np.where(np.isnan(dem), 0, 255).astype(np.uint8)
        fl = decoded_levels(*cog(dem, "f32", 16), w, h, "f32", 16)
        ml = decoded_levels(*cog(mask, "mask8", 16), w, h, "mask8", 16)
        assert len(fl) == len(ml) > 2
        for a, m in zip(fl, ml):
            assert np.array_equal(np.where(np.isnan(a), 0, 255), m)


# ---- inputs, outputs and contracts ------------------------------------------------------------------------------------------
@gpu
def test_pitched_and_misaligned_inputs():
    for fmt in FORMATS:
        img = content(fmt, 37, 41, seed=1)
        row = 41 * BPP[fmt]
        offs = (0, 4, 8, 12) if fmt == "f32" else range(8)
        for off in offs:
            cog(img, fmt, 16, pitch=row + 4 * (off + 1), off=off)


@gpu
def test_repeated_calls_give_identical_bytes_and_pinned_equals_pageable():
    for fmt in FORMATS:
        img = content(fmt, 150, 170, seed=5)
        d = Dev(img)
        first = None
        for _ in range(2):
            st, buf, n, counts = cog_dev(d, 150, 170, fmt, 32)
            assert st == 0
            got = (buf[:n].tobytes(), counts.tobytes())
            assert first is None or got == first
            first = got
    img = content("bgr8", 700, 900, seed=7)   # a few MB of tiles: large enough for the staged pageable copy
    d = Dev(img)
    L = _lib.lib()
    cap = L.amb_cog_max_size(900, 700, _lib.RASTER_BGR8, 256)
    p = C.c_void_p()
    amb.check(L.amb_host_alloc(C.byref(p), cap))
    try:
        pinned = np.frombuffer((C.c_uint8 * cap).from_address(p.value), np.uint8)
        st, _, n, c1 = cog_dev(d, 700, 900, "bgr8", 256, out=pinned)
        assert st == 0
        st, pageable, m, c2 = cog_dev(d, 700, 900, "bgr8", 256)
        assert st == 0 and n == m and pinned[:n].tobytes() == pageable[:m].tobytes() and np.array_equal(c1, c2)
        check_tiles(img, "bgr8", 256, pageable[:m].tobytes(), c2)
    finally:
        L.amb_host_free(p)


@gpu
def test_too_small_a_capacity_returns_the_size_and_writes_nothing():
    img = content("f32", 40, 50, seed=1)
    d = Dev(img)
    st, buf, n, counts = cog_dev(d, 40, 50, "f32", 16)
    assert st == 0
    want = buf[:n].tobytes()
    for cap in (0, 1, n - 1):
        out = np.full(n + 64, CANARY, np.uint8)
        cnt = np.full(len(counts), 0xA5A5A5A5, np.uint32)
        st, _, m, _ = cog_dev(d, 40, 50, "f32", 16, out=out, capacity=cap, counts=cnt)
        assert st == _lib.AMB_ERR_SIZE_MISMATCH and m == n and (out == CANARY).all() and (cnt == 0xA5A5A5A5).all()
    out = np.full(n + 64, CANARY, np.uint8)
    st, _, m, cnt = cog_dev(d, 40, 50, "f32", 16, out=out, capacity=n)
    assert st == 0 and out[:m].tobytes() == want and (out[m:] == CANARY).all() and np.array_equal(cnt, counts)


@gpu
def test_invalid_arguments_write_nothing():
    L = _lib.lib()
    ctx = api._jpeg_context(0)
    d = Dev(content("f32", 9, 9, seed=2))
    buf = np.full(1 << 16, CANARY, np.uint8)
    cnt = np.full(16, 0xA5A5A5A5, np.uint32)
    size = C.c_size_t(12345)
    INV = _lib.AMB_ERR_INVALID_ARGUMENT
    # (ctx, image, w, h, stride, format, tile, out given, counts given, size given)
    good = [ctx, d.ptr, 9, 9, 36, 0, 16, True, True, True]
    cases = [(0, None), (1, None), (7, False), (8, False), (9, False), (2, 0), (3, -1), (4, 35), (4, 38), (5, 4),
             (6, 0), (6, 8), (6, 24), (6, 4112), (1, d.ptr + 2)]
    for k, v in cases:
        a = list(good)
        a[k] = v
        st = L.amb_cog_tiles_device(a[0], a[1], a[2], a[3], a[4], a[5], a[6], buf.ctypes.data if a[7] else None,
                                    len(buf), C.byref(size) if a[9] else None, cnt.ctypes.data if a[8] else None)
        assert st == INV, (k, v, st)
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable()
    gm.to_device(0)
    gc = gm.context()
    for layer, fmt, tile in ((-1, 0, 16), (len(_lib.LAYER_NAMES), 0, 16), (0, 4, 16), (0, 0, 0), (0, 0, 40)):
        assert L.amb_export_cog_tiles(gc, layer, fmt, tile, buf.ctypes.data, len(buf), C.byref(size),
                                      cnt.ctypes.data) == INV
    assert L.amb_export_cog_tiles(None, 0, 0, 16, buf.ctypes.data, len(buf), C.byref(size), cnt.ctypes.data) == INV
    assert L.amb_export_cog_tiles(gc, 0, 0, 16, buf.ctypes.data, len(buf), C.byref(size), None) == INV
    gm.sync()
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    for kw in ({"fmt": "rgb8"}, {"tile_size": 24}, {"tile_size": 8192}, {"nodata": -9999.0}, {"fmt": "gray8", "nodata": 0}):
        with pytest.raises(ValueError):
            gm.to_cog("unused.tif", "elevation", **kw)
    with pytest.raises(ValueError):
        gm.to_cog("unused.tif", "elevation_angle")
    with pytest.raises(amb.AmbError):
        amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable().to_cog("unused.tif", "elevation")
    assert not os.path.exists("unused.tif")


# ---- files of map layers ---------------------------------------------------------------------------------------------------
@gpu
def test_files_read_back_at_every_level(tmp_path):
    cv2 = pytest.importorskip("cv2")
    gm = mapping_run()
    gm.sync()
    for name, fmt in (("elevation", "f32"), ("ortho", "gray8"), ("colored_ortho", "bgr8"),
                      ("observation_index", "mask8")):
        band = gm.to_raster(name, fmt)
        path = str(tmp_path / ("%s_%s.tif" % (name, fmt)))
        gm.to_cog(path, name, fmt=fmt, nodata="nan" if fmt == "f32" else None, tile_size=16)
        h, w = band.shape[:2]
        check_cog_structure(path, w, h, 16, fmt)
        levels = pyramid(band, fmt, 16)
        assert len(levels) == 4
        ok, pages = cv2.imreadmulti(path, flags=cv2.IMREAD_UNCHANGED)
        assert ok and len(pages) == len(levels)
        for k, lv in enumerate(levels):
            a = read_level(path, k, fmt)
            assert same_bits(a, lv), (name, k)
            assert same_bits(pages[k], lv), ("cv2", name, k)
        gt, epsg = io.read_geotiff(path)[1:3]
        assert gt == gm.geotransform() and epsg == 32632


@gpu
def test_overview_one_imports_into_a_map_of_twice_the_cell_size(tmp_path):
    gm = mapping_run(72, 56)
    path = str(tmp_path / "dem.tif")
    gm.to_cog(path, "elevation", nodata="nan", tile_size=16)
    a, gt, _, nodata = io.read_geotiff(path, overview=1)
    assert a.shape == (28, 36) and gt[1] == 2.0 and gt[5] == -2.0
    coarse = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, 72.0, 56.0, 2.0)).getMutable()
    assert coarse.getSize() == (36, 28) and coarse.geotransform() == gt
    coarse["elevation"] = np.full((36, 28), QNAN, np.float32, order="F")
    coarse.to_device(0, names=("elevation",))
    coarse.from_raster("elevation", a, gt, nodata=nodata, resample="nearest")
    assert same_bits(coarse.to_raster("elevation"), a)
    coarse.from_raster("elevation", a, gt, nodata=nodata, resample="bilinear")
    assert same_bits(coarse.to_raster("elevation"), a)


@gpu
def test_a_stripe_writes_its_band_and_export_after_queued_work(tmp_path):
    whole = mapping_run()
    whole.download(("elevation",))
    elev = whole["elevation"].copy(order="F")
    rows, cols = whole.getSize()
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * 1.0, cols * 1.0, 1.0)).getMutable()
    gm["elevation"] = elev
    gm.to_device(0, col_range=(13, 40), names=("elevation",))
    band = gm.to_raster("elevation")
    path = str(tmp_path / "stripe.tif")
    gm.to_cog(path, "elevation", nodata="nan", tile_size=16)
    check_cog_structure(path, band.shape[1], band.shape[0], 16, "f32")
    for k, lv in enumerate(pyramid(band, "f32", 16)):
        assert same_bits(io.read_geotiff(path, overview=k)[0], lv)
    full_gt = gm.geotransform()
    assert io.read_geotiff(path)[1] == (full_gt[0], full_gt[1], 0.0, full_gt[3] + 13 * full_gt[5], 0.0, full_gt[5])
    # an export queued right after the DSM, without a sync, equals one after it
    from aerial_mapper_b200 import synth
    rows, cols, res = 300, 260, 0.5
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(60000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    first, second = str(tmp_path / "first.tif"), str(tmp_path / "second.tif")
    gm.to_cog(first, "elevation", tile_size=64)
    gm.sync()
    gm.to_cog(second, "elevation", tile_size=64)
    assert open(first, "rb").read() == open(second, "rb").read()
    assert same_bits(io.read_geotiff(first)[0], gm.to_raster("elevation"))


@gpu
def test_torch_wrapper(tmp_path):
    if EMULATED:
        return   # the wrapper takes torch CUDA tensors; its C entry point is what every other test here calls
    import torch
    img = content("bgr8", 123, 77, seed=4)
    t = torch.from_numpy(img).cuda()
    data, counts = amb.cog_tiles(t, "bgr8", tile_size=32)
    check_tiles(img, "bgr8", 32, data, counts)
    big = torch.zeros((123, 100, 3), dtype=torch.uint8, device="cuda")
    big[:, :77] = t
    padded = amb.cog_tiles(big[:, :77], "bgr8", tile_size=32)
    assert padded[0] == data and np.array_equal(padded[1], counts)
    dem = content("f32", 600, 700, seed=1)
    data, counts = amb.cog_tiles(torch.from_numpy(dem).cuda(), "f32")
    check_tiles(dem, "f32", 512, data, counts)
    path = str(tmp_path / "dem.tif")
    io.write_cog(path, data, counts, 700, 600, "f32", 512, (0.0, 0.5, 0.0, 10.0, 0.0, -0.5), nodata="nan")
    assert same_bits(io.read_geotiff(path)[0], dem)
    for bad in ((t.float(), "bgr8", 32), (t[:, ::2], "bgr8", 32), (t, "rgb8", 32), (t, "bgr8", 20)):
        with pytest.raises(ValueError):
            amb.cog_tiles(*bad)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_cog.py"], sched=sched, opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
