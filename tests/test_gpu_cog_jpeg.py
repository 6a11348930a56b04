"""JPEG and 1-bit mask tiles of a Cloud-Optimized GeoTIFF on the device (amb_cog_jpeg_tiles_device,
amb_export_cog_jpeg_tiles, amb_cog_mask_tiles_device, amb_export_cog_mask_tiles; csrc/raster_pyramid.cu and
csrc/jpeg_encode.cu; convention in include/aerial_mapper_b200.h): every image tile must equal SOI + SOF0 + SOS + the
entropy-coded data + EOI of cv2.imencode of the same tile of the numpy pyramid (tests/test_cog_jpeg_cpu.py), the tables
stream OpenCV's DQT and DHT segments, and every mask tile must inflate and unpack to the MASK8 pyramid's tile != 0.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels, so the kernel logic is checked on
every CPU run too (the 10000 x 10000 case, the device decoder and the torch wrapper need a GPU)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, io  # noqa: E402
from test_cog_cpu import bound, content, layout, pyramid  # noqa: E402
from test_cog_jpeg_cpu import KINDS, EOI, SOI, cv2_tiles, ifds, splice, tiles_of, unpack_mask  # noqa: E402
from test_gpu_geotiff_deflate import CANARY, EMULATED, Dev, mapping_run  # noqa: E402

cv2 = pytest.importorskip("cv2")
gpu = pytest.mark.gpu
QUALITIES = (1, 50, 75, 100)


def jpeg_dev(d, h, w, fmt, tile, quality=75, sampling="420", out=None, capacity=None, counts=None):
    L = _lib.lib()
    f = _lib.RASTER_FORMAT[fmt]
    s = api.JPEG_SAMPLING[sampling]
    cap = L.amb_cog_jpeg_max_size(w, h, f, tile, quality, s)
    buf = np.empty(max(cap, 1), np.uint8) if out is None else out
    n_tiles = sum(-(-a // tile) * -(-b // tile) for a, b in layout(w, h, tile)[1])
    counts = np.zeros(n_tiles, np.uint32) if counts is None else counts
    size = C.c_size_t(0)
    st = L.amb_cog_jpeg_tiles_device(api._jpeg_context(0), d.ptr, w, h, d.pitch, f, tile, quality, s, buf.ctypes.data,
                                     cap if capacity is None else capacity, C.byref(size), counts.ctypes.data)
    return st, buf, size.value, counts


def mask_dev(d, h, w, tile, out=None, capacity=None, counts=None):
    L = _lib.lib()
    cap = L.amb_cog_mask_max_size(w, h, tile)
    buf = np.empty(max(cap, 1), np.uint8) if out is None else out
    n_tiles = sum(-(-a // tile) * -(-b // tile) for a, b in layout(w, h, tile)[1])
    counts = np.zeros(n_tiles, np.uint32) if counts is None else counts
    size = C.c_size_t(0)
    st = L.amb_cog_mask_tiles_device(api._jpeg_context(0), d.ptr, w, h, d.pitch, tile, buf.ctypes.data,
                                     cap if capacity is None else capacity, C.byref(size), counts.ctypes.data)
    return st, buf, size.value, counts


def streams_of(data, counts):
    at = np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64))])
    assert at[-1] == len(data)
    return [data[at[k]:at[k + 1]] for k in range(len(counts))]


def check_jpeg(img, fmt, tile, quality, sampling, data, counts):
    tables, want = cv2_tiles(img, fmt, tile, quality, sampling)
    got = streams_of(data, counts)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, (fmt, sampling, quality, tile, img.shape, k, len(g), len(w))
    assert api.cog_jpeg_tables(fmt, quality) == tables
    return tables, got


def jpeg(img, fmt, tile, quality=75, sampling="420", pitch=None, off=0):
    h, w = img.shape[:2]
    st, buf, n, counts = jpeg_dev(Dev(img, pitch, off), h, w, fmt, tile, quality, sampling)
    amb.check(st, api._jpeg_context(0))
    data = buf[:n].tobytes()
    check_jpeg(img, fmt, tile, quality, sampling, data, counts)
    return data, counts


def check_mask(mask8, tile, data, counts):
    want = tiles_of(mask8, "mask8", tile)
    got = streams_of(data, counts)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g[:2] == b"\x78\x01" and len(g) <= bound(tile * tile // 8)
        assert np.array_equal(unpack_mask(g, tile), w != 0), (tile, mask8.shape, k)


def mask(mask8, tile, pitch=None, off=0):
    h, w = mask8.shape
    st, buf, n, counts = mask_dev(Dev(mask8, pitch, off), h, w, tile)
    amb.check(st, api._jpeg_context(0))
    data = buf[:n].tobytes()
    check_mask(mask8, tile, data, counts)
    return data, counts


def smooth(fmt, h, w, seed):
    """Image-like content: gradients and waves with a little noise (the content JPEG is for)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (np.sin(xx / 9.0) * 60 + np.cos(yy / 13.0) * 50 + 120)[..., None] + rng.normal(0, 8, (h, w, 3))
    a = np.clip(base + np.array([0, 25, -25]), 0, 255).astype(np.uint8)
    return a if fmt == "bgr8" else np.ascontiguousarray(a[:, :, 1])


# ---- kinds x qualities x tile sides x sizes ---------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("tile", [16, 32, 512])
def test_every_kind_quality_tile_side_and_size(kind, tile):
    fmt, sampling = KINDS[kind]
    sizes = [(1, 1), (17, 33), (tile, tile), (tile + 1, tile)]
    if tile < 512 or not EMULATED:   # odd sizes over several levels
        sizes += [(2 * tile + 3, 4 * tile + 5), (5 * tile - 1, 3 * tile + 7)]
    qualities = QUALITIES if tile < 512 or not EMULATED else (1, 75)
    for k, (h, w) in enumerate(sizes):
        for q in qualities:
            img = (smooth if (k + q) % 2 else lambda f, a, b, seed: content(f, a, b, seed))(fmt, h, w, k + tile + q)
            jpeg(img, fmt, tile, q, sampling)


@gpu
def test_10000_by_10000_rasters():
    if EMULATED:
        return   # minutes on the emulated kernels; every path it takes is covered by the smaller cases
    for kind in ("gray", "420"):
        fmt, sampling = KINDS[kind]
        jpeg(smooth(fmt, 10000, 10000, seed=3), fmt, 512, 75, sampling)
    m = np.where(np.random.default_rng(5).random((10000, 10000)) < 0.3, 0, 255).astype(np.uint8)
    mask(m, 512)


# ---- decoding --------------------------------------------------------------------------------------------------------------
@gpu
def test_spliced_tiles_decode_as_opencv_decodes_them():
    for kind in sorted(KINDS):
        fmt, sampling = KINDS[kind]
        img = smooth(fmt, 70, 90, seed=2)
        data, counts = jpeg(img, fmt, 32, 90, sampling)
        tables = api.cog_jpeg_tables(fmt, 90)
        files = [splice(tables, s) for s in streams_of(data, counts)]
        ch = 3 if fmt == "bgr8" else 1
        want = [cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR if ch == 3 else cv2.IMREAD_GRAYSCALE)
                for f in files]
        for f, t, w in zip(files, tiles_of(img, fmt, 32), want):
            assert f[:2] == SOI and f[-2:] == EOI and w.shape == t.shape
            assert np.abs(w.astype(int) - t.astype(int)).mean() < 12   # a JPEG of the tile, not of something else
        if not EMULATED:   # the project's own decoder takes the spliced streams too
            got = amb.decode_jpeg(files, channels=ch)
            for g, w in zip(got, want):
                assert np.array_equal(g.cpu().numpy(), w)


# ---- masks -----------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("tile", [16, 32, 512])
def test_mask_tiles_at_every_tile_side_and_size(tile):
    sizes = [(1, 1), (17, 33), (tile, tile), (tile + 1, 2 * tile + 1)]
    if tile < 512 or not EMULATED:
        sizes += [(2 * tile + 3, 4 * tile + 5)]
    for k, (h, w) in enumerate(sizes):
        m = content("mask8", h, w, seed=k)
        m[m != 0] = (k * 37 + 1) % 255 + 1   # any non-zero byte is valid
        mask(m, tile)
    mask(np.zeros((40, 40), np.uint8), 16)
    mask(np.full((40, 40), 255, np.uint8), 16)


@gpu
def test_observation_index_mask_of_a_map_with_unobserved_cells():
    gm = mapping_run()
    gm.sync()
    m = gm.to_raster("observation_index", "mask8")
    assert (m == 0).any() and (m != 0).any()
    L = _lib.lib()
    h, w = m.shape
    cap = L.amb_cog_mask_max_size(w, h, 16)
    buf = np.empty(cap, np.uint8)
    counts = np.zeros(sum(-(-a // 16) * -(-b // 16) for a, b in layout(w, h, 16)[1]), np.uint32)
    size = C.c_size_t(0)
    amb.check(L.amb_export_cog_mask_tiles(gm.context(), _lib.LAYER_ID["observation_index"], 16, buf.ctypes.data, cap,
                                          C.byref(size), counts.ctypes.data))
    check_mask(m, 16, buf[:size.value].tobytes(), counts)


# ---- inputs, outputs and contracts ------------------------------------------------------------------------------------------
@gpu
def test_pitched_and_misaligned_inputs():
    for kind in sorted(KINDS):
        fmt, sampling = KINDS[kind]
        img = smooth(fmt, 37, 41, seed=1)
        row = img[0].nbytes
        for off in range(0, 8, 3):
            jpeg(img, fmt, 16, 75, sampling, pitch=row + 4 * (off + 1), off=off)
    m = content("mask8", 37, 41, seed=1)
    for off in range(0, 8, 3):
        mask(m, 16, pitch=41 + 4 * (off + 1), off=off)


@gpu
def test_repeated_calls_give_identical_bytes_and_pinned_equals_pageable():
    img = smooth("bgr8", 700, 900, seed=7)   # a few MB of tiles: large enough for the staged pageable copy
    d = Dev(img)
    first = None
    for _ in range(2):
        st, buf, n, counts = jpeg_dev(d, 700, 900, "bgr8", 256, 95, "444")
        assert st == 0
        got = (buf[:n].tobytes(), counts.tobytes())
        assert first is None or got == first
        first = got
    L = _lib.lib()
    cap = L.amb_cog_jpeg_max_size(900, 700, _lib.RASTER_BGR8, 256, 95, 1)
    p = C.c_void_p()
    amb.check(L.amb_host_alloc(C.byref(p), cap))
    try:
        pinned = np.frombuffer((C.c_uint8 * cap).from_address(p.value), np.uint8)
        st, _, n, c1 = jpeg_dev(d, 700, 900, "bgr8", 256, 95, "444", out=pinned)
        assert st == 0 and pinned[:n].tobytes() == first[0] and c1.tobytes() == first[1]
    finally:
        L.amb_host_free(p)
    check_jpeg(img, "bgr8", 256, 95, "444", first[0], np.frombuffer(first[1], np.uint32))
    md = Dev(content("mask8", 300, 200, seed=3))
    a = mask_dev(md, 300, 200, 32)
    b = mask_dev(md, 300, 200, 32)
    assert a[0] == b[0] == 0 and a[1][:a[2]].tobytes() == b[1][:b[2]].tobytes() and np.array_equal(a[3], b[3])


@gpu
def test_too_small_a_capacity_returns_the_size_and_writes_nothing():
    img = smooth("bgr8", 40, 50, seed=1)
    d = Dev(img)
    st, buf, n, counts = jpeg_dev(d, 40, 50, "bgr8", 16)
    assert st == 0
    want = buf[:n].tobytes()
    for cap in (0, 1, n - 1):
        out = np.full(n + 64, CANARY, np.uint8)
        cnt = np.full(len(counts), 0xA5A5A5A5, np.uint32)
        st, _, m, _ = jpeg_dev(d, 40, 50, "bgr8", 16, out=out, capacity=cap, counts=cnt)
        assert st == _lib.AMB_ERR_SIZE_MISMATCH and m == n and (out == CANARY).all() and (cnt == 0xA5A5A5A5).all()
    out = np.full(n + 64, CANARY, np.uint8)
    st, _, m, cnt = jpeg_dev(d, 40, 50, "bgr8", 16, out=out, capacity=n)
    assert st == 0 and out[:m].tobytes() == want and (out[m:] == CANARY).all() and np.array_equal(cnt, counts)
    md = Dev(content("mask8", 40, 50, seed=1))
    st, buf, n, counts = mask_dev(md, 40, 50, 16)
    assert st == 0
    out = np.full(n + 64, CANARY, np.uint8)
    cnt = np.full(len(counts), 0xA5A5A5A5, np.uint32)
    st, _, m, _ = mask_dev(md, 40, 50, 16, out=out, capacity=n - 1, counts=cnt)
    assert st == _lib.AMB_ERR_SIZE_MISMATCH and m == n and (out == CANARY).all() and (cnt == 0xA5A5A5A5).all()


@gpu
def test_bad_arguments_give_the_documented_status_and_write_nothing():
    L = _lib.lib()
    ctx = api._jpeg_context(0)
    d = Dev(smooth("bgr8", 9, 9, seed=2))
    buf = np.full(1 << 16, CANARY, np.uint8)
    cnt = np.full(16, 0xA5A5A5A5, np.uint32)
    size = C.c_size_t(12345)
    INV, UNS = _lib.AMB_ERR_INVALID_ARGUMENT, _lib.AMB_ERR_UNSUPPORTED
    # (ctx, image, w, h, stride, format, tile, quality, sampling, out given, counts given, size given)
    good = [ctx, d.ptr, 9, 9, 27, _lib.RASTER_BGR8, 16, 75, 0, True, True, True]
    cases = [(0, None, INV), (1, None, INV), (9, False, INV), (10, False, INV), (11, False, INV), (2, 0, INV),
             (3, -1, INV), (4, 26, INV), (5, _lib.RASTER_F32, INV), (5, _lib.RASTER_MASK8, INV), (5, 4, INV),
             (6, 0, INV), (6, 8, INV), (6, 24, INV), (6, 4112, INV), (7, 0, UNS), (7, 101, UNS), (8, 2, UNS),
             (8, -1, UNS)]
    for k, v, want in cases:
        a = list(good)
        a[k] = v
        st = L.amb_cog_jpeg_tiles_device(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8],
                                         buf.ctypes.data if a[9] else None, len(buf),
                                         C.byref(size) if a[11] else None, cnt.ctypes.data if a[10] else None)
        assert st == want, (k, v, st)
    # mask: (ctx, image, w, h, stride, tile, out, counts, size)
    good = [ctx, d.ptr, 9, 9, 9, 16, True, True, True]
    for k, v in ((0, None), (1, None), (6, False), (7, False), (8, False), (2, 0), (3, -1), (4, 8), (5, 8), (5, 4112)):
        a = list(good)
        a[k] = v
        st = L.amb_cog_mask_tiles_device(a[0], a[1], a[2], a[3], a[4], a[5], buf.ctypes.data if a[6] else None,
                                         len(buf), C.byref(size) if a[8] else None, cnt.ctypes.data if a[7] else None)
        assert st == INV, (k, v, st)
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable()
    gm.to_device(0)
    gc = gm.context()
    for layer, fmt, tile, q, s, want in ((-1, 1, 16, 75, 0, INV), (len(_lib.LAYER_NAMES), 1, 16, 75, 0, INV),
                                         (0, 0, 16, 75, 0, INV), (0, 3, 16, 75, 0, INV), (0, 1, 40, 75, 0, INV),
                                         (0, 1, 16, 0, 0, UNS), (0, 2, 16, 75, 5, UNS)):
        assert L.amb_export_cog_jpeg_tiles(gc, layer, fmt, tile, q, s, buf.ctypes.data, len(buf), C.byref(size),
                                           cnt.ctypes.data) == want
    for layer, tile in ((-1, 16), (len(_lib.LAYER_NAMES), 16), (0, 40)):
        assert L.amb_export_cog_mask_tiles(gc, layer, tile, buf.ctypes.data, len(buf), C.byref(size),
                                           cnt.ctypes.data) == INV
    gm.sync()
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    for kw in ({"compress": "lzw"}, {"compress": "jpeg", "fmt": "f32"}, {"compress": "jpeg", "fmt": "mask8"},
               {"compress": "jpeg", "quality": 0}, {"compress": "jpeg", "sampling": "422"},
               {"compress": "jpeg", "nodata": 0}, {"mask": "observation_index", "fmt": "f32"},
               {"mask": "no_such_layer"}):
        with pytest.raises(ValueError):
            gm.to_cog("unused.tif", "ortho", **kw)
    assert not os.path.exists("unused.tif")


# ---- files of map layers ---------------------------------------------------------------------------------------------------
@gpu
def test_map_files_hold_the_tiles_and_the_mask(tmp_path):
    gm = mapping_run()
    gm.sync()
    m8 = gm.to_raster("observation_index", "mask8")
    for name, fmt, sampling in (("ortho", "gray8", "420"), ("colored_ortho", "bgr8", "420"),
                                ("colored_ortho", "bgr8", "444")):
        band = gm.to_raster(name, fmt)
        path = str(tmp_path / ("%s_%s.tif" % (name, sampling)))
        gm.to_cog(path, name, tile_size=16, compress="jpeg", quality=80, sampling=sampling, mask="observation_index")
        data = open(path, "rb").read()
        chain = ifds(data)
        levels = pyramid(band, fmt, 16)
        assert len(chain) == 2 * len(levels) == 8
        tables, want = cv2_tiles(band, fmt, 16, 80, sampling)
        masks = tiles_of(m8, "mask8", 16)
        k = 0
        for lv in range(len(levels) - 1, -1, -1):
            t, mt = chain[2 * lv][2], chain[2 * lv + 1][2]
            assert bytes(t[347]) == tables and t[259] == (7,) and mt[254] == ((4,) if lv == 0 else (5,))
            for (o, n), (mo, mn) in zip(zip(t[324], t[325]), zip(mt[324], mt[325])):
                assert data[o:o + n] == want[k] and mo == o + n
                assert np.array_equal(unpack_mask(data[mo:mo + mn], 16), masks[k] != 0)
                k += 1
        assert k == len(want)
    # a Deflate COG with the mask: the image pages read back as before
    plain, masked = str(tmp_path / "plain.tif"), str(tmp_path / "masked.tif")
    gm.to_cog(plain, "colored_ortho", tile_size=16)
    gm.to_cog(masked, "colored_ortho", tile_size=16, mask="observation_index")
    for k in range(4):
        assert np.array_equal(io.read_geotiff(plain, 1, overview=k)[0], io.read_geotiff(masked, 1, overview=k)[0])


@gpu
def test_a_stripe_writes_its_band_and_export_after_queued_work(tmp_path):
    whole = mapping_run()
    whole.download(("colored_ortho", "observation_index"))
    rows, cols = whole.getSize()
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * 1.0, cols * 1.0, 1.0)).getMutable()
    for name in ("colored_ortho", "observation_index"):
        gm[name] = whole[name].copy(order="F")
    gm.to_device(0, col_range=(13, 40), names=("colored_ortho", "observation_index"))
    band = gm.to_raster("colored_ortho", "bgr8")
    assert band.shape[0] == 27
    L = _lib.lib()
    h, w = band.shape[:2]
    cap = L.amb_cog_jpeg_max_size(w, h, _lib.RASTER_BGR8, 16, 75, 0)
    buf = np.empty(cap, np.uint8)
    counts = np.zeros(sum(-(-a // 16) * -(-b // 16) for a, b in layout(w, h, 16)[1]), np.uint32)
    size = C.c_size_t(0)
    amb.check(L.amb_export_cog_jpeg_tiles(gm.context(), _lib.LAYER_ID["colored_ortho"], _lib.RASTER_BGR8, 16, 75, 0,
                                          buf.ctypes.data, cap, C.byref(size), counts.ctypes.data))
    check_jpeg(band, "bgr8", 16, 75, "420", buf[:size.value].tobytes(), counts)
    # an export queued right after the orthomosaic, without a sync, equals one after it
    gm = mapping_run(120, 96)
    first, second = str(tmp_path / "first.tif"), str(tmp_path / "second.tif")
    gm.to_cog(first, "colored_ortho", tile_size=32, compress="jpeg", mask="observation_index")
    gm.sync()
    gm.to_cog(second, "colored_ortho", tile_size=32, compress="jpeg", mask="observation_index")
    assert open(first, "rb").read() == open(second, "rb").read()


@gpu
def test_torch_wrappers(tmp_path):
    if EMULATED:
        return   # the wrappers take torch CUDA tensors; their C entry points are what every other test here calls
    import torch
    img = smooth("bgr8", 123, 77, seed=4)
    t = torch.from_numpy(img).cuda()
    data, counts, tables = amb.cog_jpeg_tiles(t, "bgr8", tile_size=32, quality=60, sampling="444")
    assert check_jpeg(img, "bgr8", 32, 60, "444", data, counts)[0] == tables
    big = torch.zeros((123, 100, 3), dtype=torch.uint8, device="cuda")
    big[:, :77] = t
    assert amb.cog_jpeg_tiles(big[:, :77], "bgr8", 32, 60, "444")[0] == data
    m = content("mask8", 123, 77, seed=2)
    md, mc = amb.cog_mask_tiles(torch.from_numpy(m).cuda(), tile_size=32)
    check_mask(m, 32, md, mc)
    path = str(tmp_path / "a.tif")
    io.write_cog(path, data, counts, 77, 123, "bgr8", 32, (0.0, 0.5, 0.0, 10.0, 0.0, -0.5), compress="jpeg",
                 jpeg_tables=tables, sampling="444", mask=(md, mc))
    assert len(ifds(open(path, "rb").read())) == 2 * len(layout(77, 123, 32)[1])
    for bad in ((t, "f32", 32), (t, "bgr8", 20), (t[:, ::2], "bgr8", 32), (t.float(), "bgr8", 32)):
        with pytest.raises(ValueError):
            amb.cog_jpeg_tiles(*bad)
    with pytest.raises(ValueError):
        amb.cog_jpeg_tiles(t, "bgr8", 32, quality=0)
    with pytest.raises(ValueError):
        amb.cog_mask_tiles(t, 32)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_cog_jpeg.py"], sched=sched, opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
