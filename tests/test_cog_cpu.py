"""Cloud-Optimized GeoTIFF without a GPU: the level rule of amb_cog_layout, the size bound of amb_cog_max_size and the
argument contract, and files io.write_cog writes from tiles compressed here with zlib over a numpy restatement of the
convention (include/aerial_mapper_b200.h, amb_cog_tiles_device): their structure (IFDs first, the smallest level's
data first, offsets increasing and contiguous, NewSubfileType, georeferencing on level 0 only) and every level read
back bit for bit by io.read_geotiff(overview=k), OpenCV and PIL.  tests/test_gpu_cog.py compares the device's tiles with
the same restatement."""
import ctypes as C
import math
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from aerial_mapper_b200 import _lib, io  # noqa: E402

FORMATS = ("f32", "gray8", "bgr8", "mask8")
BPP = {"f32": 4, "gray8": 1, "bgr8": 3, "mask8": 1}
QNAN = np.uint32(0x7FC00000).view(np.float32)


# ---- the restatement ----------------------------------------------------------------------------------------------------
def layout(w, h, tile):
    n = C.c_int32(0)
    lw, lh = (C.c_int32 * 32)(), (C.c_int32 * 32)()
    st = _lib.lib().amb_cog_layout(w, h, tile, C.byref(n), lw, lh)
    return st, [(lw[k], lh[k]) for k in range(n.value)]


def reduce(img, fmt):
    """Level k + 1 from level k: the children (2y + a, 2x + b) inside the level, in the order (0,0), (0,1), (1,0), (1,1)."""
    h, w = img.shape[:2]
    h2, w2 = -(-h // 2), -(-w // 2)
    kids = []
    for a in (0, 1):
        for b in (0, 1):
            part = img[a::2, b::2]
            present = np.zeros((h2, w2), bool)
            present[:part.shape[0], :part.shape[1]] = True
            full = np.zeros((h2, w2) + img.shape[2:], img.dtype)
            full[:part.shape[0], :part.shape[1]] = part
            kids.append((full, present))
    if fmt == "f32":
        s = np.zeros((h2, w2), np.float64)
        n = np.zeros((h2, w2), np.int64)
        with np.errstate(invalid="ignore", over="ignore"):
            for v, present in kids:
                v = v.astype(np.float64)
                ok = present & ~np.isnan(v)
                s = np.where(ok & (n == 0), v, np.where(ok, s + v, s))   # IEEE double, rounded, no FMA
                n += ok
            out = (s / np.maximum(n, 1)).astype(np.float32)
        out[(n == 0) | np.isnan(out)] = QNAN
        return out
    if fmt == "mask8":
        return np.max([np.where(p, v, 0) for v, p in kids], axis=0).astype(np.uint8)
    s = np.zeros((h2, w2) + img.shape[2:], np.int64)
    n = np.zeros((h2, w2), np.int64)
    for v, present in kids:
        s += np.where(present[..., None] if img.ndim == 3 else present, v.astype(np.int64), 0)
        n += present
    nn = n[..., None] if img.ndim == 3 else n
    return ((s + nn // 2) // nn).astype(np.uint8)


def pyramid(img, fmt, tile):
    levels = [img]
    for _ in layout(img.shape[1], img.shape[0], tile)[1][1:]:
        levels.append(reduce(levels[-1], fmt))
    return levels


def predict(img, fmt):
    """The TIFF predictor of the convention, per row: uint8 [H, row_bytes]."""
    h = img.shape[0]
    if fmt == "f32":
        w = img.shape[1]
        be = np.ascontiguousarray(img, np.float32).astype(">f4").view(np.uint8).reshape(h, w, 4)
        b = np.ascontiguousarray(be.transpose(0, 2, 1)).reshape(h, 4 * w)
        step = 1
    else:
        b = np.ascontiguousarray(img[:, :, ::-1] if fmt == "bgr8" else img).reshape(h, -1)
        step = 3 if fmt == "bgr8" else 1
    d = b.copy()
    d[:, step:] = b[:, step:] - b[:, :-step]
    return d


def predicted_tiles(img, fmt, tile):
    """Every tile's predicted bytes, in file order: the smallest level first, row-major within a level, edge tiles
    padded with zero bytes."""
    out = []
    for lv in pyramid(img, fmt, tile)[::-1]:
        h, w = lv.shape[:2]
        for ty in range(-(-h // tile)):
            for tx in range(-(-w // tile)):
                t = np.zeros((tile, tile) + lv.shape[2:], lv.dtype)
                part = lv[ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile]
                if fmt == "f32":   # zero bytes, not the value 0.0 of the sample type (the same bits)
                    t = np.zeros((tile, tile), np.uint32).view(np.float32)
                t[:part.shape[0], :part.shape[1]] = part
                out.append(predict(t, fmt).tobytes())
    return out


def bound(n):
    return n + 5 * ((n + 65534) // 65535) + 6


def content(fmt, h, w, seed):
    rng = np.random.default_rng(seed)
    if fmt == "f32":
        a = (np.add.outer(np.arange(h) * 0.37, np.arange(w) * 0.11) + rng.normal(0, 0.05, (h, w))).astype(np.float32)
        a[rng.random((h, w)) < 0.2] = np.nan
        return a
    if fmt == "mask8":
        return np.where(rng.random((h, w)) < 0.2, 0, 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w, 3) if fmt == "bgr8" else (h, w)).astype(np.uint8)


# ---- COG structure ------------------------------------------------------------------------------------------------------
def ifds(data):
    """[(offset, size in bytes with its out-of-line values, tags)] of the IFD chain."""
    out, at = [], struct.unpack_from("<I", data, 4)[0]
    while at:
        n = struct.unpack_from("<H", data, at)[0]
        tags = io._read_ifd(data, at)
        ends = [at + 2 + 12 * n + 4]
        for e in range(n):
            tag, typ, count, raw = struct.unpack_from("<HHI4s", data, at + 2 + 12 * e)
            size = struct.calcsize("<" + io._TIFF_TYPES[typ]) * count
            if size > 4:
                ends.append(struct.unpack("<I", raw)[0] + size)
        out.append((at, max(ends) - at, tags))
        at = struct.unpack_from("<I", data, at + 2 + 12 * n)[0]
    return out


def check_cog_structure(path, w, h, tile, fmt):
    data = open(path, "rb").read()
    chain = ifds(data)
    levels = layout(w, h, tile)[1]
    assert len(chain) == len(levels)
    assert chain[0][0] == 8                                                  # level 0's IFD right after the header
    first_tile = min(min(t[324]) for _, _, t in chain)
    assert all(at + size <= first_tile for at, size, _ in chain)             # every IFD and its arrays before the data
    for k, ((at, size, t), (lw, lh)) in enumerate(zip(chain, levels)):
        assert (t[256][0], t[257][0]) == (lw, lh)
        assert t[254] == (0 if k == 0 else 1,)
        assert t[322] == (tile,) and t[323] == (tile,) and t[259] == (8,)
        assert t[317] == ((3,) if fmt == "f32" else (2,))
        assert len(t[324]) == len(t[325]) == -(-lw // tile) * -(-lh // tile)
        geo = {33550, 33922, 34735, 42113} & set(t)
        assert (k == 0) == bool(geo & {33550, 33922, 34735}), k
        if k > 0:
            assert not geo
        if k > 0:                                                            # IFDs decrease in size
            pw, ph = levels[k - 1]
            assert lw <= pw and lh <= ph and lw * lh < pw * ph
    # data: the smallest level first, offsets increasing and contiguous
    at = (chain[-1][0] + chain[-1][1] + 15) & ~15
    for _, _, t in chain[::-1]:
        for off, n in zip(t[324], t[325]):
            assert off == at
            at += n
    assert at == len(data)


def write_numpy_cog(path, img, fmt, tile, gt=(500000.0, 0.5, 0.0, 5300000.0, 0.0, -0.5), nodata=None):
    tiles = [zlib.compress(p, 6) for p in predicted_tiles(img, fmt, tile)]
    io.write_cog(path, b"".join(tiles), [len(t) for t in tiles], img.shape[1], img.shape[0], fmt, tile, gt,
                 nodata=nodata)
    return tiles


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def read_level(path, k, fmt):
    if fmt == "bgr8":
        return np.stack([io.read_geotiff(path, band=c, overview=k)[0] for c in (2, 1, 0)], axis=-1)
    return io.read_geotiff(path, overview=k)[0]


# ---- the level rule and the size bound -----------------------------------------------------------------------------------
def test_levels_follow_gdal_size_rule_and_stop_at_one_tile():
    for tile in (16, 48, 512, 4096):
        sizes = sorted({1, 2, tile - 1, tile, tile + 1, 2 * tile, 2 * tile + 1, 3 * tile + 5, 65535})
        for w in sizes:
            for h in sizes:
                st, lv = layout(w, h, tile)
                assert st == 0
                want = [(w, h)]
                k = 1
                while want[-1][0] > tile or want[-1][1] > tile:
                    want.append((math.ceil(w / 2 ** k), math.ceil(h / 2 ** k)))
                    k += 1
                assert lv == want, (tile, w, h)
    assert layout(2 ** 31 - 1, 1, 16)[1][-1] == (16, 1) and len(layout(2 ** 31 - 1, 1, 16)[1]) == 28


def test_max_size_and_the_argument_contract():
    L = _lib.lib()
    for fmt in FORMATS:
        f = _lib.RASTER_FORMAT[fmt]
        for (w, h, tile) in ((1, 1, 16), (37, 17, 16), (513, 1025, 512), (10000, 10000, 512), (65535, 3, 4096)):
            lv = layout(w, h, tile)[1]
            n = sum(-(-a // tile) * -(-b // tile) for a, b in lv)
            assert L.amb_cog_max_size(w, h, f, tile) == n * bound(tile * tile * BPP[fmt]), (fmt, w, h, tile)
    INV = _lib.AMB_ERR_INVALID_ARGUMENT
    for tile in (0, 8, 24, 4112, -16, 4095):
        assert layout(100, 100, tile)[0] == INV, tile
        assert L.amb_cog_max_size(100, 100, 0, tile) == 0, tile
    for w, h in ((0, 5), (5, 0), (-1, 5)):
        assert layout(w, h, 16)[0] == INV and L.amb_cog_max_size(w, h, 0, 16) == 0
    assert L.amb_cog_max_size(9, 9, 4, 16) == 0 and L.amb_cog_max_size(9, 9, -1, 16) == 0
    n = C.c_int32(0)
    lw = (C.c_int32 * 32)()
    assert L.amb_cog_layout(9, 9, 16, None, lw, lw) == INV and L.amb_cog_layout(9, 9, 16, C.byref(n), None, lw) == INV
    # more tile rows than an int32 counts: unsupported, bound 0
    assert L.amb_cog_max_size(2 ** 31 - 1, 2 ** 31 - 1, 1, 16) == 0
    assert L.amb_cog_max_size(2 ** 31 - 1, 16, 1, 16) == 0 and L.amb_cog_max_size(2 ** 26, 16, 1, 16) > 0


def test_restatement_rules_at_edge_values():
    # F32: NaN children are left out, -0 survives as the sum's start, +inf and -inf give the quiet NaN, payloads vanish
    nan_payload = np.uint32(0x7FA00001).view(np.float32)
    neg_nan = np.uint32(0xFFC00123).view(np.float32)
    inf = np.float32(np.inf)
    img = np.array([[np.nan, np.nan, 1.0, np.nan, -0.0, -0.0, inf, 3.0, inf, 1.0, nan_payload, 2.5],
                    [np.nan, np.nan, np.nan, np.nan, -0.0, nan_payload, -inf, 1.0, inf, neg_nan, neg_nan, 0.5]],
                   np.float32)
    got = reduce(img, "f32").view(np.uint32)[0]
    want = np.array([QNAN, 1.0, -0.0, QNAN, inf, 1.5], np.float32).view(np.uint32)
    assert np.array_equal(got, want), [hex(v) for v in got]
    # 8-bit: (sum + n / 2) / n on the children that exist
    g = np.array([[0, 1, 1, 2, 0, 0, 255, 254, 7], [1, 1, 2, 2, 0, 1, 255, 255, 8]], np.uint8)
    assert reduce(g, "gray8").tolist() == [[1, 2, 0, 255, 8]]
    m = np.array([[0, 0, 255, 0, 0], [0, 0, 0, 0, 255]], np.uint8)
    assert reduce(m, "mask8").tolist() == [[0, 255, 255]]


# ---- files of numpy-compressed tiles ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_numpy_cogs_have_the_structure_and_read_back_at_every_level(fmt, tmp_path):
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    for (h, w, tile) in ((1, 1, 16), (37, 1, 16), (67, 45, 16), (33, 17, 32), (100, 130, 32)):
        img = content(fmt, h, w, seed=h * w)
        path = str(tmp_path / ("%s_%d_%d.tif" % (fmt, h, w)))
        gt = (500000.0, 0.5, 0.0, 5300000.0, 0.0, -0.5)
        write_numpy_cog(path, img, fmt, tile, gt, nodata="nan" if fmt == "f32" else (0 if fmt == "mask8" else None))
        check_cog_structure(path, w, h, tile, fmt)
        levels = pyramid(img, fmt, tile)
        ok, pages = cv2.imreadmulti(path, flags=cv2.IMREAD_UNCHANGED)
        assert ok and len(pages) == len(levels)
        im = Image.open(path)
        for k, lv in enumerate(levels):
            _, g, epsg, nodata = io.read_geotiff(path, overview=k)
            assert same_bits(read_level(path, k, fmt), lv), (fmt, h, w, k)
            assert g == (gt[0], gt[1] * w / lv.shape[1], 0.0, gt[3], 0.0, gt[5] * h / lv.shape[0])
            assert epsg == 32632 and ((nodata is None) == (fmt in ("gray8", "bgr8")))
            assert same_bits(pages[k], lv), ("cv2", fmt, k)
            im.seek(k)
            p = np.asarray(im)
            assert same_bits(p[:, :, ::-1] if fmt == "bgr8" else p, lv), ("PIL", fmt, k)
        with pytest.raises(ValueError):
            io.read_geotiff(path, overview=len(levels))
        with pytest.raises(ValueError):
            io.read_geotiff(path, overview=-1)


def test_level_zero_reads_as_before_and_strip_files_have_no_overviews(tmp_path):
    img = content("f32", 40, 50, seed=3)
    path = str(tmp_path / "plain.tif")
    io.write_geotiff(path, img, (0.0, 1.0, 0.0, 10.0, 0.0, -1.0), nodata="nan")
    assert same_bits(io.read_geotiff(path, overview=0)[0], img)
    assert io.read_geotiff(path, overview=0)[1:3] == io.read_geotiff(path)[1:3]
    with pytest.raises(ValueError):
        io.read_geotiff(path, overview=1)


def test_nodata_must_agree_with_the_reduction(tmp_path):
    path = str(tmp_path / "n.tif")
    for fmt, good, bad in (("f32", (None, "nan", "NaN", float("nan"), np.float32("nan")), ("0", 0, -9999.0, "inf")),
                           ("mask8", (None, 0, 0.0), ("0", 255, 1, "nan", float("nan"), True)),
                           ("gray8", (None,), (0, "nan", 255)), ("bgr8", (None,), (0, "nan"))):
        img = content(fmt, 20, 20, seed=1)
        for v in good:
            write_numpy_cog(path, img, fmt, 16, nodata=v)
            nd = io.read_geotiff(path)[3]
            assert (nd is None) == (v is None) and (v is None or (math.isnan(nd) if fmt == "f32" else nd == 0))
        os.remove(path)
        for v in bad:
            with pytest.raises(ValueError):
                write_numpy_cog(path, img, fmt, 16, nodata=v)
            assert not os.path.exists(path)


def test_write_cog_argument_checks(tmp_path):
    img = content("gray8", 40, 40, seed=2)
    tiles = [zlib.compress(p) for p in predicted_tiles(img, "gray8", 16)]
    path = str(tmp_path / "x.tif")
    data = b"".join(tiles)
    counts = [len(t) for t in tiles]
    gt = (0.0, 1.0, 0.0, 0.0, 0.0, -1.0)
    with pytest.raises(ValueError):
        io.write_cog(path, data, counts[:-1], 40, 40, "gray8", 16, gt)
    with pytest.raises(ValueError):
        io.write_cog(path, data + b"x", counts, 40, 40, "gray8", 16, gt)
    with pytest.raises(ValueError):
        io.write_cog(path, data, counts, 40, 40, "gray8", 24, gt)
    with pytest.raises(ValueError):
        io.write_cog(path, data, counts, 40, 40, "gray8", 16, (0.0, 1.0, 0.5, 0.0, 0.0, -1.0))
    assert not os.path.exists(path)
