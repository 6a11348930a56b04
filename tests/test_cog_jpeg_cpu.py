"""JPEG-compressed Cloud-Optimized GeoTIFF with an internal mask, without a GPU: the tables stream of amb_cog_jpeg_tables,
the size bounds and the argument contract, and files io.write_cog writes from tiles made here from OpenCV's encoder (or,
without OpenCV, the committed fixture tests/golden/cog_jpeg_cases.npz that OpenCV made) over the numpy pyramid of
tests/test_cog_cpu.py: their structure (image and mask IFDs alternating, NewSubfileType, JPEG and YCbCr tags, the
smallest level's data first, each image tile followed by its mask tile) and every page read back through PIL / libtiff.
tests/test_gpu_cog_jpeg.py compares the device's tiles with the same restatement."""
import ctypes as C
import io as pyio
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from aerial_mapper_b200 import _lib, api, io  # noqa: E402
from test_cog_cpu import bound, content, ifds, layout, pyramid, write_numpy_cog  # noqa: E402

try:
    import cv2
except ImportError:   # the fixture stands in
    cv2 = None

GOLDEN = os.path.join(HERE, "golden", "cog_jpeg_cases.npz")
SOI, EOI = b"\xff\xd8", b"\xff\xd9"
KINDS = {"gray": ("gray8", "420"), "420": ("bgr8", "420"), "444": ("bgr8", "444")}   # kind -> (fmt, sampling)
FIXTURE_QUALITIES = (50, 75)


# ---- the restatement -------------------------------------------------------------------------------------------------------
def tiles_of(img, fmt, tile):
    """Every T x T tile of the pyramid in file order (the smallest level first, row-major), zero outside the level."""
    out = []
    for lv in pyramid(img, fmt, tile)[::-1]:
        h, w = lv.shape[:2]
        for ty in range(-(-h // tile)):
            for tx in range(-(-w // tile)):
                t = np.zeros((tile, tile) + lv.shape[2:], lv.dtype)
                part = lv[ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile]
                t[:part.shape[0], :part.shape[1]] = part
                out.append(t)
    return out


def segments(jpg):
    """The marker segments of a JPEG file up to and including SOS as [(marker, bytes)], and its entropy-coded data."""
    assert jpg[:2] == SOI and jpg[-2:] == EOI
    out, at = [], 2
    while True:
        m = jpg[at + 1]
        n = struct.unpack(">H", jpg[at + 2:at + 4])[0]
        out.append((m, jpg[at:at + 2 + n]))
        at += 2 + n
        if m == 0xDA:
            return out, jpg[at:-2]


def split_file(jpg):
    """(tables stream, abbreviated tile stream) of a whole JPEG file: SOI + DQT + DHT + EOI, SOI + SOF0 + SOS + data +
    EOI."""
    segs, data = segments(jpg)
    tables = SOI + b"".join(b for m, b in segs if m in (0xDB, 0xC4)) + EOI
    return tables, SOI + b"".join(b for m, b in segs if m in (0xC0, 0xDA)) + data + EOI


def cv2_file(img, quality, sampling):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == "420" else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
    ok, b = cv2.imencode(".jpg", img, params)
    assert ok
    return b.tobytes()


def cv2_tiles(img, fmt, tile, quality, sampling):
    """(tables, [tile streams]) OpenCV's encoder gives for the pyramid's tiles."""
    tables, streams = None, []
    for t in tiles_of(img, fmt, tile):
        tables, s = split_file(cv2_file(t, quality, sampling))
        streams.append(s)
    return tables, streams


def splice(tables, stream):
    """A whole JPEG file from the tables stream and a tile stream: SOI, DQT, DHT, SOF0, SOS, data, EOI."""
    return tables[:-2] + stream[2:]


def mask_tiles(mask8, tile):
    """The 1-bit mask tiles: the MASK8 pyramid's tiles, 1 where not 0, packed most significant bit first, zlib."""
    return [zlib.compress(np.packbits(t != 0, axis=1).tobytes(), 6) for t in tiles_of(mask8, "mask8", tile)]


def unpack_mask(stream, tile):
    return np.unpackbits(np.frombuffer(zlib.decompress(stream), np.uint8).reshape(tile, tile // 8), axis=1) != 0


def fixture():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def case(kind, quality):
    """(image, mask8, tile, tables, tile streams) of the fixture's case: from OpenCV if present, else as committed."""
    g = fixture()
    fmt, sampling = KINDS[kind]
    img = g["bgr"] if fmt == "bgr8" else g["gray"]
    key = "%s_q%d" % (kind, quality)
    if cv2 is not None:
        tables, streams = cv2_tiles(img, fmt, int(g["tile"]), quality, sampling)
    else:
        tables = g[key + "_tables"].tobytes()
        lens = g[key + "_lens"]
        blob = g[key + "_tiles"].tobytes()
        at = np.concatenate([[0], np.cumsum(lens)])
        streams = [blob[at[k]:at[k + 1]] for k in range(len(lens))]
    return img, g["mask"], int(g["tile"]), tables, streams


def write_host_cog(path, kind, quality, with_mask=True):
    img, mask, tile, tables, streams = case(kind, quality)
    fmt, sampling = KINDS[kind]
    m = mask_tiles(mask, tile) if with_mask else None
    io.write_cog(path, b"".join(streams), [len(s) for s in streams], img.shape[1], img.shape[0], fmt, tile,
                 (500000.0, 0.5, 0.0, 5300000.0, 0.0, -0.5), compress="jpeg", jpeg_tables=tables, sampling=sampling,
                 mask=None if m is None else (b"".join(m), [len(t) for t in m]))
    return img, mask, tile, tables, streams


def pil_libtiff():
    """The libtiff PIL bundles, through ctypes, or None."""
    import glob
    try:
        import PIL
    except ImportError:
        return None
    libs = glob.glob(os.path.join(os.path.dirname(os.path.dirname(PIL.__file__)), "pillow.libs", "libtiff*.so*"))
    if not libs:
        return None
    L = C.CDLL(libs[0])
    L.TIFFOpen.restype, L.TIFFOpen.argtypes = C.c_void_p, [C.c_char_p, C.c_char_p]
    L.TIFFSetDirectory.restype, L.TIFFSetDirectory.argtypes = C.c_int, [C.c_void_p, C.c_uint32]
    L.TIFFNumberOfTiles.restype, L.TIFFNumberOfTiles.argtypes = C.c_uint32, [C.c_void_p]
    L.TIFFReadEncodedTile.restype = C.c_ssize_t
    L.TIFFReadEncodedTile.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_ssize_t]
    L.TIFFClose.restype, L.TIFFClose.argtypes = None, [C.c_void_p]
    L.TIFFNumberOfDirectories.restype, L.TIFFNumberOfDirectories.argtypes = C.c_uint32, [C.c_void_p]
    return L


def tiff_tiles(L, path, page, tile):
    """The decoded tiles of a 1-bit page, read by libtiff: [T * T / 8 bytes]."""
    t = L.TIFFOpen(path.encode(), b"r")
    assert t
    try:
        assert L.TIFFSetDirectory(t, page) == 1
        out = []
        for j in range(L.TIFFNumberOfTiles(t)):
            buf = C.create_string_buffer(tile * tile // 8)
            assert L.TIFFReadEncodedTile(t, j, buf, len(buf)) == len(buf)
            out.append(buf.raw)
        return out
    finally:
        L.TIFFClose(t)


# ---- tables and bounds ----------------------------------------------------------------------------------------------------
def lib_tables(channels, quality, capacity=1024):
    buf = np.full(capacity + 1, 0xA5, np.uint8)
    size = C.c_size_t(0)
    st = _lib.lib().amb_cog_jpeg_tables(channels, quality, buf.ctypes.data, capacity, C.byref(size))
    return st, buf, size.value


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("quality", [1, 50, 75, 100])
def test_tables_are_the_dqt_and_dht_of_the_encoder(kind, quality):
    fmt, sampling = KINDS[kind]
    st, buf, n = lib_tables(3 if fmt == "bgr8" else 1, quality)
    assert st == 0 and buf[:2].tobytes() == SOI and buf[n - 2:n].tobytes() == EOI
    assert api.cog_jpeg_tables(fmt, quality) == buf[:n].tobytes()
    if cv2 is not None or quality in FIXTURE_QUALITIES:
        assert buf[:n].tobytes() == case(kind, quality)[3]


def test_tables_argument_contract():
    UNS, INV, SIZE = _lib.AMB_ERR_UNSUPPORTED, _lib.AMB_ERR_INVALID_ARGUMENT, _lib.AMB_ERR_SIZE_MISMATCH
    for ch, q in ((2, 75), (0, 75), (3, 0), (1, 101)):
        st, buf, _ = lib_tables(ch, q)
        assert st == UNS and (buf == 0xA5).all()
    st, buf, n = lib_tables(3, 75)
    st2, buf2, n2 = lib_tables(3, 75, capacity=n - 1)
    assert st2 == SIZE and n2 == n and (buf2 == 0xA5).all()
    size = C.c_size_t(0)
    assert _lib.lib().amb_cog_jpeg_tables(1, 75, None, 100, C.byref(size)) == INV
    assert _lib.lib().amb_cog_jpeg_tables(1, 75, buf.ctypes.data, 100, None) == INV
    for bad in (("rgb8", 75), ("gray8", 0), ("bgr8", 101), ("bgr8", True)):
        with pytest.raises(ValueError):
            api.cog_jpeg_tables(*bad)


def test_max_sizes_bound_the_tiles_and_refuse_bad_arguments():
    L = _lib.lib()
    img, mask, tile, tables, streams = case("420", 75)
    h, w = img.shape[:2]
    assert L.amb_cog_jpeg_max_size(w, h, _lib.RASTER_BGR8, tile, 75, 0) >= sum(len(s) for s in streams)
    n_tiles = sum(-(-a // tile) * -(-b // tile) for a, b in layout(w, h, tile)[1])
    assert L.amb_cog_mask_max_size(w, h, tile) == n_tiles * bound(tile * tile // 8)
    for f, t, q, s in ((_lib.RASTER_F32, 16, 75, 0), (_lib.RASTER_MASK8, 16, 75, 0), (_lib.RASTER_GRAY8, 24, 75, 0),
                       (_lib.RASTER_GRAY8, 16, 0, 0), (_lib.RASTER_BGR8, 16, 101, 0), (_lib.RASTER_BGR8, 16, 75, 2),
                       (_lib.RASTER_BGR8, 16, 75, -1), (5, 16, 75, 0)):
        assert L.amb_cog_jpeg_max_size(w, h, f, t, q, s) == 0, (f, t, q, s)
    for a, b, t in ((0, 5, 16), (5, 0, 16), (5, 5, 8), (5, 5, 4112)):
        assert L.amb_cog_mask_max_size(a, b, t) == 0


# ---- the file ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_ifd_chain_tags_offsets_and_data_order(kind, tmp_path):
    path = str(tmp_path / "a.tif")
    img, mask, tile, tables, streams = write_host_cog(path, kind, 75)
    m = mask_tiles(mask, tile)
    data = open(path, "rb").read()
    chain = ifds(data)
    levels = layout(img.shape[1], img.shape[0], tile)[1]
    assert len(levels) > 2 and len(chain) == 2 * len(levels) and chain[0][0] == 8
    first_tile = min(min(t[324]) for _, _, t in chain)
    assert all(at + size <= first_tile for at, size, _ in chain)
    fmt, sampling = KINDS[kind]
    for k, (lw, lh) in enumerate(levels):
        t, mt = chain[2 * k][2], chain[2 * k + 1][2]
        n = -(-lw // tile) * -(-lh // tile)
        for tags in (t, mt):
            assert (tags[256][0], tags[257][0]) == (lw, lh) and tags[322] == (tile,) and tags[323] == (tile,)
            assert len(tags[324]) == len(tags[325]) == n and 317 not in tags and 42113 not in tags
        assert t[254] == (0 if k == 0 else 1,) and mt[254] == (4 if k == 0 else 5,)
        assert t[259] == (7,) and bytes(t[347]) == tables
        if fmt == "bgr8":
            assert t[262] == (6,) and t[258] == (8, 8, 8) and t[277] == (3,)
            assert t[530] == ((2, 2) if sampling == "420" else (1, 1))
            assert t[532] == (0, 1, 255, 1, 128, 1, 255, 1, 128, 1, 255, 1)
        else:
            assert t[262] == (1,) and t[258] == (8,) and 530 not in t and 532 not in t
        assert mt[259] == (8,) and mt[262] == (4,) and mt[258] == (1,) and mt[277] == (1,) and 347 not in mt
        assert (k == 0) == (33550 in t) and 33550 not in mt
    # data: the smallest level first; within a level each image tile, then its mask tile; contiguous to the end
    at = (chain[-1][0] + chain[-1][1] + 15) & ~15
    k = 0
    for lv in range(len(levels) - 1, -1, -1):
        t, mt = chain[2 * lv][2], chain[2 * lv + 1][2]
        for (o, n), (mo, mn) in zip(zip(t[324], t[325]), zip(mt[324], mt[325])):
            assert o == at and data[o:o + n] == streams[k] and mo == at + n and data[mo:mo + mn] == m[k]
            at += n + mn
            k += 1
    assert at == len(data) and k == len(streams)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_pil_reads_every_page(kind, tmp_path):
    """Every image page through PIL / libtiff equals OpenCV's decode of the spliced tile streams, every mask page the
    mask.  PIL hands YCbCr JPEG tiles to libjpeg with JPEGCOLORMODE RGB, so libjpeg converts the colours itself, as
    cv2.imdecode does; a difference would be stated here, not hidden by a tolerance."""
    Image = pytest.importorskip("PIL.Image")
    tiff = pil_libtiff()
    path = str(tmp_path / "a.tif")
    img, mask, tile, tables, streams = write_host_cog(path, kind, 75)
    fmt, _ = KINDS[kind]
    levels = layout(img.shape[1], img.shape[0], tile)[1]
    masks = pyramid(mask, "mask8", tile)
    first = np.cumsum([0] + [-(-w // tile) * -(-h // tile) for w, h in levels[::-1]])
    im = Image.open(path)
    if tiff is not None:
        t = tiff.TIFFOpen(path.encode(), b"r")
        assert tiff.TIFFNumberOfDirectories(t) == 2 * len(levels)
        tiff.TIFFClose(t)
    for k, (lw, lh) in enumerate(levels):
        im.seek(2 * k)
        assert im.size == (lw, lh) and im.mode == ("RGB" if fmt == "bgr8" else "L")
        page = np.asarray(im)
        want = np.zeros((-(-lh // tile) * tile, -(-lw // tile) * tile) + page.shape[2:], np.uint8)
        at = first[len(levels) - 1 - k]
        across = -(-lw // tile)
        for j in range(-(-lw // tile) * -(-lh // tile)):
            full = splice(tables, streams[at + j])
            if cv2 is not None:
                d = cv2.imdecode(np.frombuffer(full, np.uint8), cv2.IMREAD_UNCHANGED if fmt == "gray8" else
                                 cv2.IMREAD_COLOR)
                if fmt == "bgr8":
                    d = d[:, :, ::-1]
            else:
                d = np.asarray(Image.open(pyio.BytesIO(full)))
            ty, tx = divmod(j, across)
            want[ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile] = d
        assert np.array_equal(page, want[:lh, :lw]), (kind, k)
        # the mask page: PIL has no mode for Photometric 4, so its tiles are read through PIL's libtiff directly
        if tiff is not None:
            got = tiff_tiles(tiff, path, 2 * k + 1, tile)
            assert len(got) == -(-lw // tile) * -(-lh // tile)
            for j, raw in enumerate(got):
                ty, tx = divmod(j, -(-lw // tile))
                want_m = np.zeros((tile, tile), bool)
                part = masks[k][ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile] != 0
                want_m[:part.shape[0], :part.shape[1]] = part
                bits = np.unpackbits(np.frombuffer(raw, np.uint8).reshape(tile, tile // 8), axis=1) != 0
                assert np.array_equal(bits, want_m), (kind, k, j)


def test_read_geotiff_overviews_skip_the_mask_pages(tmp_path):
    for fmt in ("gray8", "bgr8"):
        img = content(fmt, 70, 90, seed=3)
        mask = content("mask8", 70, 90, seed=4)
        plain, masked = str(tmp_path / "plain.tif"), str(tmp_path / "masked.tif")
        tiles = write_numpy_cog(plain, img, fmt, 16)
        m = mask_tiles(mask, 16)
        io.write_cog(masked, b"".join(tiles), [len(t) for t in tiles], 90, 70, fmt, 16,
                     (500000.0, 0.5, 0.0, 5300000.0, 0.0, -0.5), mask=(b"".join(m), [len(t) for t in m]))
        assert len(ifds(open(masked, "rb").read())) == 2 * len(ifds(open(plain, "rb").read()))
        for k in range(len(layout(90, 70, 16)[1])):
            for band in range(3 if fmt == "bgr8" else 1):
                a, b = io.read_geotiff(plain, band, overview=k), io.read_geotiff(masked, band, overview=k)
                assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
        with pytest.raises(ValueError):
            io.read_geotiff(masked, overview=len(layout(90, 70, 16)[1]))


def test_jpeg_files_are_refused_by_the_reader(tmp_path):
    path = str(tmp_path / "a.tif")
    write_host_cog(path, "gray", 75)
    with pytest.raises(ValueError, match="Compression"):
        io.read_geotiff(path)


def test_write_cog_argument_checks(tmp_path):
    img, mask, tile, tables, streams = case("420", 75)
    h, w = img.shape[:2]
    data, counts = b"".join(streams), [len(s) for s in streams]
    m = mask_tiles(mask, tile)
    good = dict(compress="jpeg", jpeg_tables=tables, sampling="420", mask=(b"".join(m), [len(t) for t in m]))
    gt = (0.0, 1.0, 0.0, 0.0, 0.0, -1.0)
    path = str(tmp_path / "a.tif")
    for change in ({"compress": "lzw"}, {"jpeg_tables": None}, {"jpeg_tables": b"\xff\xd8\xff\xd9"},
                   {"sampling": "422"}, {"mask": (b"".join(m), [len(t) for t in m][:-1])},
                   {"mask": (b"".join(m)[:-1], [len(t) for t in m])}):
        with pytest.raises(ValueError):
            io.write_cog(path, data, counts, w, h, "bgr8", tile, gt, **dict(good, **change))
    with pytest.raises(ValueError):
        io.write_cog(path, data, counts, w, h, "bgr8", tile, gt, nodata=0, **good)
    for fmt in ("f32", "mask8"):
        with pytest.raises(ValueError):
            io.write_cog(path, data, counts, w, h, fmt, tile, gt, **good)
        with pytest.raises(ValueError):
            io.write_cog(path, data, counts, w, h, fmt, tile, gt, mask=good["mask"])
    assert not os.path.exists(path)


def test_fixture_is_what_opencv_writes():
    if cv2 is None:
        pytest.skip("OpenCV is what the fixture records")
    g = fixture()
    for kind in KINDS:
        for q in FIXTURE_QUALITIES:
            img, mask, tile, tables, streams = case(kind, q)
            key = "%s_q%d" % (kind, q)
            assert g[key + "_tables"].tobytes() == tables
            assert g[key + "_tiles"].tobytes() == b"".join(streams)
            assert list(g[key + "_lens"]) == [len(s) for s in streams]
