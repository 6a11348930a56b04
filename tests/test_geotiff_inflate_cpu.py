"""The host half of the device TIFF import (io.tiff_layout, read_geotiff_device, GridMap.from_geotiff; convention in
include/aerial_mapper_b200.h, amb_tiff_decode_device), no GPU: the layout helper against read_geotiff on every kind of
file the GPU tests decode, and the test writer of those tests (numpy predictors, zlib.compressobj, hand-made dynamic
blocks) against zlib.decompress and read_geotiff."""
import struct
import zlib

import numpy as np
import pytest

from aerial_mapper_b200 import io

try:
    import cv2
except ImportError:
    cv2 = None

DTYPES = (np.uint8, np.int16, np.uint16, np.int32, np.float32, np.float64)
_FORMAT = {"u": 1, "i": 2, "f": 3}


# ---- the test writer ------------------------------------------------------------------------------------------------
def predict(a, predictor):
    """The predicted bytes of rows a [rows, cols, spp] (TIFF Predictor 1, 2 or 3), little-endian samples."""
    rows, cols, spp = a.shape
    if predictor == 3:
        item = a.dtype.itemsize
        be = a.astype(a.dtype.newbyteorder(">")).view(np.uint8).reshape(rows, cols * spp, item)
        planes = be.transpose(0, 2, 1).reshape(rows, item * cols * spp)
        d = planes.copy()
        d[:, spp:] = planes[:, spp:] - planes[:, :-spp]
        return d.tobytes()
    a = a.astype(a.dtype.newbyteorder("<"))
    if predictor == 2:
        u = a.view(np.dtype("<u%d" % a.dtype.itemsize))
        d = u.copy()
        d[:, 1:] = u[:, 1:] - u[:, :-1]
        return d.tobytes()
    return a.tobytes()


def zstream(raw, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=0):
    """A zlib stream of raw; flushes > 0 cuts it with that many Z_FULL_FLUSHes (each an empty stored block)."""
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    if flushes:
        parts = np.array_split(np.frombuffer(raw, np.uint8), flushes + 1)
        out = b"".join(c.compress(p.tobytes()) + (c.flush(zlib.Z_FULL_FLUSH) if k < flushes else b"")
                       for k, p in enumerate(parts))
        return out + c.flush()
    return c.compress(raw) + c.flush()


class _BitWriter(object):
    def __init__(self):
        self.bits = []

    def put(self, v, n):              # LSB first
        self.bits += [(v >> k) & 1 for k in range(n)]

    def code(self, c, n):             # a Huffman code, most significant bit first
        self.bits += [(c >> (n - 1 - k)) & 1 for k in range(n)]

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(int("".join(map(str, b[k:k + 8][::-1])), 2) for k in range(0, len(b), 8))


def canonical(lens):
    """Codes of a canonical Huffman code (RFC 1951 3.2.2)."""
    count = [0] * 16
    for l in lens:
        if l:
            count[l] += 1
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lens:
        out.append(nxt[l] if l else None)
        if l:
            nxt[l] += 1
    return out


def dynamic_stream(data, dist="none", junk=b"", cl=None, lit=None):
    """A zlib stream of one hand-made dynamic block: every byte of `data` a literal, except that with dist="single" (a
    distance code of one length-1 code) each byte repeated three times after itself is one distance-1 match.  Literal /
    length lengths: 8 for 0..253, 10 for 254..261, 0 for 262..271; the lengths are run-length coded so that a code-18
    run crosses from the literal / length lengths into the distance lengths.  cl / lit replace the code-length code's
    lengths (19, in symbol order) or the literal / length lengths (272), e.g. to make a code over-subscribed."""
    nlen = 272
    lit = list(lit) if lit is not None else [8] * 254 + [10] * 8 + [0] * 10
    dl = [1, 0, 0] if dist == "single" else [0, 0, 0]
    seq = lit + dl
    cl = list(cl) if cl is not None else [4] * 13 + [5] * 6   # a complete code-length code over all 19 symbols
    cl_codes = canonical(cl)
    w = _BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    w.put(nlen - 257, 5)
    w.put(len(dl) - 1, 5)
    w.put(19 - 4, 4)
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    for s in order:
        w.put(cl[s], 3)
    k = 0
    while k < len(seq):
        v = seq[k]
        run = 1
        while k + run < len(seq) and seq[k + run] == v:
            run += 1
        if v == 0 and run >= 11:
            r = min(run, 138)
            w.code(cl_codes[18], cl[18])
            w.put(r - 11, 7)
        elif v == 0 and run >= 3:
            r = min(run, 10)
            w.code(cl_codes[17], cl[17])
            w.put(r - 3, 3)
        elif run >= 4:
            w.code(cl_codes[v], cl[v])
            r = 1 + min(run - 1, 6)
            w.code(cl_codes[16], cl[16])
            w.put(r - 1 - 3, 2)
        else:
            r = 1
            w.code(cl_codes[v], cl[v])
        k += r
    lc = canonical(lit)
    out = bytearray()
    i = 0
    while i < len(data):
        if dist == "single" and i > 0 and data[i] == data[i - 1] and i + 2 < len(data) and \
                data[i + 1] == data[i] and data[i + 2] == data[i]:
            w.code(lc[257], lit[257])                 # length 3
            w.code(0, 1)                              # distance code 0: distance 1
            out += data[i:i + 3]
            i += 3
            continue
        b = data[i]
        w.code(lc[b], lit[b])
        out.append(b)
        i += 1
    w.code(lc[256], lit[256])
    assert bytes(out) == bytes(data)
    return b"\x78\x9c" + w.bytes() + struct.pack(">I", zlib.adler32(bytes(data))) + junk


def fixed_stream(symbols, data=b""):
    """A zlib stream of one fixed-Huffman block of the given literal / length and distance symbols, each (code, extra
    value, extra bits) with code < 288 a literal / length symbol, ("d", code, extra value, extra bits) a distance code;
    the Adler-32 of `data` (the bytes the symbols stand for)."""
    w = _BitWriter()
    w.put(1, 1)
    w.put(1, 2)
    for s in symbols:
        if s[0] == "d":
            w.code(s[1], 5)
            if len(s) > 2:
                w.put(s[2], s[3])
            continue
        c = s[0]
        if c < 144:
            w.code(0x30 + c, 8)
        elif c < 256:
            w.code(0x190 + c - 144, 9)
        elif c < 280:
            w.code(c - 256, 7)
        else:
            w.code(0xC0 + c - 280, 8)
        if len(s) > 1:
            w.put(s[1], s[2])
    return b"\x78\x9c" + w.bytes() + struct.pack(">I", zlib.adler32(bytes(data)))


_LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
             258]
_LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
_DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
              6145, 8193, 12289, 16385, 24577]
_DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]


def match_stream(parts):
    """(zlib stream, the bytes it inflates to) of one fixed-Huffman block of `parts`: bytes (literals) or (length,
    distance) matches, any distance up to 32768 (code 29, extra 8191).  A distance past the output so far is written as
    asked for, and the bytes returned then stop before it."""
    syms, out, ok = [], bytearray(), True
    for p in parts:
        if isinstance(p, (bytes, bytearray)):
            syms += [(b,) for b in p]
            out += p
            continue
        length, dist = p
        lc = max(k for k in range(29) if _LEN_BASE[k] <= length and (k < 28 or length == 258))
        dc = max(k for k in range(30) if _DIST_BASE[k] <= dist)
        syms += [(257 + lc, length - _LEN_BASE[lc], _LEN_EXTRA[lc]),
                 ("d", dc, dist - _DIST_BASE[dc], _DIST_EXTRA[dc])]
        ok = ok and dist <= len(out)
        if ok:
            for _ in range(length):
                out.append(out[-dist])
    return fixed_stream(syms + [(256,)], out), bytes(out)


def corrupt_streams(raw):
    """(name, stream) of every class of stream zlib.decompress rejects, for a chunk whose bytes are `raw`."""
    s = zstream(raw)
    stored = zstream(raw, 0)
    data = bytes(raw[:600])
    out = [("header_check", bytes([s[0], s[1] ^ 1]) + s[2:]),
           ("method_7", b"\x77\x85" + s[2:]),               # CM 7, FCHECK valid
           ("window_64k", b"\x88\x98" + s[2:]),             # CINFO 8, FCHECK valid
           ("preset_dictionary", b"\x78\xbb" + s[2:]),      # FDICT, FCHECK valid
           ("block_type_3", b"\x78\x9c\x07\x00\x00\x00\x00\x00"),
           ("stored_length", stored[:5] + bytes([stored[5] ^ 1]) + stored[6:]),
           ("oversubscribed_cl", dynamic_stream(data, cl=[4] * 14 + [5] * 5)),
           ("incomplete_cl", dynamic_stream(data, cl=[4] * 12 + [5] * 6 + [0])),
           ("incomplete_lit", dynamic_stream(data, lit=[8] * 254 + [10] * 7 + [0] * 11)),
           ("oversubscribed_lit", dynamic_stream(data, lit=[8] * 254 + [10] * 9 + [0] * 9)),
           ("distance_before_start", fixed_stream([(257,), ("d", 0), (256,)])),
           ("distance_too_far", fixed_stream([(65,), (257,), ("d", 1), (256,)])),
           ("distance_code_30", fixed_stream([(65,), (257,), ("d", 30), (256,)])),
           ("length_code_286", fixed_stream([(65,), (286,), (256,)])),
           ("truncated_half", s[:len(s) // 2]),
           ("truncated_adler", s[:-1]),
           ("empty", b""),
           ("adler", s[:-1] + bytes([s[-1] ^ 0x40])),
           ("too_few_bytes", zstream(raw[:-1]))]
    for name, b in out:
        with pytest.raises(zlib.error) if name != "too_few_bytes" else _no_error():
            zlib.decompress(b)
    return out


class _no_error(object):
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


def chunk_streams(a, predictor, chunk, encode):
    """The chunks of a [H, W, spp] (strips ("strips", rps) or tiles ("tiles", tw, th)), each predicted and passed to
    encode(raw_bytes, k)."""
    H, W, spp = a.shape
    out = []
    if chunk[0] == "strips":
        rps = chunk[1]
        for k, r in enumerate(range(0, H, rps)):
            out.append(encode(predict(a[r:r + rps], predictor), k))
    else:
        tw, th = chunk[1], chunk[2]
        k = 0
        for r in range(0, H, th):
            for c in range(0, W, tw):
                t = np.zeros((th, tw, spp), a.dtype)
                part = a[r:r + th, c:c + tw]
                t[:part.shape[0], :part.shape[1]] = part
                out.append(encode(predict(t, predictor), k))
                k += 1
    return out


def make_tiff(a, predictor=1, chunk=("strips", 16), compression=8, encode=None, gt=None, nodata=None, shuffle=False):
    """A classic little-endian TIFF of a [H, W] or [H, W, spp]: encode(raw, k) -> chunk bytes (by default zlib level 6;
    the raw bytes for compression 1); gt: a north-up geotransform for ModelPixelScale + ModelTiepoint; shuffle: the
    chunks stored in reverse order."""
    a = np.asarray(a)
    if a.ndim == 2:
        a = a[:, :, None]
    H, W, spp = a.shape
    if encode is None:
        encode = (lambda raw, k: raw) if compression == 1 else (lambda raw, k: zstream(raw))
    chunks = chunk_streams(a, predictor, chunk, encode)
    fmt = _FORMAT[a.dtype.kind]
    bits = a.dtype.itemsize * 8
    if chunk[0] == "strips":
        layout = [(273, io._LONG, [0] * len(chunks)), (278, io._LONG, [chunk[1]]),
                  (279, io._LONG, [len(c) for c in chunks])]
        off_tag = 273
    else:
        layout = [(322, io._LONG, [chunk[1]]), (323, io._LONG, [chunk[2]]), (324, io._LONG, [0] * len(chunks)),
                  (325, io._LONG, [len(c) for c in chunks])]
        off_tag = 324
    tags = [(256, io._LONG, [W]), (257, io._LONG, [H]), (258, io._SHORT, [bits] * spp),
            (259, io._SHORT, [compression]), (262, io._SHORT, [1]), (277, io._SHORT, [spp]), (284, io._SHORT, [1]),
            (317, io._SHORT, [predictor]), (339, io._SHORT, [fmt] * spp)] + layout
    if gt is not None:
        tags += [(33550, io._DOUBLE, [gt[1], -gt[5], 0.0]), (33922, io._DOUBLE, [0.0, 0.0, 0.0, gt[0], gt[3], 0.0]),
                 (34735, io._SHORT, [1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32632])]
        if nodata is not None:
            tags.append((42113, io._ASCII, ("%s" % nodata).encode("ascii") + b"\0"))
    tags = sorted(tags, key=lambda t: t[0])
    data_at = (8 + io._ifd_size(tags) + 15) & ~15
    order = list(range(len(chunks)))[::-1] if shuffle else list(range(len(chunks)))
    offsets, at = [0] * len(chunks), data_at
    for k in order:
        offsets[k] = at
        at += len(chunks[k])
    tags = io._set_tag(tags, off_tag, io._LONG, offsets)
    head = b"II*\0" + struct.pack("<I", 8) + io._ifd(tags, 8)
    return head + b"\0" * (data_at - len(head)) + b"".join(chunks[k] for k in order)


def sample_raster(dtype, h, w, spp=1, seed=0):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt.kind == "f":
        y, x = np.mgrid[0:h, 0:w]
        base = 400 + 30 * np.sin(x / 7.0) * np.cos(y / 9.0)
        a = np.stack([base + k + rng.normal(0, 0.05, (h, w)) for k in range(spp)], -1).astype(dt)
        a.reshape(-1)[::37] = np.nan
        a.reshape(-1)[5::41] = -0.0
        if dt == np.float64:
            a.reshape(-1)[7::53] = 1e300        # overflows float32
            a.reshape(-1)[9::59] = 1.0 + 2.0 ** -30   # rounds to nearest even
        return a
    info = np.iinfo(dt)
    return rng.integers(info.min, int(info.max) + 1, (h, w, spp), dtype=np.int64).astype(dt)


def ref(data, band=0, overview=0, path=None):
    """read_geotiff(...)[0] of the file's bytes."""
    import os
    import tempfile
    fd, p = tempfile.mkstemp(suffix=".tif")
    try:
        with os.fdopen(fd, "wb") as f:
            f.write(data)
        return read_array(p, band, overview)
    finally:
        os.unlink(p)


def read_array(path, band=0, overview=0):
    """read_geotiff's array of a file that may have no georeferencing: the decode loop of read_geotiff over
    tiff_layout."""
    with open(path, "rb") as f:
        data = f.read()
    t = io.tiff_layout(data, band, overview)
    out = np.empty((t.height, t.width), t.dtype)
    for (r0, c0, rows, cols), at, n in zip(t.grid, t.offsets, t.counts):
        chunk = data[at:at + n]
        if t.compression != 1:
            chunk = zlib.decompress(chunk)
        a = io._undo_predictor(chunk, t.predictor, t.dtype, rows, cols, t.spp)
        out[r0:r0 + rows, c0:c0 + cols] = a[:t.height - r0, :t.width - c0, band]
    return out


# ---- tests ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("chunk", [("strips", 5), ("tiles", 16, 16)])
def test_the_writer_round_trips_through_read_geotiff(tmp_path, dtype, chunk):
    pred = 3 if np.dtype(dtype).kind == "f" else 2
    a = sample_raster(dtype, 37, 21, spp=2, seed=3)
    gt = (500.0, 0.5, 0.0, 900.0, 0.0, -0.5)
    p = tmp_path / "a.tif"
    p.write_bytes(make_tiff(a, pred, chunk, gt=gt, nodata="nan"))
    for band in (0, 1):
        out, g, epsg, nd = io.read_geotiff(str(p), band)
        assert np.array_equal(out.view(np.uint8), np.ascontiguousarray(a[:, :, band]).view(np.uint8))
        assert g == gt and epsg == 32632 and np.isnan(nd)


def test_the_layout_helper_is_what_read_geotiff_reads(tmp_path):
    a = sample_raster(np.float32, 50, 70)
    gt = (0.0, 1.0, 0.0, 50.0, 0.0, -1.0)
    for chunk in (("strips", 7), ("strips", 50), ("strips", 999), ("tiles", 32, 16)):
        b = make_tiff(a, 3, chunk, gt=gt)
        t = io.tiff_layout(b)
        assert (t.width, t.height, t.spp, t.compression, t.predictor) == (70, 50, 1, 8, 3)
        assert t.tiled == (chunk[0] == "tiles")
        if t.tiled:
            assert (t.chunk_width, t.chunk_height) == (32, 16) and len(t.grid) == 3 * 4
        else:
            assert t.chunk_width == 70 and t.chunk_height == min(chunk[1], 50)
            assert t.grid[-1][2] == 50 - (len(t.grid) - 1) * t.chunk_height   # the last strip short
        p = tmp_path / "a.tif"
        p.write_bytes(b)
        assert np.array_equal(read_array(str(p)).view(np.uint32), io.read_geotiff(str(p))[0].view(np.uint32))
        assert t.georeferencing() == io.read_geotiff(str(p))[1:]
        L = t.c_layout()
        assert L.n_chunks == len(t.grid) and L.sample == 4 and L.tiled == int(t.tiled)


def test_the_layout_helper_raises_read_geotiffs_errors(tmp_path):
    a = sample_raster(np.uint16, 8, 8)
    b = make_tiff(a, 2, ("strips", 4))
    with pytest.raises(ValueError, match="band 1 of 1"):
        io.tiff_layout(b, 1)
    with pytest.raises(ValueError, match="overview 1 requested"):
        io.tiff_layout(b, 0, 1)
    with pytest.raises(ValueError, match="Predictor"):
        io.tiff_layout(make_tiff(a.astype(np.float32), 2, ("strips", 4)))
    with pytest.raises(ValueError, match="big-endian"):
        io.tiff_layout(b"MM" + b[2:])
    # a grid with fewer chunks than the image needs has no device layout
    t = io.tiff_layout(b)
    t.offsets, t.counts = t.offsets[:1], t.counts[:1]
    t.grid = t.grid[:1]
    with pytest.raises(ValueError, match="grid"):
        io.TiffLayout(**dict(t.__dict__, grid=io.tiff_layout(b).grid)).c_layout()


@pytest.mark.parametrize("level", range(10))
@pytest.mark.parametrize("strategy", [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE,
                                      zlib.Z_FIXED])
def test_zlib_streams_of_the_writer(level, strategy):
    raw = predict(sample_raster(np.float32, 20, 40), 3)
    assert zlib.decompress(zstream(raw, level, strategy)) == raw
    assert zlib.decompress(zstream(raw, level, strategy, flushes=3)) == raw


@pytest.mark.parametrize("dist", ["none", "single"])
def test_hand_made_dynamic_blocks(dist):
    rng = np.random.default_rng(1)
    data = bytes(rng.integers(0, 256, 3000).astype(np.uint8)) + b"\x07" * 40
    s = dynamic_stream(data, dist, junk=b"junk")
    assert zlib.decompress(s) == data            # bytes after the stream are ignored, as zlib.decompress does
    assert zlib.decompressobj().decompress(s) == data


def test_zlib_accepts_what_the_convention_accepts_and_rejects_the_rest():
    raw = bytes(range(256)) * 40
    s = zstream(raw)
    assert zlib.decompress(s + b"\x00junk") == raw            # trailing bytes
    assert len(corrupt_streams(raw)) == 19                   # each rejected by zlib.decompress (too_few_bytes: short)
    assert len(zlib.decompress(zstream(raw[:-1]))) < len(raw)


def test_opencv_and_pil_files_through_the_layout_helper(tmp_path):
    if cv2 is None:
        pytest.skip("OpenCV is not installed")
    for dtype in (np.uint8, np.int16, np.uint16, np.int32):
        a = sample_raster(dtype, 33, 45, seed=2)[:, :, 0]
        for comp in (8, 32946):
            ok, b = cv2.imencode(".tiff", a, [cv2.IMWRITE_TIFF_COMPRESSION, comp, cv2.IMWRITE_TIFF_PREDICTOR, 2])
            assert ok
            p = tmp_path / "cv.tif"
            p.write_bytes(b.tobytes())
            t = io.tiff_layout(b.tobytes())
            assert t.compression == comp and t.predictor == 2
            assert np.array_equal(read_array(str(p)), cv2.imread(str(p), cv2.IMREAD_UNCHANGED))
    from PIL import Image
    for dtype in (np.float32, np.int16, np.uint16, np.uint8):   # PIL stores int16 as int32
        a = sample_raster(dtype, 19, 23, seed=4)[:, :, 0]
        if dtype == np.float32:
            a = np.nan_to_num(a)
        p = tmp_path / "pil.tif"
        Image.fromarray(a).save(str(p), compression="tiff_adobe_deflate")
        assert io.tiff_layout(p.read_bytes()).compression == 8
        assert np.array_equal(read_array(str(p)), a)


def test_matches_at_the_largest_distances():
    rng = np.random.default_rng(17)
    lit = bytes(rng.integers(0, 256, 33000).astype(np.uint8))
    s, out = match_stream([lit[:32768], (258, 32768), (258, 32767), (3, 32768), lit[:50]])
    assert zlib.decompress(s) == out and len(out) == 32768 + 519 + 50
    assert out[32768:32768 + 258] == lit[:258] and out[-50:] == lit[:50]
    s, _ = match_stream([lit[:32767], (3, 32768)])            # a distance one byte before the start
    with pytest.raises(zlib.error):
        zlib.decompress(s)
