"""Deflate-compressed GeoTIFF strips on the device (amb_deflate_strips_device, amb_export_deflate_strips,
csrc/deflate_encode.cu; convention in include/aerial_mapper_b200.h): every strip must inflate with zlib to exactly a
numpy restatement of the TIFF predictor, with nothing after its stream, within the stated size bound, and the files
GridMap.to_geotiff writes must read back (io.read_geotiff, OpenCV, PIL) as to_raster of the layer, bit for bit.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels, so the kernel logic is checked on
every CPU run too (the 10000 x 10000 cases and the torch wrapper need a GPU)."""
import ctypes as C
import heapq
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, io, synth  # noqa: E402

gpu = pytest.mark.gpu
EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
CANARY = 0xA5
FORMATS = ("f32", "gray8", "bgr8", "mask8")
SMALL = [(1, 1), (1, 37), (37, 1), (17, 33)]   # (height, width)


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


def from_predicted(p, fmt):
    """The 8-bit raster whose predicted bytes are p (uint8 [H, row_bytes]): to put chosen bytes in front of the coder."""
    step = 3 if fmt == "bgr8" else 1
    h, n = p.shape
    raw = np.cumsum(p.reshape(h, n // step, step), axis=1, dtype=np.uint8).reshape(h, n)
    if fmt == "bgr8":
        return np.ascontiguousarray(raw.reshape(h, n // 3, 3)[:, :, ::-1])
    return raw


def default_rps(row_bytes):
    return max(1, 8192 // row_bytes)


def bound(n):
    return n + 5 * ((n + 65534) // 65535) + 6


class Dev(object):
    """A device copy of `img` with rows `pitch` bytes apart at byte offset `off` from 16-byte alignment."""

    def __init__(self, img, pitch=None, off=0):
        img = np.ascontiguousarray(img)
        h = img.shape[0]
        row = img[0].nbytes
        self.pitch = pitch or row
        host = np.full(64 + off + h * self.pitch + 64, CANARY, np.uint8)
        rows = img.reshape(h, -1).view(np.uint8)
        for r in range(h):
            host[64 + off + r * self.pitch:64 + off + r * self.pitch + row] = rows[r]
        if EMULATED:
            self.raw = host
            self.ptr = host.ctypes.data + 64 + off   # numpy allocations are 16-byte aligned
        else:
            import torch
            self.raw = torch.empty(len(host) + 16, dtype=torch.uint8, device="cuda:0")
            base = (-self.raw.data_ptr()) % 16
            self.raw[base:base + len(host)].copy_(torch.from_numpy(host))
            self.ptr = self.raw.data_ptr() + base + 64 + off


def deflate_dev(d, h, w, fmt, rps, out=None, capacity=None, counts=None):
    L = _lib.lib()
    f = _lib.RASTER_FORMAT[fmt]
    cap = L.amb_deflate_max_size(w, h, f, rps)
    buf = np.empty(max(cap, 1), np.uint8) if out is None else out
    counts = np.zeros(-(-h // min(rps, h)), np.uint32) if counts is None else counts
    size = C.c_size_t(0)
    st = L.amb_deflate_strips_device(api._jpeg_context(0), d.ptr, w, h, d.pitch, f, rps, buf.ctypes.data,
                                     cap if capacity is None else capacity, C.byref(size), counts.ctypes.data)
    return st, buf, size.value, counts


def check_strips(img, fmt, rps, data, counts):
    """Every strip inflates to the predicted rows it covers, with nothing after it, within the bound."""
    pred = predict(img, fmt)
    h = pred.shape[0]
    rps = min(rps, h)
    assert len(counts) == -(-h // rps) and int(np.sum(counts, dtype=np.int64)) == len(data)
    at = 0
    for s, n in enumerate(counts):
        strip = data[at:at + int(n)]
        at += int(n)
        want = pred[s * rps:(s + 1) * rps].tobytes()
        z = zlib.decompressobj()
        got = z.decompress(strip)
        assert z.eof and z.unused_data == b"" and got == want, (fmt, rps, s, len(got), len(want))
        assert len(strip) <= bound(len(want)), (fmt, rps, s, len(strip), len(want))
        assert strip[:2] == b"\x78\x01"


def deflate(img, fmt, rps=None, pitch=None, off=0):
    h, w = img.shape[:2]
    bpp = {"f32": 4, "bgr8": 3}.get(fmt, 1)
    rps = rps or default_rps(w * bpp)
    st, buf, n, counts = deflate_dev(Dev(img, pitch, off), h, w, fmt, rps)
    amb.check(st, api._jpeg_context(0))
    data = buf[:n].tobytes()
    check_strips(img, fmt, rps, data, counts)
    return data, counts


def content(kind, fmt, h, w, seed):
    rng = np.random.default_rng(seed)
    if fmt == "f32":
        if kind == "noise":
            return rng.integers(0, 2 ** 32, (h, w), dtype=np.uint32).view(np.float32)
        a = (synth.analytic_elevation(w, h, 0.25).T + rng.normal(0, 0.05, (h, w))).astype(np.float32)
        a[rng.random((h, w)) < 0.02] = np.nan
        return a
    shape = (h, w, 3) if fmt == "bgr8" else (h, w)
    if kind == "noise":
        return rng.integers(0, 256, shape).astype(np.uint8)
    if fmt == "mask8":
        return np.where(rng.random(shape) < 0.05, 0, 255).astype(np.uint8)
    a = np.add.outer(np.arange(h) * 3, np.arange(w) // 2)
    if fmt == "bgr8":
        a = np.stack([a + 40 * k for k in range(3)], axis=-1)
    return ((a + rng.integers(0, 3, shape)) % 256).astype(np.uint8)


# ---- formats x strip heights x sizes ----------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_every_format_and_strip_height_at_small_sizes(fmt):
    for k, (h, w) in enumerate(SMALL):
        for kind in ("noise", "smooth"):
            img = content(kind, fmt, h, w, seed=k)
            for rps in (1, 7, None, h):
                deflate(img, fmt, rps)


@gpu
@pytest.mark.parametrize("row_bytes", [8191, 8192, 32768, 65535, 65536, 70000])
def test_rows_at_block_and_window_edges(row_bytes):
    for fmt in FORMATS:
        bpp = {"f32": 4, "bgr8": 3}.get(fmt, 1)
        if row_bytes % bpp:
            continue
        for kind in ("noise", "smooth"):
            img = content(kind, fmt, 3, row_bytes // bpp, seed=row_bytes)
            for rps in (1, 3):
                deflate(img, fmt, rps)


@gpu
def test_10000_by_10000_dem():
    if EMULATED:
        return   # minutes on the emulated kernels; every path it takes is covered by the smaller cases
    img = content("smooth", "f32", 10000, 10000, seed=3)
    for rps in (None, 40):
        deflate(img, "f32", rps)


# ---- adversarial content ----------------------------------------------------------------------------------------------
@gpu
def test_adversarial_contents():
    rng = np.random.default_rng(11)
    cases = []
    w = 70000
    cases.append(("gray8", np.zeros((2, w), np.uint8)))                        # runs of 258 at distance 1
    cases.append(("gray8", np.full((2, w), 7, np.uint8)))
    cases.append(("mask8", np.full((3, 9000), 255, np.uint8)))
    cases.append(("gray8", rng.integers(0, 256, (2, w)).astype(np.uint8)))      # stored blocks
    for period in (3, 32768, 32769):                                           # minimum matches; the largest distance
        unit = rng.integers(0, 256, period).astype(np.uint8)                  # and one past it
        p = np.tile(unit, -(-3 * 32769 // period))[:3 * 32769][None, :]
        cases.append(("gray8", from_predicted(p, "gray8")))
    p = rng.permutation(np.arange(256, dtype=np.uint8))[None, :]              # no matches, no distance codes
    cases.append(("gray8", from_predicted(p, "gray8")))
    cases.append(("gray8", np.full((1, 1), 9, np.uint8)))                     # one literal
    cases.append(("gray8", np.full((1, 2), 9, np.uint8)))
    cases.append(("f32", np.full((40, 300), np.nan, np.float32)))             # an all-NaN DEM
    cases.append(("f32", content("smooth", "f32", 40, 300, seed=2)))          # a DSM with holes
    cases.append(("bgr8", from_predicted(np.tile(rng.integers(0, 256, 3 * 11).astype(np.uint8), (4, 2000)), "bgr8")))
    for fmt, img in cases:
        row = predict(img, fmt).shape[1]
        for rps in (1, img.shape[0], default_rps(row)):
            deflate(img, fmt, rps)


# ---- Huffman codes at their length limits ------------------------------------------------------------------------------

def huffman_depth(counts):
    """The longest code of a Huffman code for the non-zero counts, built without a length limit.  On equal weights a
    leaf is taken before a merged node, which gives the smallest longest code any Huffman code of these counts has."""
    h = [(int(c), k, 0) for k, c in enumerate(counts) if c]
    if len(h) < 2:
        return len(h)
    heapq.heapify(h)
    k = len(counts)
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        heapq.heappush(h, (a[0] + b[0], k, max(a[2], b[2]) + 1))
        k += 1
    return h[0][2]


def no_repeat_sequence(counts, rng):
    """The symbols with the given counts in an order where no 3 consecutive bytes occur twice."""
    left = np.array(counts, np.int64)
    seen = set()
    out = []
    n = int(left.sum())
    for i in range(n):
        syms = np.flatnonzero(left)
        order = rng.permutation(syms)
        w = left[order].astype(float)
        # weighted order: try symbols in a random order biased by what is left
        keys = rng.random(len(order)) ** (1.0 / w)
        order = order[np.argsort(-keys)]
        for s in order:
            if i < 2 or (out[-2], out[-1], int(s)) not in seen:
                break
        else:
            raise RuntimeError("stuck at %d" % i)
        if i >= 2:
            seen.add((out[-2], out[-1], int(s)))
        out.append(int(s))
        left[s] -= 1
    return np.array(out, np.uint8)

class Bits:
    def __init__(self, data):
        self.d, self.p = data, 0
    def get(self, n):
        v = 0
        for k in range(n):
            v |= ((self.d[self.p >> 3] >> (self.p & 7)) & 1) << k
            self.p += 1
        return v

def decode_table(lengths):
    codes, code = {}, 0
    bl = [0] * 17
    for l in lengths:
        bl[l] += 1
    bl[0] = 0
    nxt = [0] * 17
    for b in range(1, 17):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    for s, l in enumerate(lengths):
        if l:
            codes[(l, nxt[l])] = s
            nxt[l] += 1
    return codes

def sym(bits, table):
    code = l = 0
    while True:
        code = (code << 1) | bits.get(1)
        l += 1
        if (l, code) in table:
            return table[(l, code)]
        assert l <= 15

LBASE = [3,4,5,6,7,8,9,10,11,13,15,17,19,23,27,31,35,43,51,59,67,83,99,115,131,163,195,227,258]
LEXT = [0]*8+[1]*4+[2]*4+[3]*4+[4]*4+[5]*4+[0]
DEXT = [0,0,0,0,1,1,2,2,3,3,4,4,5,5,6,6,7,7,8,8,9,9,10,10,11,11,12,12,13,13]
ORDER = [16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15]

def dynamic_blocks(stream):
    """Per dynamic block of a zlib stream: (literal/length lengths, code-length lengths, histogram of the
    literal/length symbols decoded, histogram of the code-length symbols)."""
    b = Bits(stream[2:])
    out = []
    while True:
        final, typ = b.get(1), b.get(2)
        if typ == 0:
            b.p = (b.p + 7) & ~7
            n = b.get(16); b.get(16); b.p += 8 * n
        else:
            if typ == 1:
                lit = [8]*144 + [9]*112 + [7]*24 + [8]*8; dist = [5]*30; cl = None; clh = None
            else:
                hlit, hdist, hclen = b.get(5) + 257, b.get(5) + 1, b.get(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[ORDER[i]] = b.get(3)
                t = decode_table(cl)
                lens, clh = [], [0] * 19
                while len(lens) < hlit + hdist:
                    s = sym(b, t); clh[s] += 1
                    if s < 16: lens.append(s)
                    elif s == 16: lens += [lens[-1]] * (3 + b.get(2))
                    elif s == 17: lens += [0] * (3 + b.get(3))
                    else: lens += [0] * (11 + b.get(7))
                lit, dist = lens[:hlit], lens[hlit:]
            lt, dt = decode_table(lit), decode_table(dist)
            hist = [0] * 286
            while True:
                s = sym(b, lt); hist[s] += 1
                if s == 256: break
                if s > 256:
                    b.get(LEXT[s - 257]); d = sym(b, dt); b.get(DEXT[d])
            if typ == 2:
                out.append((lit, cl, hist, clh))
        if final:
            return out


def interleaved_lengths(groups):
    """One code length per literal value, from {length: how many}, with no length twice in a row (so the header's
    run-length code repeats none of them)."""
    left, order, prev = dict(groups), [], None
    while sum(left.values()):
        L = max((l for l in left if left[l] and l != prev), key=lambda l: (left[l], l))
        order.append(L)
        left[L] -= 1
        prev = L
    return order


@gpu
def test_codes_that_need_the_15_and_7_bit_limits_decode_exactly():
    rng = np.random.default_rng(7)
    # literals only (no 3 bytes repeat, so nothing matches): 64 values 620 times each and a tail whose counts follow the
    # Fibonacci numbers 1, 2, 3, 5 ... 233 (the end-of-block code is the first 1); every Huffman code of these counts
    # is at least 19 bits deep
    fib = [1, 1]
    while len(fib) < 13:
        fib.append(fib[-1] + fib[-2])
    lit_counts = np.zeros(256, np.int64)
    lit_counts[:64] = 620
    lit_counts[100:112] = fib[1:13]
    # counts 2^(15 - L) give literal lengths L exactly; the numbers of literals per length (and the two distance
    # codes and the run of 7 unused values) make a code-length code at least 10 bits deep
    lengths = interleaved_lengths({7: 110, 8: 5, 9: 55, 10: 3, 11: 13, 12: 8, 13: 1, 14: 21, 15: 33})
    cl_counts = np.zeros(256, np.int64)
    cl_counts[:len(lengths)] = [2 ** (15 - L) for L in lengths]
    for counts, which, limit in ((lit_counts, "literal/length", 15), (cl_counts, "code-length", 7)):
        seq = no_repeat_sequence(counts, rng)
        data, _ = deflate(from_predicted(seq[None, :], "gray8"), "gray8", 1)   # inflates exactly, within the bound
        blocks = dynamic_blocks(data)
        assert len(blocks) == 1
        lit, cl, hist, clh = blocks[0]
        assert sum(hist[257:]) == 0 and hist[:256] == list(counts)
        coded, needed = (max(lit), huffman_depth(hist)) if limit == 15 else (max(cl), huffman_depth(clh))
        assert coded == limit and needed > limit, (which, coded, needed)


@gpu
def test_repeated_calls_give_identical_bytes():
    for fmt in FORMATS:
        img = content("smooth", fmt, 64, 700, seed=5)
        d = Dev(img)
        first = None
        for _ in range(3):
            st, buf, n, counts = deflate_dev(d, 64, 700, fmt, 5)
            assert st == 0
            got = (buf[:n].tobytes(), counts.tobytes())
            assert first is None or got == first
            first = got


@gpu
def test_pitched_and_misaligned_inputs():
    for fmt in FORMATS:
        img = content("noise", fmt, 13, 29, seed=1)
        row = predict(img, fmt).shape[1] if fmt != "f32" else 29 * 4
        offs = (0, 4, 8, 12) if fmt == "f32" else range(8)
        for off in offs:
            deflate(img, fmt, 4, pitch=row + 4 * (off + 1), off=off)


# ---- the ratio against zlib level 1 on the same predicted strips --------------------------------------------------------
def bench_rasters(n, seed=0):
    """Stand-ins for the four rasters of tools/geotiff_deflate_bench.py at n x n: a DSM-like elevation (analytic terrain,
    5 cm noise, NaN holes), gray and colour orthomosaics (procedural frame content, black where no frame reaches), and
    the observation_index mask."""
    rng = np.random.default_rng(seed)
    dem = (synth.analytic_elevation(n, n, 0.25).T + rng.normal(0, 0.05, (n, n))).astype(np.float32)
    yy, xx = np.mgrid[0:n, 0:n]
    holes = np.zeros((n, n), bool)
    for _ in range(12):
        cy, cx, r = rng.integers(0, n), rng.integers(0, n), rng.integers(n // 80 + 1, n // 20 + 2)
        holes |= (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
    dem[holes] = np.nan
    outside = (xx + yy) < n // 6
    gray = synth.procedural_image(0, n, n, 1).reshape(n, n).copy()
    gray[outside] = 0
    color = synth.procedural_image(1, n, n, 3).reshape(n, n, 3).copy()
    color[outside] = 0
    mask = np.where(outside | holes, 0, 255).astype(np.uint8)
    return {"elevation": ("f32", dem), "ortho": ("gray8", gray), "colored_ortho": ("bgr8", color),
            "observation_index": ("mask8", mask)}


def zlib1_size(img, fmt, rps):
    pred = predict(img, fmt)
    return sum(len(zlib.compress(pred[s:s + rps].tobytes(), 1)) for s in range(0, pred.shape[0], rps))


@gpu
def test_ratio_within_5_percent_of_zlib_level_1(tmp_path):
    if EMULATED:
        # rendering the benchmark's orthomosaics takes a GPU: 1024 x 1024 stand-ins exercise the same kernels
        for name, (fmt, img) in bench_rasters(1024).items():
            rps = default_rps(predict(img[:1], fmt).shape[1])
            data, _ = deflate(img, fmt, rps)
            z1 = zlib1_size(img, fmt, rps)
            assert len(data) <= 1.05 * z1, (name, len(data), z1, len(data) / z1)
        return
    # the four rasters of tools/geotiff_deflate_bench.py: the joint workload's 10000 x 10000 map, its rendered
    # orthomosaics, their observation_index and a DSM-like elevation
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import geotiff_deflate_bench as gb
    gm = gb.bench_map()
    for name, fmt in gb.BENCH_LAYERS:
        band = gm.to_raster(name, fmt)
        rps = default_rps(predict(band[:1], fmt).shape[1])
        path = str(tmp_path / "bench.tif")
        gm.to_geotiff(path, name, fmt=fmt)
        a = io.read_geotiff(path)[0] if fmt != "bgr8" else \
            np.stack([io.read_geotiff(path, band=k)[0] for k in (2, 1, 0)], axis=-1)
        assert same_bits(a, band), name
        size = sum(io._read_ifd(open(path, "rb").read())[279])
        z1 = zlib1_size(band, fmt, rps)
        assert size <= 1.05 * z1, (name, size, z1, size / z1)
        del band, a


# ---- files of map layers ------------------------------------------------------------------------------------------------
def mapping_run(rows=72, cols=56, col_range=None):
    res = 1.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0, col_range=col_range)
    xyz = synth.point_cloud(8000, rows * res / 2, cols * res / 2, seed=21, holes=2, hole_sides=(4.0, 10.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, agl=60.0, seed=4, jitter_pos=0.5)
    for colored in (False, True):
        ch = 3 if colored else 1
        imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(poses))]
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm).process(poses, imgs, gm)
    return gm


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


@gpu
def test_files_read_back_as_the_exported_rasters(tmp_path):
    gm = mapping_run()
    gm.sync()
    for name, fmt in (("elevation", "f32"), ("ortho", "gray8"), ("colored_ortho", "bgr8"),
                      ("observation_index", "mask8"), ("elevation", "gray8")):
        band = gm.to_raster(name, fmt)
        for rps in (None, 1, 7, band.shape[0]):
            path = str(tmp_path / ("%s_%s_%s.tif" % (name, fmt, rps)))
            gm.to_geotiff(path, name, fmt=fmt, nodata="nan" if fmt == "f32" else None, rows_per_strip=rps)
            a, gt, epsg, nodata = io.read_geotiff(path)
            if fmt == "bgr8":
                a = np.stack([io.read_geotiff(path, band=k)[0] for k in (2, 1, 0)], axis=-1)
            assert same_bits(a, band), (name, fmt, rps)
            assert gt == gm.geotransform() and epsg == 32632
            assert (nodata is None) == (fmt != "f32")
            plain = str(tmp_path / "plain.tif")
            io.write_geotiff(plain, band, gm.geotransform(), nodata="nan" if fmt == "f32" else None)
            want, got = io._read_ifd(open(plain, "rb").read()), io._read_ifd(open(path, "rb").read())
            layout = {259, 273, 278, 279, 317}
            assert {k: v for k, v in want.items() if k not in layout} == \
                {k: v for k, v in got.items() if k not in layout}
            assert got[259] == (8,) and got[317] == ((3,) if fmt == "f32" else (2,))


@gpu
def test_other_readers_decode_the_files(tmp_path):
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    gm = mapping_run()
    for name, fmt in (("elevation", "f32"), ("ortho", "gray8"), ("colored_ortho", "bgr8"),
                      ("observation_index", "mask8")):
        band = gm.to_raster(name, fmt)
        path = str(tmp_path / ("%s.tif" % fmt))
        gm.to_geotiff(path, name, fmt=fmt)
        assert same_bits(cv2.imread(path, cv2.IMREAD_UNCHANGED), band), ("cv2", fmt)
        im = np.asarray(Image.open(path))
        assert same_bits(im[:, :, ::-1] if fmt == "bgr8" else im, band), ("PIL", fmt)


@gpu
def test_elevation_round_trip_on_a_whole_map_and_a_stripe(tmp_path):
    whole = mapping_run()
    whole.download(("elevation",))
    elev = whole["elevation"].copy(order="F")
    rows, cols = whole.getSize()
    for col_range in (None, (0, 1), (13, 40)):
        gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * 1.0, cols * 1.0, 1.0)).getMutable()
        gm["elevation"] = elev
        gm.to_device(0, col_range=col_range, names=("elevation",))
        band = gm.to_raster("elevation")
        path = str(tmp_path / "dem.tif")
        gm.to_geotiff(path, "elevation", nodata="nan")
        a, gt, _, nodata = io.read_geotiff(path)
        assert same_bits(a, band)
        c0 = col_range[0] if col_range else 0
        full_gt = gm.geotransform()
        assert gt == (full_gt[0], full_gt[1], 0.0, full_gt[3] + c0 * full_gt[5], 0.0, full_gt[5])
        back = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * 1.0, cols * 1.0, 1.0)).getMutable()
        # NaN pixels are no-data to the import and leave their cells as they are: those cells start as the layer's NaNs
        back["elevation"] = np.where(np.isnan(elev), elev, np.float32(1234.5)).astype(np.float32, order="F")
        back.to_device(0, col_range=col_range, names=("elevation",))
        back.from_raster("elevation", a, gt, nodata=nodata)
        assert same_bits(back.to_raster("elevation"), band), col_range


@gpu
def test_compression_enqueued_right_after_process_equals_one_after_sync(tmp_path):
    rows, cols, res = 300, 260, 0.5
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(60000, rows * res / 2, cols * res / 2, seed=31, holes=2, hole_sides=(4.0, 12.0))
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    first = str(tmp_path / "first.tif")
    gm.to_geotiff(first, "elevation")   # no amb_sync in between: ordered on the context's stream
    gm.sync()
    second = str(tmp_path / "second.tif")
    gm.to_geotiff(second, "elevation")
    assert open(first, "rb").read() == open(second, "rb").read()
    assert same_bits(io.read_geotiff(first)[0], gm.to_raster("elevation"))


@gpu
def test_pinned_and_pageable_destinations_are_identical():
    img = content("noise", "bgr8", 300, 900, seed=5)     # ~800 KB of strips: large enough for the staged pageable copy
    d = Dev(img)
    L = _lib.lib()
    cap = L.amb_deflate_max_size(900, 300, _lib.RASTER_BGR8, 3)
    p = C.c_void_p()
    amb.check(L.amb_host_alloc(C.byref(p), cap))
    try:
        pinned = np.frombuffer((C.c_uint8 * cap).from_address(p.value), np.uint8)
        st, _, n, c1 = deflate_dev(d, 300, 900, "bgr8", 3, out=pinned)
        assert st == 0
        st, pageable, m, c2 = deflate_dev(d, 300, 900, "bgr8", 3)
        assert st == 0 and n == m and pinned[:n].tobytes() == pageable[:m].tobytes() and np.array_equal(c1, c2)
        check_strips(img, "bgr8", 3, pageable[:m].tobytes(), c2)
    finally:
        L.amb_host_free(p)


# ---- the argument contract ------------------------------------------------------------------------------------------
@gpu
def test_too_small_a_capacity_returns_the_size_and_writes_nothing():
    img = content("smooth", "f32", 40, 50, seed=1)
    d = Dev(img)
    st, buf, n, counts = deflate_dev(d, 40, 50, "f32", 6)
    assert st == 0
    want = buf[:n].tobytes()
    for cap in (0, 1, n - 1):
        out = np.full(n + 64, CANARY, np.uint8)
        cnt = np.full(7, 0xA5A5A5A5, np.uint32)
        st, _, m, _ = deflate_dev(d, 40, 50, "f32", 6, out=out, capacity=cap, counts=cnt)
        assert st == _lib.AMB_ERR_SIZE_MISMATCH and m == n and (out == CANARY).all() and (cnt == 0xA5A5A5A5).all()
    out = np.full(n + 64, CANARY, np.uint8)
    st, _, m, cnt = deflate_dev(d, 40, 50, "f32", 6, out=out, capacity=n)
    assert st == 0 and out[:m].tobytes() == want and (out[m:] == CANARY).all() and np.array_equal(cnt, counts)


@gpu
def test_invalid_arguments_write_nothing():
    L = _lib.lib()
    ctx = api._jpeg_context(0)
    d = Dev(content("noise", "f32", 9, 9, seed=2))
    d8 = Dev(content("noise", "gray8", 9, 9, seed=2), off=1)
    buf = np.full(4096, CANARY, np.uint8)
    cnt = np.full(16, 0xA5A5A5A5, np.uint32)
    size = C.c_size_t(12345)
    INV = _lib.AMB_ERR_INVALID_ARGUMENT
    # (ctx, image, w, h, stride, format, rows_per_strip, out given, counts given, size given)
    good = [ctx, d.ptr, 9, 9, 36, 0, 4, True, True, True]
    cases = [(0, None), (1, None), (7, False), (8, False), (9, False), (2, 0), (2, -1), (3, 0), (3, -5), (4, 35),
             (5, 4), (5, -1), (6, 0), (6, -1), (4, 38), (1, d.ptr + 2)]
    for k, v in cases:
        a = list(good)
        a[k] = v
        st = L.amb_deflate_strips_device(a[0], a[1], a[2], a[3], a[4], a[5], a[6], buf.ctypes.data if a[7] else None,
                                         len(buf), C.byref(size) if a[9] else None, cnt.ctypes.data if a[8] else None)
        assert st == INV, (k, v, st)
    # 8-bit rasters at any alignment and stride, but not a short one
    assert L.amb_deflate_strips_device(ctx, d8.ptr, 9, 9, 8, 1, 4, buf.ctypes.data, len(buf), C.byref(size),
                                       cnt.ctypes.data) == INV
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    assert L.amb_deflate_max_size(0, 9, 0, 1) == 0 and L.amb_deflate_max_size(9, 9, 4, 1) == 0
    assert L.amb_deflate_max_size(9, 9, 0, 0) == 0
    assert L.amb_deflate_max_size(9, 9, 0, 4) == 2 * bound(4 * 36) + bound(36)
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable()
    gm.to_device(0)
    gc = gm.context()
    for layer, fmt, rps in ((-1, 0, 1), (len(_lib.LAYER_NAMES), 0, 1), (0, 4, 1), (0, -1, 1), (0, 0, 0)):
        assert L.amb_export_deflate_strips(gc, layer, fmt, rps, buf.ctypes.data, len(buf), C.byref(size),
                                           cnt.ctypes.data) == INV
    assert L.amb_export_deflate_strips(None, 0, 0, 1, buf.ctypes.data, len(buf), C.byref(size), cnt.ctypes.data) == INV
    assert L.amb_export_deflate_strips(gc, 0, 0, 1, buf.ctypes.data, len(buf), C.byref(size), None) == INV
    gm.sync()
    assert (buf == CANARY).all() and (cnt == 0xA5A5A5A5).all() and size.value == 12345
    with pytest.raises(ValueError):
        gm.to_geotiff("unused.tif", "elevation_angle")
    with pytest.raises(ValueError):
        gm.to_geotiff("unused.tif", "elevation", fmt="rgb8")
    with pytest.raises(ValueError):
        gm.to_geotiff("unused.tif", "elevation", rows_per_strip=0)
    with pytest.raises(amb.AmbError):
        amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable().to_geotiff("unused.tif", "elevation")
    assert not os.path.exists("unused.tif")


@gpu
def test_torch_wrapper(tmp_path):
    if EMULATED:
        return   # the wrapper takes torch CUDA tensors; its C entry point is what every other test here calls
    import torch
    img = content("smooth", "bgr8", 123, 77, seed=4)
    t = torch.from_numpy(img).cuda()
    data, counts, rps = amb.deflate_strips(t, "bgr8")
    assert rps == 8192 // (77 * 3)
    check_strips(img, "bgr8", rps, data, counts)
    big = torch.zeros((123, 100, 3), dtype=torch.uint8, device="cuda")
    big[:, :77] = t
    padded = amb.deflate_strips(big[:, :77], "bgr8")                       # padded rows
    assert padded[0] == data and np.array_equal(padded[1], counts) and padded[2] == rps
    dem = content("smooth", "f32", 50, 60, seed=1)
    data, counts, rps = amb.deflate_strips(torch.from_numpy(dem).cuda(), "f32", 7)
    check_strips(dem, "f32", 7, data, counts)
    path = str(tmp_path / "dem.tif")
    io.write_geotiff_strips(path, data, counts, 60, 50, "f32", rps, (0.0, 0.5, 0.0, 10.0, 0.0, -0.5), nodata="nan")
    assert same_bits(io.read_geotiff(path)[0], dem)
    with pytest.raises(ValueError):
        amb.deflate_strips(t.float(), "bgr8")
    with pytest.raises(ValueError):
        amb.deflate_strips(t[:, ::2], "bgr8")
    with pytest.raises(ValueError):
        amb.deflate_strips(t, "rgb8")


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_geotiff_deflate.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
