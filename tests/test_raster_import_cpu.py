"""The host side of the raster import, without a GPU: io.read_geotiff against io.write_geotiff, OpenCV, PIL and a small
encoder for the layouts neither library writes (tiles, floating-point predictor), its refusals, and the per-axis tables
of amb_raster_import_tables against the numpy restatement of tests/test_gpu_raster_import.py."""
import ctypes as C
import struct
import zlib

import numpy as np
import pytest

from aerial_mapper_b200 import _lib
from aerial_mapper_b200.io import read_geotiff, write_geotiff
from test_gpu_raster_import import SNAP, geometry, tables

GT = (464450.0, 0.5, 0.0, 5272530.0, 0.0, -0.5)
_FMT = {3: "H", 4: "I", 12: "d"}


def ifd_file(path, entries, blobs, head=b"II*\0"):
    """A classic TIFF: header, image data `blobs` (each 16-byte aligned), then one IFD.  entries: (tag, type, values);
    values may reference blob k as ("blob", k) for offsets."""
    data = bytearray(head + b"\0\0\0\0")
    at = []
    for b in blobs:
        data += b"\0" * (-len(data) % 16)
        at.append(len(data))
        data += b
    data += b"\0" * (-len(data) % 16)
    extra = bytearray()
    ents = []
    entries = sorted(entries, key=lambda e: e[0])
    ifd_at = len(data)
    extra_at = ifd_at + 2 + 12 * len(entries) + 4
    for tag, typ, vals in entries:
        vals = [at[v[1]] if isinstance(v, tuple) else v for v in vals]
        p = bytes(vals) + b"\0" if typ == 2 else struct.pack("<%d%s" % (len(vals), _FMT[typ]), *vals)
        count = len(vals) + 1 if typ == 2 else len(vals)
        if len(p) <= 4:
            ents.append(struct.pack("<HHI", tag, typ, count) + p.ljust(4, b"\0"))
        else:
            ents.append(struct.pack("<HHII", tag, typ, count, extra_at + len(extra)))
            extra += p + b"\0" * (len(p) & 1)
    data += struct.pack("<H", len(entries)) + b"".join(ents) + struct.pack("<I", 0) + extra
    struct.pack_into("<I", data, 4, ifd_at)
    with open(path, "wb") as f:
        f.write(bytes(data))


def geo_entries(gt=GT, epsg=32633, raster_type=1, transform=None):
    keys = [1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, raster_type, 3072, 0, 1, epsg]
    e = [(34735, 3, keys)]
    if transform is not None:
        e.append((34264, 12, list(transform)))
    else:
        e += [(33550, 12, [gt[1], -gt[5], 0.0]), (33922, 12, [0.0, 0.0, 0.0, gt[0], gt[3], 0.0])]
    return e


def encode(path, a, tile=None, predictor=1, deflate=True, rows_per_strip=3, extra=(), geo=None):
    """a: [H, W] or [H, W, spp] -> a GeoTIFF in strips or (th, tw) tiles, with the given predictor."""
    a = a if a.ndim == 3 else a[:, :, None]
    h, w, spp = a.shape
    dt = a.dtype
    item = dt.itemsize
    if tile:
        th, tw = tile
        padded = np.zeros((-(-h // th) * th, -(-w // tw) * tw, spp), dt)
        padded[:h, :w] = a
        chunks = [padded[r:r + th, c:c + tw] for r in range(0, padded.shape[0], th)
                  for c in range(0, padded.shape[1], tw)]
    else:
        chunks = [a[r:r + rows_per_strip] for r in range(0, h, rows_per_strip)]
    blobs = []
    for ch in chunks:
        ch = np.ascontiguousarray(ch)
        if predictor == 2:
            d = ch.copy()
            d[:, 1:] = ch[:, 1:] - ch[:, :-1]
            raw = d.astype(dt.newbyteorder("<")).tobytes()
        elif predictor == 3:
            be = ch.astype(dt.newbyteorder(">")).view(np.uint8).reshape(ch.shape[0], -1, item)
            planes = np.ascontiguousarray(be.transpose(0, 2, 1)).reshape(ch.shape[0], -1)
            d = planes.copy()
            d[:, spp:] = planes[:, spp:] - planes[:, :-spp]
            raw = d.tobytes()
        else:
            raw = ch.astype(dt.newbyteorder("<")).tobytes()
        blobs.append(zlib.compress(raw) if deflate else raw)
    n = len(blobs)
    fmt = {"u": 1, "i": 2, "f": 3}[dt.kind]
    e = [(256, 4, [w]), (257, 4, [h]), (258, 3, [item * 8] * spp), (259, 3, [8 if deflate else 1]), (262, 3, [1]),
         (277, 3, [spp]), (284, 3, [1]), (317, 3, [predictor]), (339, 3, [fmt] * spp)]
    if tile:
        e += [(322, 4, [tile[1]]), (323, 4, [tile[0]]), (324, 4, [("blob", k) for k in range(n)]),
              (325, 4, [len(b) for b in blobs])]
    else:
        e += [(273, 4, [("blob", k) for k in range(n)]), (278, 4, [rows_per_strip]), (279, 4, [len(b) for b in blobs])]
    e += list(geo if geo is not None else geo_entries())
    e += list(extra)
    # later entries win: a test overrides a tag by passing it in `extra`
    ifd_file(path, list({t: (t, ty, v) for t, ty, v in e}.values()), blobs)


def add_geotags(path, gt=GT, epsg=32633):
    """Append a new first IFD = the file's IFD + ModelPixelScale, ModelTiepoint and GeoKeyDirectory."""
    data = bytearray(open(path, "rb").read())
    at = struct.unpack_from("<I", data, 4)[0]
    n = struct.unpack_from("<H", data, at)[0]
    ents = [bytes(data[at + 2 + 12 * k:at + 14 + 12 * k]) for k in range(n)]
    data += b"\0" * (-len(data) % 8)
    blobs = b""
    for tag, typ, cnt, p in ((33550, 12, 3, struct.pack("<3d", gt[1], -gt[5], 0.0)),
                             (33922, 12, 6, struct.pack("<6d", 0.0, 0.0, 0.0, gt[0], gt[3], 0.0)),
                             (34735, 3, 16, struct.pack("<16H", 1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1,
                                                        epsg))):
        ents.append(struct.pack("<HHII", tag, typ, cnt, len(data) + len(blobs)))
        blobs += p
    ents.sort(key=lambda e: struct.unpack_from("<H", e)[0])
    ifd_at = len(data) + len(blobs)
    data += blobs + struct.pack("<H", len(ents)) + b"".join(ents) + struct.pack("<I", 0)
    struct.pack_into("<I", data, 4, ifd_at)
    open(path, "wb").write(bytes(data))


# ---- write_geotiff -> read_geotiff ------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(1, 1), (7, 13), (600, 1111)])
def test_reads_back_write_geotiff_exactly(tmp_path, h, w):
    rng = np.random.default_rng(h * w)
    dem = rng.normal(400.0, 30.0, (h, w)).astype(np.float32)
    dem[rng.random((h, w)) < 0.2] = np.nan
    dem.ravel()[0] = -0.0
    gray = rng.integers(0, 256, (h, w), dtype=np.uint8)
    for a, nodata, epsg in ((dem, "nan", 32633), (gray, 0, 25832), (dem, None, 32632)):
        path = str(tmp_path / "x.tif")
        write_geotiff(path, a, GT, epsg=epsg, nodata=nodata)
        b, gt, e, nd = read_geotiff(path)
        assert b.dtype == a.dtype and b.tobytes() == a.tobytes()
        assert gt == GT and e == epsg
        assert (nd is None) if nodata is None else (float(nodata) == nd or (np.isnan(nd) and nodata == "nan"))


# ---- files written by OpenCV and PIL -----------------------------------------------------------------------------------
def test_reads_opencv_deflate_predictor_2_int16(tmp_path):
    cv2 = pytest.importorskip("cv2")
    a = np.random.default_rng(1).integers(-32768, 32767, (37, 53)).astype(np.int16)
    a[0, :5] = [-32768, 32767, 0, -1, 1]
    for comp in (cv2.IMWRITE_TIFF_COMPRESSION_ADOBE_DEFLATE, cv2.IMWRITE_TIFF_COMPRESSION_DEFLATE):
        path = str(tmp_path / "cv.tif")
        assert cv2.imwrite(path, a, [cv2.IMWRITE_TIFF_COMPRESSION, comp, cv2.IMWRITE_TIFF_ROWSPERSTRIP, 5])
        add_geotags(path)
        b, gt, epsg, nodata = read_geotiff(path)
        assert b.dtype == np.int16 and np.array_equal(b, cv2.imread(path, cv2.IMREAD_UNCHANGED)) and np.array_equal(b, a)
        assert gt == GT and epsg == 32633 and nodata is None


@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.uint16])
@pytest.mark.parametrize("compression", [None, "tiff_adobe_deflate"])
def test_reads_pil_files(tmp_path, dtype, compression):
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(2)
    a = (rng.normal(0, 1000, (29, 41)) if dtype == np.float32 else rng.integers(np.iinfo(dtype).min,
                                                                                np.iinfo(dtype).max, (29, 41)))
    a = a.astype(dtype)
    path = str(tmp_path / "pil.tif")
    Image.fromarray(a).save(path, compression=compression)
    add_geotags(path)
    b, gt, _, _ = read_geotiff(path)
    with Image.open(path) as im:
        want = np.array(im)
    assert np.array_equal(b, want) and np.array_equal(b.astype(np.float64), a.astype(np.float64)) and gt == GT


# ---- tiles and the floating-point predictor (own encoder), decoded by OpenCV and PIL too -------------------------------
ENCODED = [("f32 tiles p3", np.float32, (16, 32), 3), ("f64 strips p3", np.float64, None, 3),
           ("f32 strips p3", np.float32, None, 3), ("i16 tiles p2", np.int16, (16, 16), 2),
           ("u8 tiles p1", np.uint8, (32, 16), 1), ("i32 strips p2", np.int32, None, 2),
           ("u16 tiles raw", np.uint16, (16, 16), 1)]


@pytest.mark.parametrize("case", ENCODED, ids=[c[0] for c in ENCODED])
def test_tiles_and_predictors_decode_like_opencv_and_pil(tmp_path, case):
    cv2 = pytest.importorskip("cv2")
    _, dtype, tile, predictor = case
    rng = np.random.default_rng(3)
    h, w = 45, 70
    if np.dtype(dtype).kind == "f":
        a = rng.normal(300, 50, (h, w)).astype(dtype)
        a[5, 5], a[6, 6], a[7, 7] = np.nan, -np.inf, -0.0
    else:
        info = np.iinfo(dtype)
        a = rng.integers(info.min, info.max, (h, w), endpoint=True).astype(dtype)
    path = str(tmp_path / "enc.tif")
    encode(path, a, tile=tile, predictor=predictor, deflate=case[0] != "u16 tiles raw")
    b, gt, epsg, _ = read_geotiff(path)
    assert b.dtype == dtype and b.tobytes() == a.tobytes() and gt == GT and epsg == 32633
    cv = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert cv is not None and cv.dtype == b.dtype and cv.tobytes() == b.tobytes()
    try:
        from PIL import Image
        with Image.open(path) as im:
            pil = np.array(im)
    except Exception:      # PIL does not decode every layout: compared wherever it does
        return
    assert np.array_equal(pil.astype(np.float64), b.astype(np.float64), equal_nan=True)


def test_band_of_a_multi_sample_file(tmp_path):
    a = np.random.default_rng(4).integers(0, 60000, (20, 30, 3)).astype(np.uint16)
    path = str(tmp_path / "rgb.tif")
    encode(path, a, tile=(16, 16), predictor=2)
    for k in range(3):
        assert np.array_equal(read_geotiff(path, band=k)[0], a[:, :, k])
    with pytest.raises(ValueError):
        read_geotiff(path, band=3)


# ---- georeferencing --------------------------------------------------------------------------------------------------
def test_geotransform_variants(tmp_path):
    a = np.zeros((4, 6), np.float32)
    path = str(tmp_path / "g.tif")
    # PixelIsPoint: the tiepoint is a pixel centre, GDAL shifts by half a pixel
    encode(path, a, geo=geo_entries(raster_type=2))
    assert read_geotiff(path)[1] == (GT[0] - 0.25, 0.5, 0.0, GT[3] + 0.25, 0.0, -0.5)
    # ModelTransformation without rotation
    encode(path, a, geo=geo_entries(transform=[2.0, 0, 0, 100.0, 0, -3.0, 0, 200.0, 0, 0, 0, 0, 0, 0, 0, 1]))
    assert read_geotiff(path)[1] == (100.0, 2.0, 0.0, 200.0, 0.0, -3.0)
    # a tiepoint at an inner pixel (I, J) = (10, 4)
    geo = [(34735, 3, [1, 1, 0, 1, 2048, 0, 1, 4326]), (33550, 12, [0.5, 0.25, 0.0]),
           (33922, 12, [10.0, 4.0, 0.0, 1000.0, 2000.0, 0.0])]
    encode(path, a, geo=geo, extra=[(42113, 2, list(b"-32768"))])
    _, gt, epsg, nodata = read_geotiff(path)
    assert gt == (995.0, 0.5, 0.0, 2001.0, 0.0, -0.25) and epsg == 4326 and nodata == -32768.0


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_every_unsupported_feature_raises(tmp_path):
    a = np.ones((8, 8), np.float32)
    path = str(tmp_path / "u.tif")
    cases = {
        "Compression": dict(extra=[(259, 3, [5])]),                      # LZW
        "Compression ": dict(extra=[(259, 3, [7])]),                     # JPEG
        "PlanarConfiguration": dict(extra=[(284, 3, [2])]),
        "Predictor": dict(predictor=2),                                  # horizontal differencing on floats
        "BitsPerSample": dict(extra=[(258, 3, [24])]),
        "ModelTransformation": dict(geo=geo_entries(transform=[1.0, 0.1, 0, 0, 0, -1.0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1])),
        "geotransform": dict(geo=[(33550, 12, [1.0, -1.0, 0.0]), (33922, 12, [0.0] * 6)]),   # south-up
        "ModelTiepoint": dict(geo=[(33550, 12, [1.0, 1.0, 0.0]), (33922, 12, [0.0] * 12)]),  # two tiepoints
        "georeferencing": dict(geo=[]),
    }
    for name, kw in cases.items():
        encode(path, a, **kw)
        with pytest.raises(ValueError, match=name.strip()):
            read_geotiff(path)
    encode(path, np.ones((8, 8), np.int8))
    with pytest.raises(ValueError, match="SampleFormat"):
        read_geotiff(path)
    encode(path, np.ones((8, 8), np.int16), predictor=3)
    with pytest.raises(ValueError, match="Predictor"):
        read_geotiff(path)
    ifd_file(path, [(256, 4, [1])], [], head=b"II+\0")
    with pytest.raises(ValueError, match="BigTIFF"):
        read_geotiff(path)
    open(path, "wb").write(b"MM\0*\0\0\0\x08" + b"\0" * 16)
    with pytest.raises(ValueError, match="big-endian"):
        read_geotiff(path)
    cv2 = pytest.importorskip("cv2")
    assert cv2.imwrite(path, np.ones((8, 8), np.uint16))                # OpenCV's default: LZW
    add_geotags(path)
    with pytest.raises(ValueError, match="Compression = 5"):
        read_geotiff(path)


# ---- the host tables ---------------------------------------------------------------------------------------------------
def host_tables(g, width, height, gt, method, c0=0, c1=None):
    c1 = g.cols if c1 is None else c1
    sc, fx = np.zeros(g.rows, np.int32), np.zeros(g.rows)
    sr, fy = np.zeros(c1 - c0, np.int32), np.zeros(c1 - c0)
    assert _lib.lib().amb_raster_import_tables(C.byref(g), c0, c1, width, height, (C.c_double * 6)(*gt),
                                               _lib.RESAMPLE[method], sc.ctypes.data, fx.ctypes.data, sr.ctypes.data,
                                               fy.ctypes.data) == 0
    return sc, fx, sr, fy


@pytest.mark.parametrize("n", [1, 17, 10000])
@pytest.mark.parametrize("method", ["nearest", "bilinear"])
def test_host_tables_equal_the_restatement(n, method):
    res = 0.25
    edges = [0.0, SNAP, SNAP - 2.0 ** -40, SNAP + 2.0 ** -40, 1 - SNAP, 1 - SNAP - 2.0 ** -40, 1 - SNAP + 2.0 ** -40,
             0.5, 0.3]
    for center in ((0.0, 0.0), (464500.0, 5272500.0)):
        g = geometry(n, max(1, n // 3), res, center)
        for d in edges:
            for dem_res, w, h in ((res, n + 2, g.cols + 2), (1.0, n // 4 + 3, g.cols // 4 + 3), (0.1, 3 * n, 3 * g.cols)):
                # the raster's west edge `d` pixels east of the map's: fractions of d (and 1 - d) along both axes
                gt = (center[0] - n * res / 2 + d * dem_res - dem_res, dem_res, 0.0,
                      center[1] + g.cols * res / 2 - d * dem_res + dem_res, 0.0, -dem_res)
                sc, fx, sr, fy = host_tables(g, w, h, gt, method)
                (ci, f1, _), (rj, f2, _) = tables(g, w, h, gt, method)
                assert np.array_equal(sc, ci) and np.array_equal(sr, rj), (center, d, dem_res)
                assert np.array_equal(fx.view(np.uint64), f1.view(np.uint64)) and \
                    np.array_equal(fy.view(np.uint64), f2.view(np.uint64)), (center, d, dem_res)
    # a stripe's j table is the whole map's columns [c0, c1)
    g = geometry(17, 40, res)
    gt = (-2.0, 0.3, 0.0, 5.1, 0.0, -0.3)
    whole = host_tables(g, 30, 30, gt, method)
    part = host_tables(g, 30, 30, gt, method, 9, 23)
    assert np.array_equal(part[0], whole[0]) and np.array_equal(part[2], whole[2][9:23]) and \
        np.array_equal(part[3], whole[3][9:23])
    # snapped fractions do exist at the edges tested above, and the arguments are checked
    assert _lib.lib().amb_raster_import_tables(C.byref(g), 0, 41, 30, 30, (C.c_double * 6)(*gt), 1, sc.ctypes.data,
                                               fx.ctypes.data, sr.ctypes.data, fy.ctypes.data) == \
        _lib.AMB_ERR_INVALID_ARGUMENT
