"""TIFF bands inflated on the device (amb_tiff_decode_device, amb_import_tiff, amb_multi_import_tiff,
csrc/deflate_decode.cu; convention in include/aerial_mapper_b200.h): every decode equals
read_geotiff(...)[0].astype(np.float32) bit for bit (NaN positions for float64 files), and every import equals
GridMap.from_raster of that array bit for bit.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last test runs this file's `gpu` tests on the emulated kernels."""
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
from aerial_mapper_b200 import _lib, api, io, synth  # noqa: E402
from test_geotiff_inflate_cpu import (DTYPES, corrupt_streams, dynamic_stream, make_tiff, match_stream,  # noqa: E402
                                      predict, ref, sample_raster, zstream)
from test_gpu_raster_export import Dev, EMULATED  # noqa: E402

try:
    import cv2
except ImportError:
    cv2 = None

gpu = pytest.mark.gpu


class HostFile(object):
    """The file's bytes as a pageable numpy array, in pinned memory (amb_host_alloc), or as the bytes object itself."""

    def __init__(self, data, kind="pageable"):
        self.size = len(data)
        self.pinned = None
        if kind == "pinned":
            p = C.c_void_p()
            assert _lib.lib().amb_host_alloc(C.byref(p), max(1, len(data))) == 0
            C.memmove(p, data, len(data))
            self.pinned, self.ptr = p, p.value
        elif kind == "bytes":
            self.keep = data
            self.ptr = C.cast(C.c_char_p(data), C.c_void_p).value
        else:
            self.keep = np.frombuffer(data, np.uint8).copy()
            self.ptr = self.keep.ctypes.data

    def free(self):
        if self.pinned is not None:
            _lib.lib().amb_host_free(self.pinned)


def decode(data, band=0, overview=0, window=None, kind="pageable", layout=None):
    """(status, float32 [r1 - r0, c1 - c0], untouched) of amb_tiff_decode_device over the window (default: all); the
    destination's rows are padded by 3 floats and start as canaries."""
    t = io.tiff_layout(data, band, overview)
    r0, r1, c0, c1 = window or (0, t.height, 0, t.width)
    w, h = c1 - c0, r1 - r0
    stride = w + 3
    dev = Dev(4 * stride * h)
    L = layout or t.c_layout()
    f = HostFile(data, kind)
    st = _lib.lib().amb_tiff_decode_device(api._jpeg_context(0), C.c_void_p(f.ptr), f.size, C.byref(L), r0, r1, c0, c1,
                                           C.c_void_p(dev.ptr), 4 * stride)
    f.free()
    raw = dev.all()
    body = raw[dev.lo:dev.lo + 4 * stride * h].view(np.float32).reshape(h, stride)
    untouched = bool(np.all(raw == 0xA5))
    return st, body[:, :w].copy(), untouched


def same(got, want, f64=False):
    if f64:
        assert np.array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32))
    else:
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def check(data, band=0, overview=0, window=None, kind="pageable"):
    want = ref(data, band, overview)
    f64 = want.dtype == np.float64
    want = want.astype(np.float32)
    if window:
        want = want[window[0]:window[1], window[2]:window[3]]
    st, got, _ = decode(data, band, overview, window, kind)
    assert st == _lib.AMB_OK
    same(got, want, f64)


# ---- decodes --------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("chunk", [("strips", 4), ("tiles", 16, 8)])
def test_every_sample_type_predictor_spp_and_band(dtype, chunk):
    preds = (1, 3) if np.dtype(dtype).kind == "f" else (1, 2)
    for spp in (1, 2, 3, 4):
        a = sample_raster(dtype, 19, 37, spp, seed=spp)      # tiles: partial edge tiles on both axes
        for pred in preds:
            b = make_tiff(a, pred, chunk)
            for band in range(spp):
                check(b, band)
        check(make_tiff(a, 1, chunk, compression=1), spp - 1)


@gpu
def test_zlib_levels_and_strategies():
    a = sample_raster(np.float32, 24, 61)
    for level in range(10):
        for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
            check(make_tiff(a, 3, ("strips", 8), encode=lambda raw, k: zstream(raw, level, strategy)))
    b = make_tiff(a, 3, ("tiles", 32, 16), encode=lambda raw, k: zstream(raw, 6, zlib.Z_DEFAULT_STRATEGY, flushes=4))
    check(b)                                             # empty stored blocks between the parts


@gpu
def test_long_matches_far_distances_and_runs():
    rng = np.random.default_rng(5)
    const = np.full((64, 600), 7, np.uint8)              # distance-1 runs and 258-byte matches
    check(make_tiff(const, 1, ("strips", 64)))
    check(make_tiff(const.astype(np.float64), 3, ("strips", 7)))
    # zlib never writes a distance above 32506 (32768 - 262): a period of 32506 bytes makes every match that far back
    period = rng.integers(0, 256, 32506).astype(np.uint8)
    far = np.tile(period, 4)[:96 * 1024].reshape(96, 1024)
    b = make_tiff(far, 1, ("strips", 96), encode=lambda raw, k: zstream(raw, 9))
    assert len(zstream(far.tobytes(), 9)) < 40000          # back-references, not stored blocks
    check(b)


@gpu
def test_matches_at_distance_32768_in_the_region_and_in_the_ring():
    # hand-made fixed blocks (zlib never writes these distances): 32767 and 32768, with code 29's 13 extra bits
    rng = np.random.default_rng(18)
    lit = bytes(rng.integers(0, 256, 34000).astype(np.uint8))
    far = [(258, 32768), (258, 32767), (3, 32768), (100, 32767)]
    s, out = match_stream([lit[:32768]] + far + [lit[:77]])
    a = np.frombuffer(out, np.uint8).reshape(1, -1)         # one row: every match lands in the chunk's region
    check(make_tiff(a, 1, ("strips", 1), encode=lambda raw, k: s))
    # a 16 x 16 chunk (256 bytes) whose stream goes on for 33 KB more: the far matches read from and write to the ring
    tile = np.frombuffer(lit[:256], np.uint8).reshape(16, 16)
    s, out = match_stream([lit[:256], lit[1000:34000]] + far + [lit[:9]])
    assert out[:256] == lit[:256] and 256 + 33000 - 32768 >= 256     # the first far match reads past the region
    check(make_tiff(tile, 1, ("strips", 16), encode=lambda raw, k: s))
    wrong = s[:-4] + bytes(4)                              # the ring's bytes count in the Adler-32
    assert decode(make_tiff(tile, 1, ("strips", 16), encode=lambda raw, k: wrong))[0] == _lib.AMB_ERR_CORRUPT_DATA
    # distance 32768 with only 32767 bytes out: one byte before the start
    s, _ = match_stream([lit[:32767], (3, 32768)])
    a = np.frombuffer(lit[:32767], np.uint8).reshape(1, -1)
    st, _, untouched = decode(make_tiff(a, 1, ("strips", 1), encode=lambda raw, k: s))
    assert st == _lib.AMB_ERR_CORRUPT_DATA and untouched


@gpu
@pytest.mark.parametrize("dist", ["none", "single"])
def test_hand_made_dynamic_blocks(dist):
    a = sample_raster(np.uint8, 9, 41, seed=8)
    a[3:5] = 9
    check(make_tiff(a, 1, ("strips", 9), encode=lambda raw, k: dynamic_stream(raw, dist, junk=b"\x01junk")))


@gpu
def test_junk_after_the_stream_and_more_bytes_than_the_chunk_needs():
    a = sample_raster(np.int16, 30, 50, seed=9)
    rng = np.random.default_rng(9)
    check(make_tiff(a, 2, ("strips", 7), encode=lambda raw, k: zstream(raw) + bytes(rng.integers(0, 256, 5 + k,
                                                                                                 ).astype(np.uint8))))
    # each chunk inflates past its bytes by up to 70000 bytes: the excess goes to the ring and its Adler-32 still counts
    extra = lambda raw, k: zstream(raw + bytes(rng.integers(0, 256, 70000 * (k % 2)).astype(np.uint8)) + raw * 3)
    check(make_tiff(a, 2, ("tiles", 16, 16), encode=extra))
    check(make_tiff(a, 2, ("tiles", 16, 16), compression=1,
                    encode=lambda raw, k: raw + b"\x55" * k))  # uncompressed chunks longer than needed


@gpu
def test_uncompressed_chunks_that_share_their_bytes():
    # deduplicated tiles: every tile's offset points at the same bytes of the file; predictor 3 must not sum them twice
    tile = sample_raster(np.float32, 16, 16, 2, seed=19)
    a = np.tile(tile, (3, 4, 1))
    b = make_tiff(a, 3, ("tiles", 16, 16), compression=1)
    t = io.tiff_layout(b, 1)
    L = t.c_layout()
    L._keep[0][:] = L._keep[0][0]
    for win in (None, (5, 40, 3, 60)):
        st, got, _ = decode(b, 1, window=win, layout=L)
        want = a[:, :, 1] if win is None else a[win[0]:win[1], win[2]:win[3], 1]
        assert st == 0
        same(got, want)


@gpu
def test_tiny_odd_and_one_strip_rasters():
    for h, w in ((1, 1), (1, 7), (7, 1), (3, 5), (17, 33)):
        a = sample_raster(np.float32, h, w, seed=h * w)
        check(make_tiff(a, 3, ("strips", h)))
        check(make_tiff(a, 3, ("tiles", 16, 16)))
    a = sample_raster(np.float32, 200, 301, seed=3)
    check(make_tiff(a, 3, ("strips", 200)))              # one stream for the whole image
    check(make_tiff(a, 3, ("strips", 1)))


@gpu
def test_windows_of_a_file():
    a = sample_raster(np.float32, 70, 90, 2, seed=4)
    for chunk in (("strips", 9), ("tiles", 16, 32)):
        b = make_tiff(a, 3, chunk, shuffle=True)         # chunks stored out of order in the file
        for win in ((0, 1, 0, 1), (5, 6, 0, 90), (0, 70, 89, 90), (13, 40, 17, 66), (69, 70, 80, 90)):
            check(b, 1, window=win)


@gpu
def test_opencv_and_pil_files():
    if cv2 is None:
        pytest.skip("OpenCV is not installed")
    import tempfile
    for dtype in (np.uint8, np.int16, np.uint16, np.int32):
        a = sample_raster(dtype, 45, 67, seed=2)[:, :, 0]
        for comp in (8, 32946):
            ok, enc = cv2.imencode(".tiff", a, [cv2.IMWRITE_TIFF_COMPRESSION, comp, cv2.IMWRITE_TIFF_PREDICTOR, 2])
            b = enc.tobytes()
            st, got, _ = decode(b)
            assert st == 0 and np.array_equal(got, cv2.imdecode(enc, cv2.IMREAD_UNCHANGED).astype(np.float32))
            check(b)
    from PIL import Image
    for dtype in (np.float32, np.int16, np.uint16, np.uint8):
        a = sample_raster(dtype, 29, 31, seed=6)[:, :, 0]
        with tempfile.NamedTemporaryFile(suffix=".tif") as fh:
            Image.fromarray(a).save(fh.name, compression="tiff_adobe_deflate")
            b = open(fh.name, "rb").read()
        check(b)
        st, got, _ = decode(b)
        same(got, a.astype(np.float32))


def dem_map(rows=40, cols=56, res=0.5, center=(464500.0, 5272500.0), seed=1):
    """A device-resident map whose elevation holds a DEM with NaN holes, and its host copy."""
    gm = amb.AerialGridMap(amb.GridMapSettings(center[0], center[1], rows * res, cols * res, res)).getMutable()
    e = sample_raster(np.float32, rows, cols, seed=seed)[:, :, 0]
    gm["elevation"] = np.asfortranarray(e)
    gm["ortho"] = np.asfortranarray(np.where(np.isnan(e), 0, np.abs(e) % 256).astype(np.float32))
    gm.to_device(0, names=("elevation", "ortho"))
    return gm


def fresh_map(like, col_range=None):
    g = like.geometry
    gm = amb.AerialGridMap(amb.GridMapSettings(g.pos_x, g.pos_y, g.length_x, g.length_y, g.resolution)).getMutable()
    gm["elevation"] = np.full(gm.getSize(), np.float32(-5.5), order="F")
    gm.to_device(0, col_range=col_range, names=("elevation",))
    return gm


def layer(gm, name="elevation"):
    gm.download((name,))
    return np.array(gm[name], copy=True)


@gpu
def test_files_the_project_writes(tmp_path):
    gm = dem_map()
    for name, fmt, nd in (("elevation", "f32", "nan"), ("ortho", "gray8", None), ("elevation", "mask8", None)):
        p = str(tmp_path / ("%s.tif" % fmt))
        gm.to_geotiff(p, name, fmt=fmt, nodata=nd, rows_per_strip=7)
        check(open(p, "rb").read())
        p = str(tmp_path / ("%s_cog.tif" % fmt))
        gm.to_cog(p, name, fmt=fmt, nodata=nd, tile_size=16)
        b = open(p, "rb").read()
        n_levels = len(io.cog_layout(56, 40, 16))
        assert n_levels >= 3
        for k in range(n_levels):
            check(b, 0, k)


def import_both(b, gm_like, resample="bilinear", overview=0, col_range=None, kind=None):
    """(layer after from_geotiff, layer after from_raster of read_geotiff's array) on fresh maps like gm_like."""
    a, gt, _, nd = _read(b, overview)
    g1 = fresh_map(gm_like, col_range)
    g1.from_geotiff("elevation", b if kind is None else kind(b), overview=overview, resample=resample)
    g2 = fresh_map(gm_like, col_range)
    g2.from_raster("elevation", a.astype(np.float32), gt, nodata=nd, resample=resample)
    return layer(g1), layer(g2)


def _read(b, overview=0):
    import tempfile
    with tempfile.NamedTemporaryFile(suffix=".tif") as fh:
        fh.write(b)
        fh.flush()
        return io.read_geotiff(fh.name, 0, overview)


@gpu
@pytest.mark.parametrize("resample", ["bilinear", "nearest"])
def test_imports_equal_from_raster(resample):
    gm = dem_map()
    g = gm.geometry
    west, north = g.pos_x - g.length_x / 2, g.pos_y + g.length_y / 2
    for gt, dtype, nd in (((west + 0.3, 0.37, 0.0, north - 1.1, 0.0, -0.41), np.float32, "nan"),
                          ((west - 3.0, 0.5, 0.0, north + 2.0, 0.0, -0.5), np.int16, -7),
                          ((west + 5.0, 1.3, 0.0, north, 0.0, -0.9), np.float64, None)):
        a = sample_raster(dtype, 33, 47, seed=11)[:, :, 0]
        if dtype == np.int16:
            a[::5, ::3] = -7
        for chunk in (("strips", 5), ("tiles", 16, 16)):
            b = make_tiff(a, 3 if np.dtype(dtype).kind == "f" else 2, chunk, gt=gt, nodata=nd)
            got, want = import_both(b, gm, resample)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@gpu
def test_corrupt_chunks_write_nothing():
    a = sample_raster(np.float32, 24, 40, seed=12)[:, :, 0]
    raw_chunk = predict(a[8:16, :, None], 3)
    gm = dem_map()
    g = gm.geometry
    gt = (g.pos_x - g.length_x / 2, 0.5, 0.0, g.pos_y + g.length_y / 2, 0.0, -0.5)
    for name, bad in corrupt_streams(raw_chunk):
        b = make_tiff(a, 3, ("strips", 8), gt=gt, encode=lambda raw, k: bad if k == 1 else zstream(raw))
        st, _, untouched = decode(b)
        assert st == _lib.AMB_ERR_CORRUPT_DATA and untouched, name
        g1 = fresh_map(gm)
        before = layer(g1)
        with pytest.raises(amb.AmbError) as e:
            g1.from_geotiff("elevation", b)
        assert e.value.status == _lib.AMB_ERR_CORRUPT_DATA, name
        assert np.array_equal(layer(g1).view(np.uint32), before.view(np.uint32)), name
    b = make_tiff(a, 3, ("strips", 8), compression=1, encode=lambda raw, k: raw[:-1] if k == 2 else raw)
    assert decode(b)[0] == _lib.AMB_ERR_CORRUPT_DATA


@gpu
def test_layouts_inconsistent_with_the_file_are_refused():
    a = sample_raster(np.uint16, 20, 20)
    b = make_tiff(a, 2, ("tiles", 16, 16))
    t = io.tiff_layout(b)
    for field, value in (("n_chunks", 3), ("band", 1), ("spp", 0), ("sample", 9), ("compression", 5),
                         ("predictor", 3), ("tiled", 0), ("chunk_width", 0)):
        L = t.c_layout()
        setattr(L, field, value)
        st, _, untouched = decode(b, layout=L)
        assert st == _lib.AMB_ERR_INVALID_ARGUMENT and untouched, field
    L = t.c_layout()
    L._keep[0][3] = len(b) - 2                           # a chunk past the end of the file
    assert decode(b, layout=L)[0] == _lib.AMB_ERR_INVALID_ARGUMENT
    assert decode(b, window=(0, 21, 0, 5))[0] == _lib.AMB_ERR_INVALID_ARGUMENT


@gpu
def test_only_the_window_is_read():
    gm = dem_map(rows=40, cols=40, res=1.0)
    g = gm.geometry
    west, north = g.pos_x - g.length_x / 2, g.pos_y + g.length_y / 2
    a = sample_raster(np.float32, 160, 160, seed=13)[:, :, 0]
    gt = (west, 1.0, 0.0, north, 0.0, -1.0)             # the map covers the top-left 40 x 40 pixels: tiles 0, 1, 10, 11
    clean = make_tiff(a, 3, ("tiles", 16, 16), gt=gt)
    across = 10
    inside = {r * across + c for r in range(3) for c in range(3)}
    b = make_tiff(a, 3, ("tiles", 16, 16), gt=gt,
                  encode=lambda raw, k: zstream(raw) if k in inside else b"\x00corrupt")
    for resample in ("bilinear", "nearest"):
        g1 = fresh_map(gm)
        g1.from_geotiff("elevation", b, resample=resample)
        _, want = import_both(clean, gm, resample)
        assert np.array_equal(layer(g1).view(np.uint32), want.view(np.uint32))
    # no overlap: nothing is read, nothing written
    far = make_tiff(a, 3, ("tiles", 16, 16), gt=(west + 1e5, 1.0, 0.0, north, 0.0, -1.0),
                    encode=lambda raw, k: b"\x00corrupt")
    g1 = fresh_map(gm)
    g1.from_geotiff("elevation", far)
    assert np.all(layer(g1) == np.float32(-5.5))


@gpu
def test_round_trip_of_a_dsm_and_the_orthomosaic_on_it(tmp_path):
    rows, cols, res = 64, 64, 1.0
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0)
    xyz = synth.point_cloud(6000, 32.0, 32.0, seed=11)
    amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
    elev = layer(gm)
    elev_f = np.asfortranarray(elev)
    elev_f[3, 4] = -0.0
    gm["elevation"] = elev_f
    gm.upload(("elevation",))
    elev = layer(gm)
    p = str(tmp_path / "dsm.tif")
    gm.to_cog(p, "elevation", nodata="nan", tile_size=16)
    g2 = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res)).getMutable()
    g2.to_device(0)
    g2.from_geotiff("elevation", p)
    back = layer(g2)
    assert np.array_equal(back.view(np.uint32), elev.view(np.uint32))
    assert np.signbit(back[3, 4]) and back[3, 4] == 0
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(2, 3, 32.0, 32.0, agl=60.0, seed=4, jitter_pos=0.5)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"]) for k in range(len(poses))]
    for m in (gm, g2):
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), m).process(poses, imgs, m)
    for name in ("ortho", "observation_index", "elevation_angle"):
        assert np.array_equal(layer(gm, name).view(np.uint32), layer(g2, name).view(np.uint32)), name


@gpu
def test_stripes_multi_and_staging():
    gm = dem_map(rows=48, cols=50, seed=3)
    g = gm.geometry
    gt = (g.pos_x - g.length_x / 2 - 0.7, 0.45, 0.0, g.pos_y + g.length_y / 2 + 0.3, 0.0, -0.45)
    a = sample_raster(np.float32, 70, 60, seed=14)[:, :, 0]
    b = make_tiff(a, 3, ("strips", 6), gt=gt, nodata="nan")
    whole, want = import_both(b, gm)
    assert np.array_equal(whole.view(np.uint32), want.view(np.uint32))
    for kind in (bytearray, lambda x: memoryview(bytearray(x)), lambda x: np.frombuffer(x, np.uint8)):
        got, _ = import_both(b, gm, kind=kind)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    for c0, c1 in ((0, 17), (17, 50), (20, 21)):          # stripe contexts write their columns of the whole import
        got, _ = import_both(b, gm, col_range=(c0, c1))
        assert np.array_equal(got[:, c0:c1].view(np.uint32), want[:, c0:c1].view(np.uint32))
    t = io.tiff_layout(b)
    L = t.c_layout()
    m = C.c_void_p()
    assert _lib.lib().amb_multi_create(C.byref(g), 1, C.byref(m)) == 0
    try:
        host = np.full(g.rows * g.cols, np.float32(-5.5))
        assert _lib.lib().amb_multi_upload_layer(m, _lib.LAYER_ID["elevation"], host.ctypes.data_as(C.c_void_p)) == 0
        for kind in ("pageable", "pinned", "bytes"):
            f = HostFile(b, kind)
            st = _lib.lib().amb_multi_import_tiff(m, _lib.LAYER_ID["elevation"], C.c_void_p(f.ptr), f.size, C.byref(L),
                                                  (C.c_double * 6)(*gt), 0, 0.0, 1)
            f.free()
            assert st == 0
            out = np.empty_like(host)
            assert _lib.lib().amb_multi_download_layer(m, _lib.LAYER_ID["elevation"],
                                                       out.ctypes.data_as(C.c_void_p)) == 0
            assert np.array_equal(out.reshape(g.cols, g.rows).T.view(np.uint32), want.view(np.uint32))
    finally:
        _lib.lib().amb_multi_destroy(m)
    for kind in ("pinned", "bytes"):
        check(b, kind=kind)


@gpu
def test_a_corrupt_chunk_stops_only_the_stripe_whose_window_holds_it():
    gm = dem_map(rows=48, cols=50, seed=4)
    g = gm.geometry
    gt = (g.pos_x - g.length_x / 2, 0.5, 0.0, g.pos_y + g.length_y / 2, 0.0, -0.5)   # the map's own grid
    a = sample_raster(np.float32, 50, 48, seed=16)[:, :, 0]  # raster row r is map column r
    clean = make_tiff(a, 3, ("strips", 5), gt=gt)
    bad = make_tiff(a, 3, ("strips", 5), gt=gt, encode=lambda raw, k: zstream(raw)[:-1] if k == 9 else zstream(raw))
    _, want = import_both(clean, gm)
    north, south = fresh_map(gm, (0, 25)), fresh_map(gm, (25, 50))
    north.from_geotiff("elevation", bad)                   # its window ends at row 24: strip 9 is never read
    assert np.array_equal(layer(north)[:, :25].view(np.uint32), want[:, :25].view(np.uint32))
    before = layer(south)
    with pytest.raises(amb.AmbError) as e:
        south.from_geotiff("elevation", bad)
    assert e.value.status == _lib.AMB_ERR_CORRUPT_DATA
    assert np.array_equal(layer(south).view(np.uint32), before.view(np.uint32))
    if _lib.lib().amb_device_count() < 2:
        pytest.skip("amb_multi_import_tiff over two stripes needs two devices")
    m = C.c_void_p()
    assert _lib.lib().amb_multi_create(C.byref(g), 2, C.byref(m)) == 0
    try:
        host = np.full(g.rows * g.cols, np.float32(-5.5))
        assert _lib.lib().amb_multi_upload_layer(m, _lib.LAYER_ID["elevation"], host.ctypes.data_as(C.c_void_p)) == 0
        f = HostFile(bad)
        L = io.tiff_layout(bad).c_layout()
        st = _lib.lib().amb_multi_import_tiff(m, _lib.LAYER_ID["elevation"], C.c_void_p(f.ptr), f.size, C.byref(L),
                                              (C.c_double * 6)(*gt), 0, 0.0, 1)
        assert st == _lib.AMB_ERR_CORRUPT_DATA
        out = np.empty_like(host)
        assert _lib.lib().amb_multi_download_layer(m, _lib.LAYER_ID["elevation"], out.ctypes.data_as(C.c_void_p)) == 0
        out = out.reshape(g.cols, g.rows).T
        assert np.array_equal(out[:, :25].view(np.uint32), want[:, :25].view(np.uint32))
        assert np.all(out[:, 25:] == np.float32(-5.5))
    finally:
        _lib.lib().amb_multi_destroy(m)


@gpu
def test_read_geotiff_device_returns_a_torch_tensor(tmp_path):
    if EMULATED:
        return   # torch CUDA tensors need a GPU
    a = sample_raster(np.float64, 50, 70, seed=15)[:, :, 0]
    gt = (1000.0, 2.0, 0.0, 5000.0, 0.0, -2.0)
    b = make_tiff(a, 3, ("tiles", 32, 32), gt=gt, nodata="-9999")
    p = tmp_path / "d.tif"
    p.write_bytes(b)
    t, g, epsg, nd = io.read_geotiff_device(str(p))
    assert t.is_cuda and t.dtype.__str__() == "torch.float32" and tuple(t.shape) == (50, 70)
    want, g0, e0, n0 = io.read_geotiff(str(p))
    same(t.cpu().numpy(), want.astype(np.float32), f64=True)
    assert (g, epsg, nd) == (g0, e0, n0)
    with pytest.raises(amb.AmbError) as e:
        io.read_geotiff_device(make_tiff(a, 3, ("tiles", 32, 32), gt=gt, encode=lambda raw, k: raw[:5]))
    assert e.value.status == _lib.AMB_ERR_CORRUPT_DATA


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_geotiff_inflate.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail
