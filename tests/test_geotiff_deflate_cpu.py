"""The host side of Deflate GeoTIFFs, no GPU: io.write_geotiff_strips around strips made here with host zlib (the
device encoder's own strips are checked in test_gpu_geotiff_deflate.py), the file layout shared with write_geotiff, the
size bound of amb_deflate_max_size and the Python argument contract."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from aerial_mapper_b200 import api, io  # noqa: E402
from test_gpu_geotiff_deflate import bound, predict  # noqa: E402

GT = (500000.0, 0.25, 0.0, 5200000.0, 0.0, -0.25)


def rasters(h=37, w=23, seed=0):
    rng = np.random.default_rng(seed)
    dem = rng.normal(400.0, 3.0, (h, w)).astype(np.float32)
    dem[rng.random((h, w)) < 0.1] = np.nan
    dem.view(np.uint32)[0, 0] = 0x7fc00123                 # a NaN payload
    return {"f32": dem, "gray8": rng.integers(0, 256, (h, w)).astype(np.uint8),
            "bgr8": rng.integers(0, 256, (h, w, 3)).astype(np.uint8),
            "mask8": np.where(np.isnan(dem), 0, 255).astype(np.uint8)}


def host_strips(img, fmt, rps):
    pred = predict(img, fmt)
    strips = [zlib.compress(pred[s:s + rps].tobytes(), 6) for s in range(0, pred.shape[0], rps)]
    return b"".join(strips), np.array([len(s) for s in strips], np.uint32)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        return a.shape == b.shape and np.array_equal(a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("fmt", ["f32", "gray8", "bgr8", "mask8"])
@pytest.mark.parametrize("rps", [1, 7, 37, 100])
def test_strips_read_back_through_every_reader(tmp_path, fmt, rps):
    img = rasters()[fmt]
    data, counts = host_strips(img, fmt, min(rps, 37))
    path = str(tmp_path / "a.tif")
    io.write_geotiff_strips(path, data, counts, 23, 37, fmt, rps, GT, epsg=25832, nodata="nan" if fmt == "f32" else None)
    bands = 3 if fmt == "bgr8" else 1
    a = np.stack([io.read_geotiff(path, band=k)[0] for k in range(bands)], axis=-1)
    a = a[:, :, ::-1] if bands == 3 else a[:, :, 0]
    assert same_bits(a, img)
    _, gt, epsg, nodata = io.read_geotiff(path)
    assert gt == GT and epsg == 25832 and (nodata is None) == (fmt != "f32")
    cv2 = pytest.importorskip("cv2")
    assert same_bits(cv2.imread(path, cv2.IMREAD_UNCHANGED), img)
    Image = pytest.importorskip("PIL.Image")
    im = np.asarray(Image.open(path))
    assert same_bits(im[:, :, ::-1] if bands == 3 else im, img)


def test_tags_equal_write_geotiffs_but_for_the_layout(tmp_path):
    for fmt, img in rasters().items():
        plain, packed = str(tmp_path / "plain.tif"), str(tmp_path / "deflate.tif")
        io.write_geotiff(plain, img, GT, nodata="nan")
        data, counts = host_strips(img, fmt, 5)
        io.write_geotiff_strips(packed, data, counts, 23, 37, fmt, 5, GT, nodata="nan")
        want, got = io._read_ifd(open(plain, "rb").read()), io._read_ifd(open(packed, "rb").read())
        layout = {259, 273, 278, 279, 317}
        assert {k: v for k, v in want.items() if k not in layout} == {k: v for k, v in got.items() if k not in layout}
        assert got[259] == (8,) and got[317] == ((3,) if fmt == "f32" else (2,)) and got[278] == (5,)
        assert got[279] == tuple(int(c) for c in counts)
        raw = open(packed, "rb").read()
        assert raw[got[273][0]:got[273][0] + int(counts[0])] == data[:int(counts[0])]


def test_write_geotiff_bytes_are_unchanged(tmp_path):
    """The uncompressed layout, restated: header, IFD at 8, values, strips from a 16-byte boundary, RGB strips."""
    img = rasters(3, 4)["bgr8"]
    path = str(tmp_path / "a.tif")
    io.write_geotiff(path, img, GT)
    raw = open(path, "rb").read()
    tags = io._read_ifd(raw)
    assert raw[:8] == b"II*\0\x08\0\0\0" and struct.unpack_from("<H", raw, 8)[0] == 14 and 317 not in tags
    assert tags[259] == (1,) and tags[278] == (3,) and tags[279] == (36,) and tags[273][0] % 16 == 0
    assert raw[tags[273][0]:] == img[:, :, ::-1].tobytes()


def test_geotiff_strips_argument_checks(tmp_path):
    img = rasters()["gray8"]
    data, counts = host_strips(img, "gray8", 5)
    path = str(tmp_path / "a.tif")
    with pytest.raises(ValueError):
        io.write_geotiff_strips(path, data[:-1], counts, 23, 37, "gray8", 5, GT)
    with pytest.raises(ValueError):
        io.write_geotiff_strips(path, data, counts[:-1], 23, 37, "gray8", 5, GT)
    with pytest.raises(ValueError):
        io.write_geotiff_strips(path, data, counts, 23, 37, "gray8", 5, (0.0, 1.0, 0.1, 0.0, 0.0, -1.0))
    with pytest.raises(KeyError):
        io.write_geotiff_strips(path, data, counts, 23, 37, "rgb8", 5, GT)
    big = [0xFFFFFF00] * 2
    with pytest.raises(ValueError, match="4 GiB"):
        io._tiff_layout(65535, 2, 1, 8, 1, big, GT, 32632, None, 2)
    assert not os.path.exists(path)


def test_default_rows_per_strip_is_libtiffs():
    assert api._deflate_rows(40000, 10000, None) == 1
    assert api._deflate_rows(10000, 10000, None) == 1
    assert api._deflate_rows(1000, 10000, None) == 8
    assert api._deflate_rows(1, 3, None) == 3
    assert api._deflate_rows(4, 100, 1000) == 100
    for bad in (0, -1, 1.5, True, "8"):
        with pytest.raises(ValueError):
            api._deflate_rows(4, 100, bad)


def test_max_size_is_the_sum_of_the_strip_bounds():
    from aerial_mapper_b200 import _lib
    L = _lib.lib()
    for w, h, fmt, rps in ((10000, 10000, "f32", 1), (10000, 7, "bgr8", 3), (1, 1, "gray8", 1), (70000, 3, "mask8", 5),
                           (16384, 4096, "f32", 4096)):
        f = _lib.RASTER_FORMAT[fmt]
        row = w * _lib.RASTER_BPP[f]
        r = min(rps, h)
        want = sum(bound(min(r, h - s) * row) for s in range(0, h, r))
        assert L.amb_deflate_max_size(w, h, f, rps) == want, (w, h, fmt, rps)
    assert L.amb_deflate_max_size(65535, 65535, _lib.RASTER_F32, 65535) == 0   # a 17 GB strip: TIFF cannot count it
    assert L.amb_deflate_max_size(65535, 65535, _lib.RASTER_F32, 1) > 0
