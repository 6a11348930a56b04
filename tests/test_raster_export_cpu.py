"""The host side of the raster export, without a GPU: the geotransform against amb_geometry_position, io.write_geotiff
read back by OpenCV and PIL, and the gray8 restatement of tests/test_gpu_raster_export.py against OpenCV itself."""
import ctypes as C

import numpy as np
import pytest

import aerial_mapper_b200 as amb
from aerial_mapper_b200 import _lib
from aerial_mapper_b200.io import write_geotiff
from test_gpu_raster_export import restate

cv2 = pytest.importorskip("cv2")


def geometry(rows, cols, res, center):
    g = amb.Geometry()
    assert _lib.lib().amb_geometry_init(rows * res, cols * res, res, center[0], center[1], C.byref(g)) == 0
    assert (g.rows, g.cols) == (rows, cols)
    return g


@pytest.mark.parametrize("rows,cols,res,center", [(7, 5, 1.0, (0.0, 0.0)), (31, 17, 0.3, (12.7, -41.9)),
                                                  (1001, 999, 0.25, (464500.0, 5272500.0)),
                                                  (3, 9, 0.1, (464499.95, 5272700.05))])
def test_geotransform_centres_are_the_cell_positions(rows, cols, res, center):
    L = _lib.lib()
    g = geometry(rows, cols, res, center)
    gt = (C.c_double * 6)()
    assert L.amb_raster_geotransform(C.byref(g), gt) == 0
    assert gt[2] == 0.0 and gt[4] == 0.0 and gt[1] == res and gt[5] == -res
    rng = np.random.default_rng(rows)
    pixels = [(0, 0), (0, rows - 1), (cols - 1, 0), (cols - 1, rows - 1)] + \
        [(int(rng.integers(cols)), int(rng.integers(rows))) for _ in range(200)]
    x, y = C.c_double(), C.c_double()
    for r, c in pixels:
        assert L.amb_geometry_position(C.byref(g), rows - 1 - c, r, C.byref(x), C.byref(y)) == 0
        px, py = gt[0] + (c + 0.5) * gt[1], gt[3] + (r + 0.5) * gt[5]
        assert abs(px - x.value) <= 4 * np.spacing(abs(x.value)) + 4 * np.spacing(res), (r, c, px, x.value)
        assert abs(py - y.value) <= 4 * np.spacing(abs(y.value)) + 4 * np.spacing(res), (r, c, py, y.value)


def test_python_geotransform_and_resident_only_export():
    gm = amb.AerialGridMap(amb.GridMapSettings(464500.0, 5272500.0, 100.0, 60.0, 0.5)).getMutable()
    assert gm.geotransform() == (464450.0, 0.5, 0.0, 5272530.0, 0.0, -0.5)
    with pytest.raises(amb.AmbError) as ei:
        gm.to_raster("ortho", "gray8")
    assert "to_device()" in str(ei.value)


def test_gray8_restatement_is_opencv_saturate_cast():
    ties = np.arange(-4, 260, dtype=np.float32) + np.float32(0.5)
    odd = np.float32([np.nan, np.inf, -np.inf, -0.0, 2.0 ** 31, 2.0 ** 31 - 128, 3e9, -3e9, 1e-45, 255.49998,
                      0.49999997, 0.50000006]).astype(np.float32)
    bits = np.uint32([0x7FC00000, 0xFFC00001, 0x7F800001, 0x00123456]).view(np.float32)
    v = np.concatenate([ties, odd, bits, np.random.default_rng(1).uniform(-300, 600, 5000).astype(np.float32)])
    layer = v.reshape(-1, 1)                       # one column: the exported row is the values reversed
    assert np.array_equal(restate(layer, "gray8")[0, ::-1], cv2.add(v.reshape(1, -1), 0, dtype=cv2.CV_8U)[0])


GT = (464450.0, 0.5, 0.0, 5272530.0, 0.0, -0.5)


@pytest.mark.parametrize("h,w", [(1, 1), (7, 13), (300, 1111)])
def test_geotiff_round_trips_through_opencv(tmp_path, h, w):
    rng = np.random.default_rng(h * w)
    gray = rng.integers(0, 256, (h, w), dtype=np.uint8)
    bgr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    dem = rng.normal(400.0, 30.0, (h, w)).astype(np.float32)
    dem[rng.random((h, w)) < 0.2] = np.nan
    for name, a, nodata in (("gray", gray, None), ("bgr", bgr, None), ("dem", dem, "nan")):
        path = str(tmp_path / (name + ".tif"))
        write_geotiff(path, a, GT, nodata=nodata)
        back = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        assert back is not None and back.dtype == a.dtype and back.shape == a.shape, name
        assert back.tobytes() == np.ascontiguousarray(a).tobytes(), name      # cv2 returns B, G, R: the input's order


def test_geotiff_tags(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    path = str(tmp_path / "dem.tif")
    dem = np.full((40, 30), 12.5, np.float32)
    write_geotiff(path, dem, GT, epsg=32633, nodata="nan")
    with Image.open(path) as im:
        tags = im.tag_v2
        assert tuple(tags[33550]) == (0.5, 0.5, 0.0)
        assert tuple(tags[33922]) == (0.0, 0.0, 0.0, 464450.0, 5272530.0, 0.0)
        assert tuple(tags[34735]) == (1, 1, 0, 3, 1024, 0, 1, 1, 1025, 0, 1, 1, 3072, 0, 1, 32633)
        assert tags[42113] == "nan"
        assert tuple(np.ravel(tags[339])) == (3,) and tuple(np.ravel(tags[258])) == (32,) and im.size == (30, 40)
    path = str(tmp_path / "rgb.tif")
    write_geotiff(path, np.zeros((4, 5, 3), np.uint8), GT)
    with Image.open(path) as im:
        assert im.mode == "RGB" and 42113 not in im.tag_v2 and tuple(im.tag_v2[34735])[-1] == 32632


def test_geotiff_refuses_what_it_cannot_write(tmp_path):
    path = str(tmp_path / "x.tif")
    huge = np.broadcast_to(np.uint8(7), (70000, 70000))          # 4.9 GB, not allocated
    with pytest.raises(ValueError, match="4 GiB"):
        write_geotiff(path, huge, GT)
    with pytest.raises(ValueError):
        write_geotiff(path, np.zeros((4, 4), np.float64), GT)
    with pytest.raises(ValueError):
        write_geotiff(path, np.zeros((4, 4), np.uint8), (0.0, 1.0, 0.1, 0.0, 0.0, -1.0))
