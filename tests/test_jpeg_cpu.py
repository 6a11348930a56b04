"""Host side of the JPEG encoder: amb_jpeg_max_size, io.write_jpeg and its world file, the argument contract of the
Python wrappers, and the fixture tests/golden/jpeg_cases.npz (no GPU needed)."""
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

cv2 = pytest.importorskip("cv2")


def cv2_jpeg(img, quality, sampling, restart):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == 0 else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
    return cv2.imencode(".jpg", img, params)[1].tobytes()


@pytest.mark.parametrize("h,w", [(1, 1), (7, 9), (17, 33), (64, 9), (120, 130)])
def test_max_size_bounds_noise_at_quality_100_with_restart_1(h, w):
    L = _lib.lib()
    rng = np.random.default_rng(h * w)
    for channels, sampling in ((1, 0), (3, 0), (3, 1)):
        img = rng.integers(0, 256, (h, w) if channels == 1 else (h, w, 3)).astype(np.uint8)
        bound = L.amb_jpeg_max_size(w, h, channels, 100, sampling, 1)
        assert bound >= len(cv2_jpeg(img, 100, sampling, 1)) > 0
        checker = np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, 255, 0).astype(np.uint8)
        if channels == 3:
            checker = np.repeat(checker[:, :, None], 3, axis=2)
        assert bound >= len(cv2_jpeg(checker, 100, sampling, 1))


def test_max_size_is_zero_for_unsupported_parameters():
    L = _lib.lib()
    assert L.amb_jpeg_max_size(10, 10, 3, 95, 0, 0) > 0
    for args in ((0, 10, 3, 95, 0, 0), (65536, 10, 1, 95, 0, 0), (10, 10, 2, 95, 0, 0), (10, 10, 3, 0, 0, 0),
                 (10, 10, 3, 101, 0, 0), (10, 10, 3, 95, 2, 0), (10, 10, 3, 95, 0, -1), (10, 10, 3, 95, 0, 65536)):
        assert L.amb_jpeg_max_size(*args) == 0, args


def test_write_jpeg_reads_back_through_opencv_and_pil(tmp_path):
    from PIL import Image
    img = np.add.outer(np.arange(40), np.arange(50)).astype(np.uint8)
    img = np.stack([img, 255 - img, 2 * img], axis=-1)
    data = cv2_jpeg(img, 95, 0, 0)
    path = str(tmp_path / "ortho.jpg")
    io.write_jpeg(path, data)
    assert open(path, "rb").read() == data
    assert not os.path.exists(str(tmp_path / "ortho.jgw"))
    back = cv2.imread(path, cv2.IMREAD_COLOR)
    assert back.shape == img.shape and np.abs(back.astype(int) - img).mean() < 8
    with Image.open(path) as im:
        assert im.format == "JPEG" and im.size == (50, 40) and im.mode == "RGB"
        assert np.array_equal(np.asarray(im)[:, :, ::-1], back)
    with pytest.raises(ValueError):
        io.write_jpeg(path, b"not a jpeg")
    with pytest.raises(ValueError):
        io.write_jpeg(path, data, geotransform=(0, 1, 0, 0, 0))


def test_world_file_locates_pixel_centres(tmp_path):
    g = amb.Geometry()
    L = _lib.lib()
    assert L.amb_geometry_init(37.5, 21.0, 0.5, 464512.25, 5272498.5, C.byref(g)) == 0
    gt = (C.c_double * 6)()
    assert L.amb_raster_geotransform(C.byref(g), gt) == 0
    data = cv2_jpeg(np.zeros((g.cols, g.rows), np.uint8), 95, 0, 0)
    path = str(tmp_path / "map.jpg")
    io.write_jpeg(path, data, geotransform=tuple(gt))
    vals = [float(v) for v in open(str(tmp_path / "map.jgw")).read().split()]
    assert vals == [gt[1], 0.0, 0.0, gt[5], gt[0] + gt[1] / 2, gt[3] + gt[5] / 2]
    # the centre of pixel (r, c) = (0, 0) is the position of cell (rows - 1, 0)
    x, y = C.c_double(), C.c_double()
    assert L.amb_geometry_position(C.byref(g), g.rows - 1, 0, C.byref(x), C.byref(y)) == 0
    assert abs(vals[4] - x.value) < 1e-6 and abs(vals[5] - y.value) < 1e-6


def test_python_argument_contract():
    for bad in (dict(sampling="422"), dict(sampling=420), dict(quality=0), dict(quality=101), dict(quality=95.0),
                dict(quality=True), dict(restart_interval=-1), dict(restart_interval=65536)):
        kw = dict(quality=95, sampling="420", restart_interval=0)
        kw.update(bad)
        with pytest.raises(ValueError):
            api._jpeg_args(10, 10, 3, kw["quality"], kw["sampling"], kw["restart_interval"])
    for w, h in ((0, 5), (5, 0), (65536, 5), (5, 65536)):
        with pytest.raises(ValueError):
            api._jpeg_args(w, h, 1, 95, "420", 0)
    assert api._jpeg_args(65535, 1, 3, 1, "444", 65535) == (65535, 1, 3, 1, 1, 65535)
    with pytest.raises(ValueError):
        amb.encode_jpeg(np.zeros((4, 4), np.uint8))          # not a torch CUDA tensor
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, 5, 4, 1.0)).getMutable()
    with pytest.raises(amb.AmbError) as ei:
        gm.to_jpeg("ortho")
    assert "to_device()" in str(ei.value)


def test_fixture_is_what_opencv_writes():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_jpeg_golden as mg
    z = np.load(mg.OUT)
    live = mg.encode_all()
    assert sorted(z.files) == sorted(live)
    for k in live:
        assert z[k].tobytes() == live[k].tobytes(), k
