"""The per-tile DOMINANCE cull of the orthomosaic's frame list (amb_ortho_set_dominance_cull; csrc/ortho_kernels.cu,
DESIGN.md §4; the default since round 2): it must not change a single output bit.  Both cull modes run through the one
kernel ortho_kernel_dom, the plain list with the dominance switch off.  Every
scenario runs with the cull on and is compared (i) bit for bit with the same run without it (AMB_ORTHO_DOMINANCE=0) and
(ii) with the CPU oracle.  The argument and the expected saving
are also checked on the CPU by tools/ortho_dominance_study.py (oracle restricted to the surviving frames == full
oracle; 8.5 -> 1.2 frames per tile at the benchmark geometry)."""
import os

import numpy as np
import pytest

from common import GOLDEN, ulp_diff
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from test_gpu_ortho import assert_parity, gpu_ortho, make_inputs, oracle_ortho

pytestmark = pytest.mark.gpu

OUT_LAYERS = ("ortho", "colored_ortho", "elevation_angle", "observation_index")


def both(monkeypatch, *args, **kw):
    """The same gpu_ortho() run without and with the dominance cull; asserts bit identity, returns the culled map."""
    monkeypatch.setenv("AMB_ORTHO_DOMINANCE", "0")
    plain = gpu_ortho(*args, **kw)
    monkeypatch.setenv("AMB_ORTHO_DOMINANCE", "1")
    culled = gpu_ortho(*args, **kw)
    for k in OUT_LAYERS:
        assert np.array_equal(plain[k].view(np.uint32), culled[k].view(np.uint32)), k
    return culled


@pytest.mark.parametrize("colored", [False, True])
@pytest.mark.parametrize("dist_type", [0, 1, 2, 3])   # 2 (equidistant), 3 (FOV): inner view CONE instead of the inner rectangle
def test_dominance_cull_changes_nothing(monkeypatch, colored, dist_type):
    rows, cols, res = 200, 160, 0.5
    camd, poses, imgs = make_inputs(rows, cols, res, 3, 4, 60.0, 0.1, colored, dist_type)
    elev = synth.analytic_elevation(rows, cols, res)
    elev[50:60, 70:90] = np.nan
    gm = both(monkeypatch, rows, cols, res, elev, camd, poses, imgs, colored)
    assert_parity(gm, oracle_ortho(rows, cols, res, elev, camd, poses, imgs, colored), colored)


def frames_per_tile(key):
    """tests/emu only: mean length of the tiles' frame lists since the last call (None on the real library)."""
    import ctypes as C
    L = amb.lib()
    if not hasattr(L, "amb_emu_counter"):
        return None
    s, n = C.c_longlong(), C.c_longlong()
    L.amb_emu_counter(key, C.byref(s), C.byref(n))
    return s.value / max(1, n.value)


def test_wide_map_many_frames_where_the_cull_bites(monkeypatch):
    # footprints much smaller than the map, 60 frames: most tiles keep 1-3 of ~10 candidates
    rows, cols, res = 960, 640, 0.5
    camd, poses, imgs = make_inputs(rows, cols, res, 6, 10, 60.0, 0.1, False)
    elev = synth.analytic_elevation(rows, cols, res)
    frames_per_tile(b"ortho_list"), frames_per_tile(b"ortho_dom_list")
    gm = both(monkeypatch, rows, cols, res, elev, camd, poses, imgs, False)
    plain_n, dom_n = frames_per_tile(b"ortho_list"), frames_per_tile(b"ortho_dom_list")
    if plain_n is not None:                  # emulated kernels: the dominance variant really ran, and it culled
        assert 0 < dom_n < plain_n
    assert_parity(gm, oracle_ortho(rows, cols, res, elev, camd, poses, imgs, False), False)
    monkeypatch.setenv("AMB_ORTHO_DOMINANCE", "1")
    brute = gpu_ortho(rows, cols, res, elev, camd, poses, imgs, False, brute=True)   # brute force ignores the cull
    assert np.array_equal(gm["observation_index"], brute["observation_index"], equal_nan=True)


def test_benchmark_like_geometry_keeps_one_or_two_frames_per_tile(monkeypatch):
    # flight height >> tile size, every frame sees every tile (like joint_10k): 30 candidates -> ~2 survivors per tile
    rows, cols, res = 640, 640, 0.25
    camd, poses, imgs = make_inputs(rows, cols, res, 5, 6, 400.0, 0.1, False)
    elev = synth.analytic_elevation(rows, cols, res)
    frames_per_tile(b"ortho_list"), frames_per_tile(b"ortho_dom_list")
    gm = both(monkeypatch, rows, cols, res, elev, camd, poses, imgs, False)
    assert_parity(gm, oracle_ortho(rows, cols, res, elev, camd, poses, imgs, False), False)
    plain_n, dom_n = frames_per_tile(b"ortho_list"), frames_per_tile(b"ortho_dom_list")
    if plain_n is not None:
        assert plain_n > 25 and dom_n < 4


def test_rough_terrain_and_tilted_cameras(monkeypatch):
    # large elevation range per tile (bigger bounding spheres) and strongly tilted views (off-nadir winners)
    rows, cols, res = 320, 256, 1.0
    camd, poses, imgs = make_inputs(rows, cols, res, 3, 5, 80.0, 0.1, True)
    rng = np.random.default_rng(5)
    from scipy.spatial.transform import Rotation as R
    for p in poses:                                   # extra tilt of up to ~15 degrees about a random horizontal axis
        q = R.from_quat([p[4], p[5], p[6], p[3]]) * R.from_rotvec(rng.normal(0, 0.15, 3) * [1, 1, 0])
        x, y, z, w = q.as_quat()
        p[3:7] = (w, x, y, z)
    elev = synth.analytic_elevation(rows, cols, res)
    elev += (25.0 * np.sin(np.arange(rows)[:, None] / 7.0) * np.cos(np.arange(cols)[None, :] / 5.0)).astype(np.float32)
    gm = both(monkeypatch, rows, cols, res, elev, camd, poses, imgs, True)
    assert_parity(gm, oracle_ortho(rows, cols, res, elev, camd, poses, imgs, True), True)


def test_state_in_the_layers_across_calls(monkeypatch):
    # incremental batches: a dominated frame must stay irrelevant when the running best starts from the layer
    rows, cols, res = 256, 256, 0.5
    camd, poses, imgs = make_inputs(rows, cols, res, 4, 5, 50.0, 0.08, False)
    elev = synth.analytic_elevation(rows, cols, res)
    monkeypatch.setenv("AMB_ORTHO_DOMINANCE", "1")
    gm = None
    L = None
    for lo, hi in ((0, 7), (7, 12), (12, 20)):
        gm = gpu_ortho(rows, cols, res, elev, camd, poses[lo:hi], imgs[lo:hi], False, gm=gm)
        L = oracle_ortho(rows, cols, res, elev, camd, poses[lo:hi], imgs[lo:hi], False, L=L)
        assert_parity(gm, L, False)


@pytest.mark.parametrize("colored", [False, True])
def test_golden_fixture_with_the_cull(monkeypatch, colored):
    monkeypatch.setenv("AMB_ORTHO_DOMINANCE", "1")
    z = np.load(os.path.join(GOLDEN, "ortho_color_96x80.npz" if colored else "ortho_gray_96x80.npz"))
    rows, cols, res = int(z["rows"]), int(z["cols"]), float(z["res"])
    camd = synth.scaled_camera(float(z["cam_scale"]), dist_type=1)
    ch = 3 if colored else 1
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(z["poses"]))]
    gm = gpu_ortho(rows, cols, res, z["elevation"], camd, z["poses"], imgs, colored)
    assert np.array_equal(gm["observation_index"], z["observation_index"], equal_nan=True)
    assert np.array_equal(gm["colored_ortho" if colored else "ortho"].view(np.uint32), z["out"])
    assert ulp_diff(gm["elevation_angle"], z["elevation_angle"]).max() <= 1


def test_resident_frames_path_with_the_cull(monkeypatch):
    # frames already in HBM (the fused kernel, SELECT = false): amb_ortho_process_device
    emulated = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")   # tests/emu: host memory IS device memory
    torch = None if emulated else pytest.importorskip("torch")
    rows, cols, res = 256, 192, 0.5
    camd, poses, imgs = make_inputs(rows, cols, res, 3, 5, 60.0, 0.1, False)
    elev = synth.analytic_elevation(rows, cols, res)
    outs = []
    for flag in ("0", "1"):
        monkeypatch.setenv("AMB_ORTHO_DOMINANCE", flag)
        gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
        gm["elevation"] = elev
        gm.to_device(0)
        d_imgs = imgs if emulated else [torch.from_numpy(im).cuda() for im in imgs]
        o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm)
        o.process_device(poses, [im.ctypes.data if emulated else im.data_ptr() for im in d_imgs], camd["width"], gm)
        gm.download()
        outs.append(gm)
    for k in ("ortho", "elevation_angle", "observation_index"):
        assert np.array_equal(outs[0][k].view(np.uint32), outs[1][k].view(np.uint32)), k
    assert_parity(outs[1], oracle_ortho(rows, cols, res, elev, camd, poses, imgs, False), False)
