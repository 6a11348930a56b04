"""The deferred layer reset (amb_init_layers marks the slabs fresh; the first reader fills them, and the DSM and the
orthomosaic store the initial values themselves where they have no result) against the eager reset
(AMB_EAGER_LAYER_INIT=1: one fill per slab inside amb_init_layers): every sequence below must leave every layer and
every read path bit for bit as the eager reset does.  The library reads the switch at amb_create, so each case runs
twice in this process, on a context created under each setting.

Before the reset the layers hold a poison pattern (a NaN with a payload no kernel writes), so a cell that a writer
leaves unwritten shows up instead of passing as a leftover correct value."""
import ctypes as C
import os

import numpy as np
import pytest

import aerial_mapper_b200 as amb
from aerial_mapper_b200 import _lib, synth

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
POISON = np.array([0x7FA5A5A5], np.uint32).view(np.float32)[0]
ORTHO_LAYERS = ("elevation", "elevation_angle", "observation_index", "ortho", "colored_ortho")


def both(case, *args):
    """case(*args) with the deferred and with the eager reset: the two results, dicts of arrays, must match bit for bit."""
    out = {}
    for eager in ("0", "1"):
        os.environ["AMB_EAGER_LAYER_INIT"] = eager
        try:
            out[eager] = case(*args)
        finally:
            os.environ.pop("AMB_EAGER_LAYER_INIT", None)
    lazy, ref = out["0"], out["1"]
    assert sorted(lazy) == sorted(ref)
    for name in ref:
        a, b = np.asarray(lazy[name]), np.asarray(ref[name])
        assert a.shape == b.shape and a.dtype == b.dtype, name
        bits = (lambda x: x.view(np.uint32)) if a.dtype == np.float32 else (lambda x: x)
        diff = np.count_nonzero(bits(np.ascontiguousarray(a)) != bits(np.ascontiguousarray(b)))
        assert diff == 0, "%s: %d cells differ from the eager reset" % (name, diff)
    return ref


def resident_map(rows, cols, res=1.0, col_range=None, names=ORTHO_LAYERS, poison=True):
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res), layer_names=names).getMutable()
    if poison:
        for name in names:
            gm[name] = POISON
    gm.to_device(0, col_range=col_range, names=names)
    return gm


def init(gm):
    amb.check(amb.lib().amb_init_layers(gm.context()), gm.context())


def download(gm, names=ORTHO_LAYERS, tag=""):
    gm.download(names)
    c0, c1 = gm._col_range
    return {tag + n: np.array(gm[n][:, c0:c1]) for n in names}


class DeviceImages(object):
    """Frames as the fused kernel reads them: torch tensors on the GPU; host arrays for the emulated kernels."""

    def __init__(self, imgs):
        if EMULATED:
            self.keep = [np.ascontiguousarray(im) for im in imgs]
            self.ptrs = [im.ctypes.data for im in self.keep]
        else:
            torch = pytest.importorskip("torch")
            self.keep = [torch.from_numpy(np.ascontiguousarray(im)).cuda() for im in imgs]
            self.ptrs = [t.data_ptr() for t in self.keep]


def frames(half_x, half_y, n_lines=2, per_line=3, colored=False):
    camd = synth.scaled_camera(0.05)
    poses = synth.lawnmower_poses(n_lines, per_line, half_x, half_y, agl=60.0, seed=4, jitter_pos=0.5)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], 3 if colored else 1) for k in range(len(poses))]
    return camd, poses, imgs


def holed_elevation(rows, cols, res):
    elev = synth.analytic_elevation(rows, cols, res)
    elev[5:20, 3:11] = np.nan      # holes inside frames' views
    elev[:, cols - 7:] = np.nan    # a band of tiles with no elevation at all
    return elev


# ---- every read path right after the reset, after an upload, after two resets ----
def read_paths(sequence):
    gm = resident_map(70, 45)
    if sequence in ("init", "init_twice", "init_upload"):
        init(gm)
    if sequence == "init_twice":
        init(gm)
    if sequence == "init_upload":
        gm["elevation"] = synth.analytic_elevation(70, 45, 1.0)
        gm.upload(("elevation",))
    out = {}
    # the asynchronous download first: it must not see a slab before its reset is written
    mirror = np.full((70, 45), 7.0, np.float32, order="F")
    amb.check(amb.lib().amb_download_layer_async(gm.context(), _lib.LAYER_ID["observation_index"],
                                                 mirror.ctypes.data_as(C.c_void_p)), gm.context())
    gm.sync()
    out["async_observation_index"] = mirror.copy()
    out.update(download(gm))
    out["raster_elevation"] = gm.to_raster("elevation")
    out["raster_ortho"] = gm.to_raster("ortho", "gray8")
    out["jpeg_ortho"] = np.frombuffer(gm.to_jpeg("ortho"), np.uint8)
    if not EMULATED:
        torch = pytest.importorskip("torch")
        p = C.c_void_p()
        amb.check(amb.lib().amb_layer_device_ptr(gm.context(), _lib.LAYER_ID["elevation_angle"], C.byref(p)),
                  gm.context())
        h = type("H", (), {})()
        h.__cuda_array_interface__ = {"shape": (70 * 45,), "typestr": "<f4", "data": (p.value, False), "version": 2}
        out["device_ptr_elevation_angle"] = torch.as_tensor(h, device="cuda:0").cpu().numpy()
    return out


@pytest.mark.parametrize("sequence", ["init", "init_twice", "init_upload"])
def test_read_paths_see_the_initial_values(sequence):
    ref = both(read_paths, sequence)
    assert np.isnan(ref["elevation"]).all() == (sequence != "init_upload")
    assert (ref["ortho"] == 255.0).all() and (ref["elevation_angle"] == 0).all()


# ---- the DSM ----
def dsm_case(rows, cols, res, points, col_ranges=(None,), precision=None, chunks=1, steps=2):
    out = {}
    for k, cr in enumerate(col_ranges):
        gm = resident_map(rows, cols, res, col_range=cr, names=("elevation",))
        dsm = amb.Dsm(amb.DsmSettings(), gm)
        dsm.precision = precision
        dsm.stream_chunks = chunks
        if chunks > 1:
            gm.set_mirrors(("elevation",))
        for s in range(steps):   # the second step resets a slab the first one wrote
            init(gm)
            dsm.process(points[s % len(points)], gm)
            gm.sync()
            out.update(download(gm, ("elevation",), "stripe%d_step%d_" % (k, s)))
    return out


def sparse_cloud(rows, cols, res, n, seed):
    # empty regions (cells no retry level reaches) and a cluster dense enough to hand whole tiles to the cell kernel
    hx, hy = rows * res / 2, cols * res / 2
    rng = np.random.default_rng(seed)
    base = synth.point_cloud(n, hx, hy, seed=seed, holes=6, hole_sides=(8.0, 20.0))
    base = base[(base[:, 0] < hx * 0.4) | (base[:, 1] < 0)]
    cluster = np.c_[rng.uniform(-6, 2, 4 * n), rng.uniform(5, 12, 4 * n), 100 + rng.normal(0, 0.05, 4 * n)]
    return np.ascontiguousarray(np.r_[base, cluster])


@pytest.mark.parametrize("rows,cols", [(70, 45), (129, 97)])
def test_dsm_partial_tiles_empty_regions_dense_tiles(rows, cols):
    pts = [sparse_cloud(rows, cols, 1.0, 3000, 11), synth.point_cloud(2500, rows / 2, cols / 2, seed=12)]
    ref = both(dsm_case, rows, cols, 1.0, pts)
    assert np.isnan(ref["stripe0_step0_elevation"]).any() and not np.isnan(ref["stripe0_step0_elevation"]).all()


def test_dsm_stripes_and_chunks():
    pts = [sparse_cloud(96, 90, 1.0, 3000, 13)]
    both(dsm_case, 96, 90, 1.0, pts, ((0, 29), (29, 61), (61, 90)))
    both(dsm_case, 96, 90, 1.0, pts, (None,), None, 3)


def test_dsm_f64():
    both(dsm_case, 70, 45, 1.0, [sparse_cloud(70, 45, 1.0, 3000, 14)], (None,), "f64")


# ---- the orthomosaic ----
def ortho_case(kind, colored=False, cull="dominance", batch=0, steps=2):
    rows, cols, res = 80, 70, 1.0
    out_name = "colored_ortho" if colored else "ortho"
    gm = resident_map(rows, cols, res)
    camd, poses, imgs = frames(rows / 2, cols / 2, colored=colored)
    o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm)
    o.brute_force = cull == "brute"
    o.dominance_cull = cull == "dominance"
    dev = DeviceImages(imgs) if kind == "device" else None
    elev = holed_elevation(rows, cols, res)
    out = {}
    for s in range(steps):
        init(gm)
        gm["elevation"] = elev if s == 0 else elev + 1.0
        gm.upload(("elevation",))
        chunks = [(0, len(poses))] if not batch else [(b, min(b + batch, len(poses))) for b in range(0, len(poses), batch)]
        for b0, b1 in chunks:
            if kind == "device":
                o.process_device(poses[b0:b1], dev.ptrs[b0:b1], camd["width"] * (3 if colored else 1), gm)
            else:
                o.process(poses[b0:b1], imgs[b0:b1], gm)
        gm.sync()
        out.update(download(gm, ("elevation_angle", "observation_index", out_name), "step%d_" % s))
    return out


@pytest.mark.parametrize("cull", ["dominance", "plain", "brute"])
def test_ortho_fused_over_holes_and_unseen_tiles(cull):
    ref = both(ortho_case, "device", False, cull)
    assert (ref["step0_ortho"] == 255.0).any() and (ref["step0_ortho"] != 255.0).any()


def test_ortho_colored():
    both(ortho_case, "device", True)


def test_ortho_host_frames():
    both(ortho_case, "host")


def test_ortho_batched():
    both(ortho_case, "device", False, "dominance", 2)


# ---- DSM then orthomosaic in one step, OrthoFromPcl after a reset ----
def joint_case():
    rows, cols = 80, 70
    gm = resident_map(rows, cols)
    pts = sparse_cloud(rows, cols, 1.0, 4000, 15)
    camd, poses, imgs = frames(rows / 2, cols / 2)
    dev = DeviceImages(imgs)
    dsm = amb.Dsm(amb.DsmSettings(), gm)
    o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm)
    out = {}
    for s in range(2):
        init(gm)
        dsm.process(pts, gm)
        o.process_device(poses, dev.ptrs, camd["width"], gm)
        gm.sync()
        out.update(download(gm, ORTHO_LAYERS, "step%d_" % s))
    return out


def test_dsm_then_ortho():
    both(joint_case)


def pcl_case(adaptive):
    rows, cols = 70, 45
    gm = resident_map(rows, cols)
    pts = sparse_cloud(rows, cols, 1.0, 3000, 16)
    inten = (np.arange(pts.shape[0]) * 37 % 256).astype(np.int32)
    o = amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=2, use_adaptive_interpolation=adaptive))
    init(gm)
    o.process(pts, inten, gm)
    gm.sync()
    return download(gm)


@pytest.mark.parametrize("adaptive", [False, True])
def test_ortho_from_pcl_after_init(adaptive):
    both(pcl_case, adaptive)
