"""Every orthomosaic entry point of the C ABI on the same frames: host frames (amb_ortho_process), device frames
(amb_ortho_process_device), JPEG files (amb_ortho_process_jpeg, against the host route on the decoded pixels of the same
files) and amb_multi_ortho_process with one device must write the same layer bits, return the statuses of their argument
checks in one order, write nothing and keep the previous call's timings when they refuse a call, and report their
timings the same way.  The Python mirror's process* methods keep their exceptions.

The tests also run on the emulated kernels (tests/emu) through tests/test_emulated_kernels.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402
from test_jpeg_decode_cpu import segment  # noqa: E402

try:
    import cv2
except ImportError:   # the frames of tests/golden/jpeg_decode_cases.npz stand in
    cv2 = None

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
ROWS, COLS, RES = 48, 40, 1.0
W, H = 34, 40          # the frame size of some of the fixture's files
OK, EMPTY, INVALID, SIZE, UNSUPPORTED, CORRUPT = (_lib.AMB_OK, _lib.AMB_ERR_EMPTY, _lib.AMB_ERR_INVALID_ARGUMENT,
                                                  _lib.AMB_ERR_SIZE_MISMATCH, _lib.AMB_ERR_UNSUPPORTED,
                                                  _lib.AMB_ERR_CORRUPT_DATA)
ROUTES = ("host", "device", "jpeg", "multi")
ORTHO_FIELDS = ("ortho_h2d_ms", "ortho_kernel_ms", "ortho_total_ms", "ortho_kernel_launches", "ortho_h2d_bytes")


def L():
    return amb.lib()


def camera():
    return amb.NCamera(W, H, 0.75 * W, 0.75 * W, W / 2.0, H / 2.0, dist_type=_lib.DIST_RADTAN,
                       dist=(-0.05, 0.01, 1e-4, 1e-4)).camera


def frames(n, colored, seed=3):
    """Poses, the JPEG files of n frames and their decoded pixels (what cv2.imread returns)."""
    ch = 3 if colored else 1
    lines = max(1, int(np.sqrt(n)))
    poses = synth.lawnmower_poses(lines, -(-n // lines), ROWS * RES / 2, COLS * RES / 2, 60.0, seed,
                                  jitter_pos=0.6)[:n]
    if cv2 is not None:
        files = []
        for k in range(n):
            ok, b = cv2.imencode(".jpg", synth.procedural_image(k, W, H, ch), [cv2.IMWRITE_JPEG_QUALITY, 90])
            assert ok
            files.append(b.tobytes())
        images = [cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR if colored else cv2.IMREAD_GRAYSCALE)
                  for f in files]
    else:
        z = np.load(os.path.join(HERE, "golden", "jpeg_decode_cases.npz"))
        ks = [k for k in range(len([f for f in z.files if f.startswith("file_")])) if z["gray_%d" % k].shape == (H, W)]
        assert ks
        files = [z["file_%d" % ks[k % len(ks)]].tobytes() for k in range(n)]
        images = [z[("bgr_%d" if colored else "gray_%d") % ks[k % len(ks)]] for k in range(n)]
    return np.ascontiguousarray(poses), files, [np.ascontiguousarray(im) for im in images]


def written(colored):
    return ("elevation_angle", "observation_index", "colored_ortho" if colored else "ortho")


class Call(object):
    """The C arrays of one call over (poses, files, images); device copies of the images for the device route."""

    def __init__(self, poses, files, images):
        self.n = len(poses)
        self.poses = np.ascontiguousarray(poses, np.float64)
        self.ch = 1 if images[0].ndim == 2 else 3
        self.row_step = W * self.ch
        self.images = images
        self.img_ptrs = (C.c_void_p * self.n)(*[im.ctypes.data for im in images])
        self.keep = [np.frombuffer(f, np.uint8).copy() for f in files]
        self.file_ptrs = (C.c_void_p * self.n)(*[a.ctypes.data for a in self.keep])
        self.sizes = (C.c_size_t * self.n)(*[len(f) for f in files])
        stack = np.ascontiguousarray(np.stack(images))
        if EMULATED:   # the emulated kernels take host memory as device memory
            self.dev, base = stack, stack.ctypes.data
        else:
            import torch
            self.dev = torch.from_numpy(stack).to("cuda:0")
            base = self.dev.data_ptr()
        self.dev_ptrs = (C.c_void_p * self.n)(*[base + k * H * self.row_step for k in range(self.n)])
        self.cam = camera()

    def run(self, route, ctx, colored, **kw):
        """The route's status; keyword arguments replace arguments of the call (None: a null pointer)."""
        a = dict(cam=C.byref(self.cam), T=self.poses.ctypes.data, n=self.n, ch=self.ch, row_step=self.row_step,
                 imgs=self.dev_ptrs if route == "device" else self.img_ptrs, files=self.file_ptrs, sizes=self.sizes)
        a.update(kw)
        if route == "jpeg":
            return L().amb_ortho_process_jpeg(ctx, a["cam"], a["T"], a["files"], a["sizes"], a["n"], colored)
        fn = {"host": L().amb_ortho_process, "multi": L().amb_multi_ortho_process,
              "device": L().amb_ortho_process_device}[route]
        return fn(ctx, a["cam"], a["T"], a["imgs"], a["n"], a["ch"], a["row_step"], colored)


def grid_map(col_range=None):
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, ROWS * RES, COLS * RES, RES)).getMutable()
    gm["elevation"] = np.full((ROWS, COLS), 2.0, np.float32, order="F")
    gm.context(0, col_range)
    gm.upload(("elevation",))
    return gm


def layers(gm, colored):
    gm.sync()
    gm.download(written(colored))
    c0, c1 = gm._col_range
    return [gm[name][:, c0:c1].copy() for name in written(colored)]


def run_route(route, calls, colored, col_range=None):
    """The layers the route writes over `calls` (one after the other on the same map)."""
    if route == "multi":
        gm = grid_map()                                   # for its geometry
        m = C.c_void_p()
        amb.check(L().amb_multi_create(C.byref(gm.geometry), 1, C.byref(m)))
        try:
            assert L().amb_multi_size(m) == 1
            amb.check(L().amb_multi_upload_layer(m, _lib.LAYER_ID["elevation"], gm["elevation"].ctypes.data))
            for call in calls:
                assert call.run(route, m, colored) == OK
            assert L().amb_multi_sync(m) == OK
            out = []
            for name in written(colored):
                a = np.full((ROWS, COLS), np.nan, np.float32, order="F")
                amb.check(L().amb_multi_download_layer(m, _lib.LAYER_ID[name], a.ctypes.data))
                out.append(a)
        finally:
            L().amb_multi_destroy(m)
        return out
    gm = grid_map(col_range)
    for call in calls:
        assert call.run(route, gm.context(), colored) == OK, route
    return layers(gm, colored)


def same_bits(a, b):
    return all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


# ---- the same layer bits from every route ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("colored", [0, 1])
@pytest.mark.parametrize("case", ["fresh", "written", "two_chunks", "stripe"])
def test_every_route_writes_the_same_layers(colored, case):
    n = 520 if case == "two_chunks" else 9            # > 512 frames: two chunks of the constant-memory frame table
    calls = [Call(*frames(n, colored))]
    if case == "written":                             # layers an earlier call wrote
        calls.insert(0, Call(*frames(6, colored, seed=5)))
    routes = ROUTES if case != "stripe" else ROUTES[:3]
    col_range = (13, 31) if case == "stripe" else None
    ref = run_route("host", calls, colored, col_range)
    assert np.isfinite(ref[1]).sum() > 0.9 * ref[1].size   # frames contribute
    for route in routes[1:]:
        assert same_bits(run_route(route, calls, colored, col_range), ref), (route, case)


# ---- argument checks, in their order; a refused call writes nothing and keeps the previous timings ------------------
def refusals(call, route, colored):
    """[(status wanted, keyword arguments of Call.run)]: one fault each, in the order run_ortho checks them."""
    cam = call.cam

    def cam_with(**kw):
        c = _lib.Camera()
        C.memmove(C.byref(c), C.byref(cam), C.sizeof(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return C.byref(c), c

    wide, wide_keep = cam_with(width=70000)
    zero_w, zero_w_keep = cam_with(width=0)
    zero_h, zero_h_keep = cam_with(height=0)
    bad_dist, bad_dist_keep = cam_with(dist_type=9)
    cases = [(INVALID, dict(ctx=None)),
             (EMPTY, dict(n=0, cam=None, T=None, imgs=None, files=None, sizes=None)),
             (INVALID, dict(cam=None)),
             (INVALID, dict(T=None)),
             (SIZE, dict(cam=zero_w)),
             (SIZE, dict(cam=zero_h)),
             (UNSUPPORTED, dict(cam=bad_dist))]
    if route == "jpeg":
        null_late = (C.c_void_p * call.n)(*list(call.file_ptrs))
        null_late[5] = None
        junk = np.frombuffer(b"not a JPEG file", np.uint8).copy()
        garbage = (C.c_void_p * call.n)(*list(call.file_ptrs))
        garbage[2] = junk.ctypes.data
        sizes = (C.c_size_t * call.n)(*list(call.sizes))
        sizes[2] = junk.size
        # a frame of another size (a camera of another size): first a null frame, then a header status, then sizes
        other = cam_with(width=W + 1)
        cases += [(INVALID, dict(files=None)), (INVALID, dict(sizes=None)), (INVALID, dict(files=null_late)),
                  (INVALID, dict(files=garbage, sizes=sizes)), (SIZE, dict(cam=other[0])),
                  (INVALID, dict(cam=other[0], files=null_late))]
        keep = [null_late, junk, garbage, sizes, other]
    else:
        cases += [(INVALID, dict(imgs=None)), (UNSUPPORTED, dict(cam=wide)),
                  (SIZE, dict(ch=1 if colored else 3, row_step=W * 3)), (SIZE, dict(row_step=W * call.ch - 1)),
                  (UNSUPPORTED, dict(cam=wide, ch=1 if colored else 3))]      # width before channels
        if route != "device":                         # device frame pointers are not inspected
            nulls = (C.c_void_p * call.n)(*list(call.img_ptrs))
            nulls[4] = None
            cases += [(INVALID, dict(imgs=nulls)), (INVALID, dict(imgs=nulls, cam=wide))]
            keep = [nulls]
        else:
            keep = []
    return cases, [wide_keep, zero_w_keep, zero_h_keep, bad_dist_keep, keep]


@pytest.mark.gpu
@pytest.mark.parametrize("colored", [0, 1])
@pytest.mark.parametrize("route", ["host", "device", "jpeg"])
def test_refused_calls_return_their_status_write_nothing_and_keep_the_timings(route, colored):
    call = Call(*frames(9, colored))
    gm = grid_map()
    ctx = gm.context()
    assert call.run(route, ctx, colored) == OK
    before = layers(gm, colored)
    timed = gm.timings()
    assert timed["ortho_kernel_launches"] > 0
    cases, keep = refusals(call, route, colored)
    for k, (want, kw) in enumerate(cases):
        c = kw.pop("ctx", ctx)
        assert call.run(route, c, colored, **kw) == want, (k, route, kw)
        assert gm.timings() == timed, (k, route)
    assert same_bits(layers(gm, colored), before)
    assert L().amb_sync(ctx) == OK


@pytest.mark.gpu
def test_multi_passes_the_statuses_of_its_context_through():
    call = Call(*frames(9, 0))
    gm = grid_map()
    m = C.c_void_p()
    amb.check(L().amb_multi_create(C.byref(gm.geometry), 1, C.byref(m)))
    try:
        cases, keep = refusals(call, "multi", 0)
        for k, (want, kw) in enumerate(cases):
            if kw.pop("ctx", m) is None:
                continue
            assert call.run("multi", m, 0, **kw) == want, (k, kw)
    finally:
        L().amb_multi_destroy(m)


# ---- timings ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [9, 520])
def test_h2d_only_for_host_and_jpeg_frames_and_one_more_launch(n):
    call = Call(*frames(n, 0))
    chunks = -(-n // 512)
    for route in ("host", "device", "jpeg"):
        gm = grid_map()
        assert call.run(route, gm.context(), 0) == OK
        t = gm.timings()
        two_phase = route != "device"
        assert t["ortho_kernel_launches"] == chunks + (1 if two_phase else 0), route
        assert (t["ortho_h2d_ms"] > 0.0) == two_phase and (t["ortho_h2d_bytes"] > 0) == two_phase, (route, t)
        assert t["ortho_total_ms"] > 0.0, route


@pytest.mark.gpu
def test_a_corrupt_contributing_jpeg_frame_reports_no_ortho_timings():
    call = Call(*frames(9, 0))
    gm = grid_map()
    assert call.run("host", gm.context(), 0) == OK
    assert gm.timings()["ortho_kernel_launches"] > 0
    cut = [f[:(segment(f, 0xDA)[1] + len(f)) // 2] for f in (bytes(a) for a in call.keep)]   # every scan cut in half
    bad = Call(call.poses, cut, call.images)
    assert bad.run("jpeg", gm.context(), 0) == CORRUPT
    t = gm.timings()
    assert all(t[k] == 0 for k in ORTHO_FIELDS), t


# ---- the Python mirror --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_mirror_keeps_its_exceptions():
    poses, files, images = frames(4, 0)
    gm = grid_map()
    grid = amb.OrthoBackwardGrid(amb.NCamera(W, H, 0.75 * W, 0.75 * W, W / 2.0, H / 2.0), amb.OrthoSettings(), gm)

    def status(fn, *args):
        with pytest.raises(amb.AmbError) as e:
            fn(*args)
        return e.value.status

    assert status(grid.process, poses[:0], [], gm) == EMPTY
    assert status(grid.process, poses, images[:3], gm) == SIZE
    assert status(grid.process, poses, images, None) == INVALID
    assert status(grid.process, poses, images[:3] + [images[0][:, :-1]], gm) == SIZE
    assert status(grid.process_jpeg, poses[:0], [], gm) == EMPTY
    assert status(grid.process_jpeg, poses, files[:3], gm) == SIZE
    assert status(grid.process_jpeg, poses, files, None) == INVALID
    assert status(grid.process_device, poses[:0], [], W, gm) == SIZE
    assert status(grid.process_device, poses, [0, 0, 0], W, gm) == SIZE
