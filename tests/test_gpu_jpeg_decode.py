"""JPEG frames decoded on the device (amb_jpeg_decode_device, amb_ortho_process_jpeg, csrc/jpeg_decode.cu; convention in
include/aerial_mapper_b200.h): every decode is compared byte for byte with cv2.imread of the same file (through
cv2.imdecode), and where OpenCV is not installed with the fixture tests/golden/jpeg_decode_cases.npz.

Device buffers are torch CUDA tensors; under AMB_TEST_EMU=1 (the emulated kernels) device memory is host memory and they
are numpy arrays.  The last tests run this file's `gpu` tests on the emulated kernels (the 4000 x 3000 frames and the
torch wrapper need a GPU)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, synth  # noqa: E402
from test_jpeg_decode_cpu import base_file, huff_file, pil_jpeg, refused_files, segment  # noqa: E402

try:
    import cv2
except ImportError:   # the fixture cases still run
    cv2 = None

gpu = pytest.mark.gpu
EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")
CANARY = 0xA5
GOLDEN = os.path.join(HERE, "golden", "jpeg_decode_cases.npz")
SAMPLINGS = ("444", "422", "420")


def need_cv2():
    if cv2 is None:
        pytest.skip("OpenCV is not installed (the fixture cases cover this host)")


def cv2_file(img, quality=95, sampling="420", restart=0, optimize=False):
    flags = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart,
              cv2.IMWRITE_JPEG_OPTIMIZE, 1 if optimize else 0]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, flags[sampling]]
    ok, b = cv2.imencode(".jpg", img, params)
    assert ok
    return b.tobytes()


def imread(b, channels):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR if channels == 3 else cv2.IMREAD_GRAYSCALE)


def content(kind, h, w, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
    if kind == "constant":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    if kind == "checker":
        a = np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, 255, 0).astype(np.uint8)
        return np.repeat(a[:, :, None], 3, axis=2) ^ np.uint8([0, 255, 0])
    if kind == "smooth":   # noise blurred: the usual mix of short and long codes
        return cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3)).astype(np.uint8), (7, 7), 2)
    a = np.add.outer(np.arange(h) * 3, np.arange(w) * 2)
    return np.stack([(a + 40 * k) % 256 for k in range(3)], axis=-1).astype(np.uint8)


class Out(object):
    """A device destination of h rows of w * channels bytes, `pad` bytes of canary after every row and around it."""

    def __init__(self, h, w, channels, pad=5):
        self.h, self.w, self.channels = h, w, channels
        self.step = w * channels + pad
        host = np.full(64 + h * self.step + 64, CANARY, np.uint8)
        if EMULATED:
            self.raw = host
            self.ptr = host.ctypes.data + 64
        else:
            import torch
            self.raw = torch.from_numpy(host).to("cuda:0")
            self.ptr = self.raw.data_ptr() + 64

    def host(self):
        return self.raw.copy() if EMULATED else self.raw.cpu().numpy()

    def image(self):
        a = self.host()[64:64 + self.h * self.step].reshape(self.h, self.step)[:, :self.w * self.channels]
        return a.reshape(self.h, self.w, 3) if self.channels == 3 else a

    def untouched(self):
        return bool(np.all(self.host() == CANARY))


class HostFiles(object):
    """The files in pageable (numpy) or pinned (amb_host_alloc) host memory, as the C arrays of the decode call."""

    def __init__(self, files, pinned=False):
        self.pinned = []
        ptrs = []
        self.keep = []
        for f in files:
            if pinned and len(f):
                p = C.c_void_p()
                assert _lib.lib().amb_host_alloc(C.byref(p), len(f)) == 0
                C.memmove(p, f, len(f))
                self.pinned.append(p)
                ptrs.append(p.value)
            else:
                a = np.frombuffer(f, np.uint8).copy() if len(f) else np.zeros(1, np.uint8)
                self.keep.append(a)
                ptrs.append(a.ctypes.data)
        n = len(files)
        self.ptrs = (C.c_void_p * n)(*ptrs)
        self.sizes = (C.c_size_t * n)(*[len(f) for f in files])

    def free(self):
        for p in self.pinned:
            _lib.lib().amb_host_free(p)


def decode(files, channels, pinned=False, shapes=None):
    """(return status, [status], [Out]) of one amb_jpeg_decode_device call over `files`."""
    n = len(files)
    outs = []
    for k, f in enumerate(files):
        if shapes:
            h, w = shapes[k]
        else:
            i = amb.jpeg_info(f)
            h, w = i["height"], i["width"]
        outs.append(Out(h, w, channels))
    hf = HostFiles(files, pinned)
    status = (C.c_int * n)()
    rc = _lib.lib().amb_jpeg_decode_device(api._jpeg_context(0), hf.ptrs, hf.sizes, n, channels,
                                           (C.c_void_p * n)(*[o.ptr for o in outs]),
                                           (C.c_size_t * n)(*[o.step for o in outs]), status)
    hf.free()
    return rc, list(status), outs


def assert_decodes_like_imread(files, channels=None, pinned=False):
    for ch in ((1, 3) if channels is None else (channels,)):
        rc, status, outs = decode(files, ch, pinned)
        assert rc == 0 and status == [0] * len(files)
        for k, f in enumerate(files):
            assert np.array_equal(outs[k].image(), imread(f, ch)), (k, ch, amb.jpeg_info(f))


# ---- the fixture (no OpenCV needed) -----------------------------------------------------------------------------------
@gpu
def test_fixture_cases_equal_cv2_imread():
    z = np.load(GOLDEN)
    n = len([k for k in z.files if k.startswith("file_")])
    files = [z["file_%d" % k].tobytes() for k in range(n)]
    for ch, key in ((3, "bgr"), (1, "gray")):
        rc, status, outs = decode(files, ch)   # one batch: mixed sizes, samplings, gray and colour files
        assert rc == 0 and status == [0] * n
        for k in range(n):
            assert np.array_equal(outs[k].image(), z["%s_%d" % (key, k)]), (k, ch)


@gpu
def test_colour_decodes_equal_pil():
    # PIL's libjpeg-turbo decode of the colour files (RGB, reversed to B, G, R) is the same raster
    Image = pytest.importorskip("PIL.Image")
    import io
    z = np.load(GOLDEN)
    files = [z["file_%d" % k].tobytes() for k in range(len([f for f in z.files if f.startswith("file_")]))]
    files = [f for f in files if amb.jpeg_info(f)["components"] == 3]
    rc, status, outs = decode(files, 3)
    assert rc == 0 and len(files) > 40
    for k, f in enumerate(files):
        assert np.array_equal(outs[k].image(), np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))[:, :, ::-1]), k


# ---- encodings --------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_qualities_and_restart_intervals(sampling):
    need_cv2()
    img = content("smooth", 250, 333, seed=3)
    files = [cv2_file(img, q, sampling, r) for q in (1, 10, 50, 75, 95, 100) for r in (0, 1, 3, 8, 1000)]
    assert_decodes_like_imread(files)


@gpu
def test_gray_files():
    need_cv2()
    img = content("smooth", 250, 333, seed=4)[:, :, 1].copy()
    assert_decodes_like_imread([cv2_file(img, q, "420", r) for q in (1, 50, 95, 100) for r in (0, 1, 7)])


@gpu
def test_every_mcu_remainder():
    # 1 x 1 up to 17 x 9: every remainder of the 8- and 16-pixel MCUs; widths 1..5 take the box replication (chroma
    # width <= 2) and the triangle filter at its edges
    need_cv2()
    for sampling in SAMPLINGS + ("gray",):
        files = []
        for h in range(1, 18):
            for w in range(1, 10):
                img = content("noise", h, w, seed=h * 31 + w)
                files.append(cv2_file(img[:, :, 0].copy() if sampling == "gray" else img, 75,
                                      "420" if sampling == "gray" else sampling, 0))
        assert_decodes_like_imread(files)


@gpu
@pytest.mark.parametrize("kind", ["noise", "constant", "checker", "gradient"])
def test_contents(kind):
    need_cv2()
    img = content(kind, 48, 72, seed=5)
    assert_decodes_like_imread([cv2_file(img, q, s, r) for s in SAMPLINGS for q in (10, 95) for r in (0, 2)])


@gpu
def test_a_real_orthomosaic_layer():
    need_cv2()
    z = np.load(os.path.join(HERE, "golden", "ortho_color_96x80.npz"))
    packed = z["out"].astype(np.uint32)
    img = np.ascontiguousarray(np.stack([packed & 255, (packed >> 8) & 255, (packed >> 16) & 255], -1).astype(np.uint8))
    assert_decodes_like_imread([cv2_file(img, q, s, r) for s in SAMPLINGS for q in (75, 95) for r in (0, 4)])


@gpu
def test_optimised_tables_and_pil_files():
    need_cv2()
    img = content("smooth", 61, 83, seed=6)
    files = [cv2_file(img, q, s, 0, optimize=True) for s in SAMPLINGS for q in (30, 95)]
    files += [pil_jpeg(img, quality=q, subsampling=sub, optimize=opt) for sub in (0, 1, 2) for q in (40, 90)
              for opt in (False, True)]
    files.append(pil_jpeg(img, qtables=[[300] * 64, [700] * 64], subsampling=2))   # 16-bit DQT: SOF1
    assert b"\xFF\xC1" in files[-1][:400]
    assert_decodes_like_imread(files)


@gpu
def test_scan_shifted_by_1_to_127_bytes():
    # the same scan shifted by a COM segment of 1..127 bytes: the unstuffing's 4 KB chunks of the file, and the 16-byte
    # pieces of its threads, start at 127 different byte offsets of the scan
    need_cv2()
    b = cv2_file(content("smooth", 64, 96, seed=7), 95, "420", 0)
    files = [b[:2] + b"\xFF\xFE" + bytes([0, n + 2]) + bytes(n) + b[2:] for n in range(1, 128)]
    rc, status, outs = decode(files, 3)
    ref = imread(b, 3)
    assert rc == 0 and status == [0] * len(files)
    assert all(np.array_equal(o.image(), ref) for o in outs)


@gpu
def test_mixed_batches():
    need_cv2()
    files = []
    for k, (h, w) in enumerate(((9, 7), (120, 161), (1, 1), (33, 48), (250, 333))):
        img = content("smooth" if h > 8 else "noise", h, w, seed=k)
        files += [cv2_file(img, 90, SAMPLINGS[k % 3], k % 2), cv2_file(img[:, :, 2].copy(), 80, "420", 0),
                  cv2_file(img, 70, SAMPLINGS[(k + 1) % 3], 0)]
    assert_decodes_like_imread(files)


@gpu
def test_pinned_and_pageable_files_are_identical():
    # a file over the 4 MB the library stages pageable copies from
    need_cv2()
    b = cv2_file(content("noise", 1100, 1400, seed=8), 100, "444", 0)
    assert len(b) > (4 << 20)
    _, s1, pageable = decode([b], 3, pinned=False)
    _, s2, pinned = decode([b], 3, pinned=True)
    assert s1 == s2 == [0]
    assert np.array_equal(pageable[0].image(), pinned[0].image())
    assert np.array_equal(pinned[0].image(), imread(b, 3))


@gpu
@pytest.mark.parametrize("sampling", ["420", "422"])
def test_4000x3000_frames(sampling):
    if EMULATED:
        return   # minutes on the emulated kernels; every path it takes is covered by the smaller cases
    need_cv2()
    img = np.ascontiguousarray(synth.procedural_image(3, 4000, 3000, 3))
    files = [cv2_file(img, 95, sampling, r) for r in (0, 250)]
    assert_decodes_like_imread(files, channels=3)
    assert_decodes_like_imread(files[:1], channels=1)


# ---- contracts ---------------------------------------------------------------------------------------------------------
@gpu
def test_refusals_write_nothing():
    named = refused_files()
    files = [f for _, f in named] + [base_file()]
    rc, status, outs = decode(files, 3, shapes=[(17, 33)] * len(files))
    assert rc == _lib.AMB_ERR_UNSUPPORTED
    for k, (name, _) in enumerate(named):
        assert status[k] == _lib.AMB_ERR_UNSUPPORTED and outs[k].untouched(), name
    assert status[-1] == 0 and not outs[-1].untouched()   # the supported file of the same batch is decoded


@gpu
def test_bad_arguments():
    b = base_file()
    hf = HostFiles([b])
    o = Out(17, 33, 3)
    st = (C.c_int * 1)()
    L, ctx = _lib.lib(), api._jpeg_context(0)
    ptr, short = (C.c_void_p * 1)(o.ptr), (C.c_size_t * 1)(33 * 3 - 1)
    assert L.amb_jpeg_decode_device(ctx, hf.ptrs, hf.sizes, 1, 2, ptr, (C.c_size_t * 1)(o.step), st) == \
        _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_jpeg_decode_device(ctx, hf.ptrs, hf.sizes, 1, 3, ptr, short, st) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert st[0] == _lib.AMB_ERR_INVALID_ARGUMENT and o.untouched()
    assert L.amb_jpeg_decode_device(ctx, None, hf.sizes, 1, 3, ptr, short, st) == _lib.AMB_ERR_INVALID_ARGUMENT
    assert L.amb_jpeg_decode_device(ctx, hf.ptrs, hf.sizes, 0, 3, ptr, short, st) == 0


# ---- corruption ---------------------------------------------------------------------------------------------------------
def corrupt_files():
    """[(name, file)]: scans that are not valid for their headers."""
    img = content("smooth", 40, 56, seed=9)
    b = cv2_file(img, 90, "420", 0)
    r = cv2_file(img, 90, "420", 1)
    start = segment(r, 0xDA)[1]
    rst0 = r.index(b"\xFF\xD0", start)
    rst1 = r.index(b"\xFF\xD1", start)
    mid = (segment(b, 0xDA)[1] + len(b)) // 2   # inside the scan
    return [("truncated_half", b[:mid]), ("truncated_near_end", b[:len(b) - 40]),
            ("scan_empty", b[:segment(b, 0xDA)[1]] + b"\xFF\xD9"),
            ("rst_out_of_sequence", r[:rst0 + 1] + b"\xD3" + r[rst0 + 2:]),
            ("rst_missing", r[:rst1] + r[rst1 + 2:]),
            ("run_past_63", huff_file(0xF1, "0" + "01" * 4)),   # ZRL + value four times: k = 17, 33, 49, 65
            ("no_such_code", huff_file(0x00, "0" + "1" * 16))]


@gpu
def test_corrupt_scans_return_corrupt_data_and_write_nothing():
    need_cv2()
    named = corrupt_files()
    good = cv2_file(content("smooth", 40, 56, seed=10), 90, "444", 0)
    files = [f for _, f in named] + [good]
    shapes = [(8, 8) if name in ("run_past_63", "no_such_code") else (40, 56) for name, _ in named] + [(40, 56)]
    for ch in (1, 3):
        rc, status, outs = decode(files, ch, shapes=shapes)
        assert rc == _lib.AMB_ERR_CORRUPT_DATA
        for k, (name, _) in enumerate(named):
            assert status[k] == _lib.AMB_ERR_CORRUPT_DATA and outs[k].untouched(), (name, ch)
        assert status[-1] == 0 and np.array_equal(outs[-1].image(), imread(good, ch))


@gpu
def test_data_after_the_last_mcu_is_ignored():
    need_cv2()
    b = cv2_file(content("smooth", 40, 56, seed=11), 90, "420", 2)
    files = [b[:-2], b[:-2] + b"\x12\x34\xFF\xD9", b + b"trailing bytes"]
    rc, status, outs = decode(files, 3)
    assert rc == 0 and status == [0, 0, 0]
    assert all(np.array_equal(o.image(), imread(b, 3)) for o in outs)


@gpu
@pytest.mark.parametrize("restart", [0, 2])
def test_a_restart_marker_spliced_into_the_last_segment(restart):
    # An RSTn past the ones the restart interval calls for (any RSTn without a DRI) ends the entropy data for libjpeg:
    # MCUs that need bits beyond it are AMB_ERR_CORRUPT_DATA with the destination untouched, and one written after the
    # last MCU leaves the image as cv2.imread decodes it.
    need_cv2()
    b = cv2_file(content("smooth", 64, 96, seed=14), 90, "420", restart)
    start = segment(b, 0xDA)[1]
    if restart:
        # after the last restart marker: the last segment
        start = max(b.rfind(bytes([0xFF, 0xD0 + k]), start, len(b) - 2) for k in range(8)) + 2
    cuts = [p for p in np.linspace(start + 1, len(b) - 3, 24).astype(int) if b[p - 1] != 0xFF]
    files = [b[:p] + bytes([0xFF, 0xD0 + k % 8]) + b[p:] for k, p in enumerate(cuts)]
    files.append(b[:-2] + b"\xFF\xD3" + b[-2:])   # after the last MCU, before EOI
    for ch in (1, 3):
        rc, status, outs = decode(files, ch, shapes=[(64, 96)] * len(files))
        for k, f in enumerate(files):
            if status[k] == 0:
                assert np.array_equal(outs[k].image(), imread(f, ch)), (k, ch)
            else:
                assert status[k] == _lib.AMB_ERR_CORRUPT_DATA and outs[k].untouched(), (k, ch)
        assert status.count(_lib.AMB_ERR_CORRUPT_DATA) >= len(cuts) - 2   # (a splice right at the end may be harmless)
        assert status[-1] == 0 and np.array_equal(outs[-1].image(), imread(b, ch))


@gpu
def test_short_app_segments_are_what_libjpeg_reads():
    # libjpeg counts a JFIF APP0 only with 14 bytes of payload and an Adobe APP14 only with 12: a shorter "Adobe"
    # segment is skipped and the file decodes like cv2.imread
    need_cv2()
    b = cv2_file(content("smooth", 24, 40, seed=15), 90, "420", 0)
    f = b[:2] + b"\xFF\xEE\x00\x09Adobe\x00\x64" + b[2:]
    assert amb.jpeg_info(f)["components"] == 3
    rc, status, outs = decode([f], 3)
    assert rc == 0 and np.array_equal(outs[0].image(), imread(f, 3))


@gpu
@pytest.mark.parametrize("restart", [0, 2])
def test_single_bit_flips_decode_like_imread_or_are_refused(restart):
    # property: a decode either succeeds and equals cv2.imread, or returns AMB_ERR_CORRUPT_DATA and writes nothing
    need_cv2()
    rng = np.random.default_rng(12 + restart)
    for s in SAMPLINGS:
        b = cv2_file(content("smooth", 32, 48, seed=13), 90, s, restart)
        start = segment(b, 0xDA)[1]
        files = []
        for _ in range(60):
            a = bytearray(b)
            a[int(rng.integers(start, len(b) - 2))] ^= 1 << int(rng.integers(0, 8))
            files.append(bytes(a))
        for ch in (1, 3):
            _, status, outs = decode(files, ch, shapes=[(32, 48)] * len(files))
            for k, f in enumerate(files):
                if status[k] == 0:
                    assert np.array_equal(outs[k].image(), imread(f, ch)), (s, k, ch)
                else:
                    assert status[k] == _lib.AMB_ERR_CORRUPT_DATA and outs[k].untouched(), (s, k, ch)


# ---- the orthomosaic from JPEG files -------------------------------------------------------------------------------------
ORTHO = dict(rows=60, cols=56, res=1.0)


def ortho_case(colored, restart, area=None):
    """Camera, 3 x 3 lawnmower poses over `area` (half extents, m; default the map's) and their frames as JPEG files."""
    camd = synth.scaled_camera(0.05)
    hx, hy = area or (ORTHO["rows"] / 2, ORTHO["cols"] / 2)
    poses = synth.lawnmower_poses(3, 3, hx, hy, 60.0, 4, jitter_pos=0.6)
    ch = 3 if colored else 1
    imgs = [np.ascontiguousarray(synth.procedural_image(k, camd["width"], camd["height"], ch))
            for k in range(len(poses))]
    return camd, poses, [cv2_file(im, 90, "420", restart) for im in imgs]


def new_map(rows=None, cols=None):
    rows, cols = rows or ORTHO["rows"], cols or ORTHO["cols"]
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * ORTHO["res"], cols * ORTHO["res"],
                                               ORTHO["res"])).getMutable()
    gm["elevation"] = np.full((rows, cols), 2.0, np.float32, order="F")
    return gm


def written(colored):
    return ("elevation_angle", "observation_index", "colored_ortho" if colored else "ortho")


def run_both(camd, poses, files, colored, frames=None, shape=(None, None)):
    """process() on `frames` (default: cv2.imread of the files) and process_jpeg() on the files, each on a new map."""
    ch = 3 if colored else 1
    settings = amb.OrthoSettings(colored_ortho=colored)
    a, b = new_map(*shape), new_map(*shape)
    if frames is None:
        frames = [imread(f, ch) for f in files]
    amb.OrthoBackwardGrid(amb.NCamera(**camd), settings, a).process(poses, frames, a)
    amb.OrthoBackwardGrid(amb.NCamera(**camd), settings, b).process_jpeg(poses, files, b)
    return a, b


def assert_same_layers(a, b, colored):
    for name in written(colored):
        x, y = np.asarray(a[name]), np.asarray(b[name])
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), name


@gpu
@pytest.mark.parametrize("colored", [False, True])
@pytest.mark.parametrize("restart", [0, 3])
def test_process_jpeg_equals_process_on_imread_frames(colored, restart):
    need_cv2()
    camd, poses, files = ortho_case(colored, restart)
    a, b = run_both(camd, poses, files, colored)
    assert np.isfinite(np.asarray(a["observation_index"])).sum() > 100   # frames contribute
    assert_same_layers(a, b, colored)


@gpu
@pytest.mark.parametrize("shape", [(1, 56), (2, 56), (60, 1), (60, 2)])
def test_process_jpeg_on_strips_of_the_map(shape):
    # a map one or two cells wide, under frames spread over ten times its width: each frame's winners lie in a thin
    # band that falls in the first, the last or a single MCU row (or column) of the frame, or nowhere
    need_cv2()
    camd, poses, files = ortho_case(False, 0, area=(15.0, 28.0))
    a, b = run_both(camd, poses, files, False, shape=shape)
    assert np.isfinite(np.asarray(a["observation_index"])).sum() > 0
    assert_same_layers(a, b, False)


@gpu
def test_a_corrupt_frame_that_contributes_nothing_is_never_decoded():
    need_cv2()
    camd, poses, files = ortho_case(True, 0)
    far = poses[0].copy()
    far[:2] += 5000.0   # sees none of the map
    bad = files[0][:(segment(files[0], 0xDA)[1] + len(files[0])) // 2]   # a scan cut in half
    frames = [imread(f, 3) for f in files] + [np.zeros((camd["height"], camd["width"], 3), np.uint8)]
    a, b = run_both(camd, np.vstack([poses, far]), files + [bad], True, frames)
    assert_same_layers(a, b, True)


@gpu
def test_a_corrupt_contributing_frame_leaves_the_selection_and_no_ortho():
    need_cv2()
    camd, poses, files = ortho_case(False, 0)
    frames = [imread(f, 1) for f in files]   # the selection does not read pixels
    files[4] = files[4][:(segment(files[4], 0xDA)[1] + len(files[4])) // 2]
    a, b = new_map(), new_map()
    before = np.asarray(b["ortho"]).copy()
    amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), a).process(poses, frames, a)
    with pytest.raises(amb.AmbError) as e:
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), b).process_jpeg(poses, files, b)
    assert e.value.status == _lib.AMB_ERR_CORRUPT_DATA
    for name in ("elevation_angle", "observation_index"):
        assert np.array_equal(np.asarray(a[name]).view(np.uint32), np.asarray(b[name]).view(np.uint32)), name
    assert np.array_equal(np.asarray(b["ortho"]), before)


@gpu
def test_size_mismatch_and_unsupported_files_touch_no_layer():
    need_cv2()
    camd, poses, files = ortho_case(False, 0)
    small = cv2_file(content("smooth", 20, 30, seed=1)[:, :, 0].copy(), 90, "420", 0)
    h, w = imread(files[0], 1).shape
    progressive = pil_jpeg(imread(files[1], 1), progressive=True)
    for bad, status in ((small, _lib.AMB_ERR_SIZE_MISMATCH), (progressive, _lib.AMB_ERR_UNSUPPORTED)):
        gm = new_map()
        before = {n: np.asarray(gm[n]).copy() for n in written(False)}
        with pytest.raises(amb.AmbError) as e:
            amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm).process_jpeg(
                poses, files[:3] + [bad] + files[4:], gm)
        assert e.value.status == status
        for n in written(False):
            assert np.array_equal(np.asarray(gm[n]), before[n], equal_nan=True), n
    assert (h, w) == (camd["height"], camd["width"])


# ---- the torch wrapper ----------------------------------------------------------------------------------------------------
@gpu
def test_decode_jpeg_returns_cuda_tensors():
    if EMULATED:
        return   # needs torch.cuda
    z = np.load(GOLDEN)
    files = [z["file_%d" % k].tobytes() for k in range(6)]
    t = amb.decode_jpeg(files, channels=3)
    assert all(x.is_cuda and x.dtype.is_floating_point is False for x in t)
    for k in range(6):
        assert np.array_equal(t[k].cpu().numpy(), z["bgr_%d" % k])
    g = amb.decode_jpeg(files[0], channels=1)
    assert np.array_equal(g.cpu().numpy(), z["gray_0"])
    with pytest.raises(amb.AmbError) as e:
        amb.decode_jpeg([files[0], files[1][:len(files[1]) // 2]])
    assert e.value.status in (_lib.AMB_ERR_CORRUPT_DATA, _lib.AMB_ERR_INVALID_ARGUMENT)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched,pageable", [(None, False), ("reverse", False), ("random:5", False), (None, True)])
def test_this_file_passes_on_the_emulated_kernels(sched, pageable):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_jpeg_decode.py"], sched=sched,
                     opt_in={"AMB_EMU_PAGEABLE": "1"} if pageable else None)
    assert " passed" in tail and "failed" not in tail
