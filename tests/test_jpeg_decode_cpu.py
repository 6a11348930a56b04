"""JPEG frames decoded on the device, the host side (no GPU): amb_jpeg_info against PIL's reading of the same headers and
for every refusal, the Python contracts of jpeg_info / decode_jpeg / io.read_jpeg_files, and the decode fixture
(tests/golden/jpeg_decode_cases.npz) against live OpenCV.  The crafting helpers here are shared with
tests/test_gpu_jpeg_decode.py."""
import ctypes as C
import io
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api  # noqa: E402
from aerial_mapper_b200 import io as amb_io  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "jpeg_decode_cases.npz")


# ---- crafting ---------------------------------------------------------------------------------------------------------
def segments(b):
    """[(marker, start, end)] of the segments from SOI up to and including SOS (end: one past the segment)."""
    out, i = [], 2
    while True:
        assert b[i] == 0xFF
        m = b[i + 1]
        n = struct.unpack(">H", b[i + 2:i + 4])[0]
        out.append((m, i, i + 2 + n))
        if m == 0xDA:
            return out
        i += 2 + n


def segment(b, marker):
    for m, s, e in segments(b):
        if m == marker:
            return s, e
    raise KeyError(hex(marker))


def replace_segment(b, marker, body):
    """b with the first segment of `marker` replaced by `body` (marker and length included); body b"" removes it."""
    s, e = segment(b, marker)
    return b[:s] + body + b[e:]


def sof_marker(b):
    for m, s, e in segments(b):
        if m in (0xC0, 0xC1):
            return m, s, e
    raise KeyError("SOF")


def patch(b, at, value):
    a = bytearray(b)
    a[at] = value
    return bytes(a)


def pil_jpeg(img, **kw):
    from PIL import Image
    bio = io.BytesIO()
    Image.fromarray(img[:, :, ::-1] if img.ndim == 3 else img).save(bio, "JPEG", **kw)
    return bio.getvalue()


def base_file():
    """A 17 x 33 colour 4:2:0 JFIF file (PIL), the starting point of the refusals."""
    rng = np.random.default_rng(7)
    return pil_jpeg(rng.integers(0, 256, (17, 33, 3)).astype(np.uint8), quality=90, subsampling=2)


def refused_files():
    """[(name, file)]: each outside the supported set; every one must give AMB_ERR_UNSUPPORTED."""
    from PIL import Image
    rng = np.random.default_rng(8)
    img = rng.integers(0, 256, (17, 33, 3)).astype(np.uint8)
    b = base_file()
    m, s, e = sof_marker(b)
    out = [("progressive", pil_jpeg(img, progressive=True)),
           ("arithmetic", patch(b, s + 1, 0xC9)), ("lossless", patch(b, s + 1, 0xC3)),
           ("hierarchical", patch(b, s + 1, 0xC5)), ("progressive_marker", patch(b, s + 1, 0xC2)),
           ("12-bit", patch(b, s + 4, 12)), ("dnl_height_0", patch(patch(b, s + 5, 0), s + 6, 0)),
           ("411", patch(b, s + 11, 0x41)), ("440", patch(b, s + 11, 0x12)),
           ("chroma_2x1", patch(b, s + 14, 0x21))]
    # one scan carrying only the first component: multi-scan sequential
    ns, ne = segment(b, 0xDA)
    sos = bytes([0xFF, 0xDA, 0, 8, 1, b[ns + 5], b[ns + 6], 0, 63, 0])
    out.append(("multi_scan", b[:ns] + sos + b[ne:]))
    # 4 components: CMYK with an Adobe segment
    bio = io.BytesIO()
    Image.fromarray(img[:, :, ::-1]).convert("CMYK").save(bio, "JPEG", quality=90)
    out.append(("cmyk_adobe", bio.getvalue()))
    # an Adobe segment on a three-component file (colour transform flag)
    adobe = b"\xFF\xEE\x00\x0EAdobe\x00\x64\x00\x00\x00\x00\x01"
    out.append(("adobe_ycc", b[:2] + adobe + b[2:]))
    # 2 components
    sof = bytearray(b[s:e])
    two = bytes(sof[:4 + 5]) + bytes([2]) + bytes(sof[10:16])
    two = two[:2] + struct.pack(">H", len(two) - 2) + two[4:]
    out.append(("two_components", b[:s] + two + b[e:]))
    # R, G, B component ids without JFIF: libjpeg takes it as RGB
    rgb = bytearray(b)
    for k in range(3):
        rgb[s + 10 + 3 * k] = b"RGB"[k]
    for k in range(3):
        rgb[ns + 5 + 2 * k] = b"RGB"[k]
    out.append(("rgb_ids", replace_segment(bytes(rgb), 0xE0, b"")))
    # EXIF orientation other than 1: cv2.imread would rotate the image
    for o in (3, 6, 8):
        ex = Image.Exif()
        ex[0x0112] = o
        out.append(("exif_orientation_%d" % o, pil_jpeg(img, quality=90, exif=ex.tobytes())))
    # tables left out (Motion-JPEG style)
    out.append(("no_dht", replace_segment(replace_segment(replace_segment(replace_segment(b, 0xC4, b""), 0xC4, b""),
                                                           0xC4, b""), 0xC4, b"")))
    return out


def invalid_files():
    """[(name, file)]: not JPEG, or a malformed header: AMB_ERR_INVALID_ARGUMENT."""
    b = base_file()
    s, e = segment(b, 0xDB)
    return [("empty", b""), ("text", b"not a jpeg at all"), ("soi_only", b"\xFF\xD8"), ("header_cut", b[:e - 5]),
            ("eoi_before_sos", b[:s] + b"\xFF\xD9"), ("bad_segment_length", patch(patch(b, s + 2, 0xFF), s + 3, 0xFF))]


def huff_file(ac_symbol, stream_bits, width=8, height=8):
    """A gray baseline file with one-code tables: DC code '0' -> 0, AC code '0' -> ac_symbol; `stream_bits` ('0'/'1')
    padded with 1s.  For streams no encoder writes (a run past coefficient 63, a code no table holds)."""
    q = b"\xFF\xDB\x00\x43\x00" + bytes([1] * 64)
    sof = b"\xFF\xC0\x00\x0B\x08" + struct.pack(">HH", height, width) + b"\x01\x01\x11\x00"
    dht = b"\xFF\xC4\x00\x14\x00" + bytes([1] + [0] * 15) + b"\x00"
    dht += b"\xFF\xC4\x00\x14\x10" + bytes([1] + [0] * 15) + bytes([ac_symbol])
    sos = b"\xFF\xDA\x00\x08\x01\x01\x00\x00\x3F\x00"
    bits = stream_bits + "1" * (-len(stream_bits) % 8)
    data = bytearray(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))
    data = bytes(data).replace(b"\xFF", b"\xFF\x00")
    return b"\xFF\xD8" + q + sof + dht + sos + data + b"\xFF\xD9"


# ---- amb_jpeg_info ------------------------------------------------------------------------------------------------------
def info(b):
    w, h, c, s, r = C.c_int32(), C.c_int32(), C.c_int(), C.c_int(), C.c_int32()
    st = _lib.lib().amb_jpeg_info(b, len(b), C.byref(w), C.byref(h), C.byref(c), C.byref(s), C.byref(r))
    return st, (w.value, h.value, c.value, s.value, r.value)


def test_info_matches_pil_headers():
    from PIL import Image, JpegImagePlugin
    rng = np.random.default_rng(1)
    for (h, w) in ((1, 1), (17, 9), (250, 333)):
        img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
        for sub in (0, 1, 2):
            for opt in ((False, True) if h < 100 else (False,)):   # (PIL cannot optimise large 4:4:4 noise)
                b = pil_jpeg(img, quality=80, subsampling=sub, optimize=opt)
                im = Image.open(io.BytesIO(b))
                st, (iw, ih, ic, isamp, rst) = info(b)
                assert st == 0 and (iw, ih) == im.size and ic == len(im.getbands()) == 3 and rst == 0
                assert api.JPEG_SAMPLING_NAME[isamp] == {0: "444", 1: "422", 2: "420"}[
                    JpegImagePlugin.get_sampling(im)]
        g = pil_jpeg(img[:, :, 0].copy(), quality=60)
        assert info(g) == (0, (w, h, 1, 1, 0))
    assert amb.jpeg_info(pil_jpeg(np.zeros((5, 7, 3), np.uint8), qtables=[[300] * 64, [300] * 64]))["components"] == 3


def test_info_reads_the_restart_interval():
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(2).integers(0, 256, (40, 50, 3)).astype(np.uint8)
    for rst in (0, 1, 3, 8, 1000):
        ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
        assert amb.jpeg_info(b.tobytes()) == {"width": 50, "height": 40, "components": 3, "sampling": "420",
                                              "restart_interval": rst}


def test_info_refuses_every_unsupported_file():
    for name, b in refused_files():
        assert info(b)[0] == _lib.AMB_ERR_UNSUPPORTED, name
        with pytest.raises(amb.AmbError) as e:
            amb.jpeg_info(b)
        assert e.value.status == _lib.AMB_ERR_UNSUPPORTED, name


def test_info_rejects_malformed_headers():
    for name, b in invalid_files():
        assert info(b)[0] == _lib.AMB_ERR_INVALID_ARGUMENT, name
    # a Huffman table with a full code length (the all-ones code is reserved): libjpeg rejects it too
    assert info(huff_file(0x00, "0").replace(b"\x00\x14\x00\x01", b"\x00\x14\x00\x02"))[0] == _lib.AMB_ERR_INVALID_ARGUMENT
    assert _lib.lib().amb_jpeg_info(None, 10, None, None, None, None, None) == _lib.AMB_ERR_INVALID_ARGUMENT


def test_info_accepts_what_the_decoder_skips():
    b = base_file()
    com = b"\xFF\xFE\x00\x05abc"
    app = b"\xFF\xE5\x00\x06xyzw"
    assert info(b[:2] + com + app + b[2:])[0] == 0
    from PIL import Image
    ex = Image.Exif()
    ex[0x0112] = 1   # orientation 1: nothing to rotate
    assert info(pil_jpeg(np.zeros((9, 9, 3), np.uint8), exif=ex.tobytes()))[0] == 0
    assert info(b[:2] + b"\xFF\xFF" + b[2:])[0] == 0   # fill bytes before a marker
    assert info(huff_file(0xF1, "0"))[0] == 0


def test_app_segments_count_only_at_libjpeg_lengths():
    # jdmarker.c: a JFIF APP0 needs 14 bytes of payload, an Adobe APP14 12.  A file whose ids spell R, G, B is RGB to
    # libjpeg unless a full JFIF segment says otherwise, so with a truncated one it is refused.
    b = base_file()
    m, s, e = sof_marker(b)
    ns, ne = segment(b, 0xDA)
    rgb = bytearray(b)
    for k in range(3):
        rgb[s + 10 + 3 * k] = b"RGB"[k]
        rgb[ns + 5 + 2 * k] = b"RGB"[k]
    rgb = bytes(rgb)
    full, short = segment(rgb, 0xE0)
    assert info(rgb)[0] == 0   # the file's own 16-byte JFIF segment
    assert info(replace_segment(rgb, 0xE0, b"\xFF\xE0\x00\x07JFIF\x00"))[0] == _lib.AMB_ERR_UNSUPPORTED
    assert info(b[:2] + b"\xFF\xEE\x00\x09Adobe\x00\x64" + b[2:])[0] == 0
    assert info(b[:2] + b"\xFF\xEE\x00\x0EAdobe\x00\x64\x00\x00\x00\x00\x01" + b[2:])[0] == _lib.AMB_ERR_UNSUPPORTED
    assert full < short


def test_status_strings():
    L = _lib.lib()
    assert _lib.AMB_ERR_CORRUPT_DATA == -9
    assert b"corrupt" in L.amb_status_string(_lib.AMB_ERR_CORRUPT_DATA)


# ---- Python contracts ---------------------------------------------------------------------------------------------------
def test_python_contracts():
    with pytest.raises(ValueError):
        amb.jpeg_info(12345)
    with pytest.raises(ValueError):
        amb.jpeg_info(np.zeros(4, np.float32))
    with pytest.raises(amb.AmbError):
        amb.jpeg_info(b"\x00\x01")
    with pytest.raises(ValueError):
        amb.decode_jpeg(base_file(), channels=2)
    assert amb.jpeg_info(np.frombuffer(base_file(), np.uint8))["width"] == 33
    assert amb.jpeg_info(bytearray(base_file()))["sampling"] == "420"


def test_read_jpeg_files(tmp_path):
    prefix = str(tmp_path / "frame_")
    blobs = [base_file(), pil_jpeg(np.zeros((3, 4), np.uint8))]
    for i, bl in enumerate(blobs):
        with open("%s%d.jpg" % (prefix, i), "wb") as f:
            f.write(bl)
    assert amb_io.read_jpeg_files(prefix, 2) == blobs
    with pytest.raises(IOError):
        amb_io.read_jpeg_files(prefix, 3)
    with pytest.raises(ValueError):
        amb_io.read_jpeg_files(prefix, 0)
    cv2 = pytest.importorskip("cv2")  # the same errors as load_images_from_file
    with pytest.raises(IOError):
        amb_io.load_images_from_file(prefix, 3)
    with pytest.raises(ValueError):
        amb_io.load_images_from_file(prefix, 0)
    assert cv2 is not None


# ---- the fixture --------------------------------------------------------------------------------------------------------
def test_fixture_equals_live_opencv():
    cv2 = pytest.importorskip("cv2")
    z = np.load(GOLDEN)
    n = len([k for k in z.files if k.startswith("file_")])
    assert n >= 60
    for k in range(n):
        a = z["file_%d" % k]
        assert np.array_equal(cv2.imdecode(a, cv2.IMREAD_COLOR), z["bgr_%d" % k]), k
        assert np.array_equal(cv2.imdecode(a, cv2.IMREAD_GRAYSCALE), z["gray_%d" % k]), k
        assert info(a.tobytes())[0] == 0, k


def test_fixture_covers_the_supported_set():
    z = np.load(GOLDEN)
    seen = set()
    for k in range(len([f for f in z.files if f.startswith("file_")])):
        b = z["file_%d" % k].tobytes()
        st, (w, h, c, s, r) = info(b)
        seen.add((c, s if c == 3 else -1, r > 0, sof_marker(b)[0]))
    assert {(3, 0, False, 0xC0), (3, 1, True, 0xC0), (3, 2, True, 0xC0), (1, -1, False, 0xC0),
            (3, 1, False, 0xC1)} <= seen
