"""The synthetic JPEG files of tests/jpeg_synth.py and their restated decode, pinned against OpenCV (no GPU): for every
case file the restatement equals cv2.imdecode, gray and BGR; the fixture tests/golden/jpeg_extreme_cases.npz holds
these same files and equals live OpenCV; amb_jpeg_info reads them; and the case set meets each 16-bit wrap and
saturation of the IDCT, and each synchronisation path, as often as the device tests rely on."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aerial_mapper_b200 as amb  # noqa: E402
import jpeg_synth as js  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "jpeg_extreme_cases.npz")


@pytest.fixture(scope="module")
def cases():
    return js.cases()


@pytest.fixture(scope="module")
def decoded(cases):
    return {name: {ch: js.decode(f, ch) for ch in (1, 3)} for name, f in cases}


def imdecode(cv2, f, ch):
    return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR if ch == 3 else cv2.IMREAD_GRAYSCALE)


def test_restatement_equals_opencv(cases, decoded):
    cv2 = pytest.importorskip("cv2")
    for name, f in cases:
        for ch in (1, 3):
            assert np.array_equal(decoded[name][ch][0], imdecode(cv2, f, ch)), (name, ch)


def test_restatement_equals_opencv_on_random_extreme_files():
    # every sampling and size up to two MCUs, random coefficients of every magnitude, quantisers up to 65535
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    dc, ac = js.standard_tables()
    for trial in range(48):
        sampling = ("gray", "444", "422", "420")[trial % 4]
        w, h = int(rng.integers(1, 34)), int(rng.integers(1, 34))
        qmax, vmax = ((255, 1023), (65535, 32767), (4000, 2000), (2, 32767))[trial // 4 % 4]
        planes = []
        for s in js.plane_shapes(w, h, sampling):
            p = rng.integers(-vmax, vmax + 1, s + (64,))
            p[rng.random(s + (64,)) < 0.5] = 0
            p[..., 0] = rng.integers(-16383, 16384, s)
            planes.append(p)
        q = [rng.integers(1, qmax + 1, 64) for _ in planes]
        f = js.write(planes, w, h, sampling, q, [dc] * len(planes), [ac] * len(planes), restart=trial % 3)
        for ch in (1, 3):
            assert np.array_equal(js.decode(f, ch)[0], imdecode(cv2, f, ch)), (trial, ch)


def test_fixture_holds_the_case_set_and_equals_live_opencv(cases):
    z = np.load(GOLDEN)
    names = [k[5:] for k in z.files if k.startswith("file_")]
    assert sorted(names) == sorted(n for n, _ in cases)
    cv2 = None
    try:
        import cv2
    except ImportError:
        pass
    for name, f in cases:
        assert z["file_" + name].tobytes() == f, name   # the writer is deterministic
        if cv2 is not None:
            assert np.array_equal(imdecode(cv2, f, 3), z["bgr_" + name]), name
            assert np.array_equal(imdecode(cv2, f, 1), z["gray_" + name]), name


def test_the_files_parse(cases):
    for name, f in cases:
        i = amb.jpeg_info(f)
        F = js.Frame(f)
        assert (i["width"], i["height"], i["components"], i["restart_interval"]) == \
            (F.width, F.height, F.ncomp, F.restart), name
    sofs = {js.Frame(f).sof for _, f in cases}
    assert sofs == {0xC0, 0xC1}


def test_the_case_set_meets_every_idct_wrap(decoded):
    totals = {k: 0 for k in js.IDCT_FLAGS}
    for name, d in decoded.items():
        for k in js.IDCT_FLAGS:
            totals[k] += d[3][1]["flags"][k]
    assert min(totals.values()) >= 200, totals
    # each lane case meets its own wrap in every block, and the shortcut case with row-0 AC terms
    for name, d in decoded.items():
        f = d[3][1]["flags"]
        n = d[3][1]["coef"][0].shape[0] * d[3][1]["coef"][0].shape[1]
        if name.startswith("lanes_") and not name.startswith("lanes_clamp") and not name.startswith("lanes_deq_edges"):
            kind = name[6:-2]
            assert f[kind] == n, (name, f)
        if name.startswith("lanes_deq_edges"):
            assert f["deq_wrap"] == 0 and f["deq_max"] > n // 2 and f["deq_min"] > n // 2, (name, f)
        if name.startswith("lanes_shortcut"):
            assert f["shortcut_row0_ac"] == f["shortcut_wrap"] == n and f["deq_wrap"] == 0, (name, f)
        if name.startswith("lanes_clamp"):
            assert f["deq_wrap"] == f["even_wrap"] == f["odd_wrap"] == 0 and f["clamp_lo"] and f["clamp_hi"], (name, f)


def test_the_case_set_meets_the_entropy_edges(cases, decoded):
    dc_cats, ac_cats, lengths = set(), set(), set()
    for name, f in cases:
        F = decoded[name][1][1]["frame"]
        pos, j, k = 0, 0, 0
        for s in range(len(F.seg_bytes) - 1):
            pos, j, k = 8 * F.seg_bytes[s], 0, 0
            blocks = F.bpm * (min((s + 1) * F.ri, F.n_mcu) - s * F.ri)
            while blocks:
                c = F.blk_comp[j]
                tab = F.dc[c] if k == 0 else F.ac[c]
                length, sym = tab.look[int(F.bits[pos:pos + 16], 2)]
                lengths.add(length)
                (dc_cats if k == 0 else ac_cats).add(sym if k == 0 else sym & 15)
                pos, j, k = F.step(pos, j, k)[:3]
                blocks -= k == 0
    assert set(range(12, 16)) <= dc_cats and set(range(11, 16)) <= ac_cats
    assert 16 in lengths
    long_codes = js.Frame(dict(cases)["long_codes"])
    assert sum(1 for e in set(map(tuple, [x for x in long_codes.ac[0].look if x]))) == 256
    # blocks whose run ends exactly at k = 63, with and without an EOB, and with ZRLs to k = 64
    assert dict(cases)["k63_zrl_tail"] != dict(cases)["k63_eob"]
    assert np.array_equal(decoded["k63_zrl_tail"][1][1]["coef"][0], decoded["k63_eob"][1][1]["coef"][0])
    assert np.count_nonzero(decoded["k63_eob"][1][1]["coef"][0][..., 63]) >= 8


def test_the_dc_predictor_drifts_past_int16(decoded):
    for name in ("dc_drift_0", "dc_drift_1", "sync_never"):
        info = decoded[name][1][1]
        F, pred, start = info["frame"], info["pred"][0], info["start"][0]
        far = np.abs(pred) > 32767
        assert far.sum() >= 40, name
        # past int16 in subsequences other than their segment's first
        seg_start = np.array(F.seg_bytes[:-1]) * 8
        rel = start - seg_start[np.searchsorted(seg_start, start, side="right") - 1]
        assert (far & (rel >= js.SUB_BITS)).sum() >= 10, name
        assert np.array_equal(info["coef"][0][..., 0], js.wrap16(pred).astype(np.int16)), name
    assert js.Frame(dict(js.cases())["dc_drift_1"]).restart == 48


def test_the_sync_cases_take_the_paths_they_are_for():
    c = dict(js.sync_cases())
    never = js.sync_model(c["sync_never"])
    assert never["subs"][0] > 2 * js.SYNC_LAUNCHES_PER_READ * js.SYNC_HOPS
    assert not any(m for m in never["guess_meets"] if m is not None)
    assert never["rounds"] >= 3
    inv = js.sync_model(c["sync_invalid"])
    assert sum(1 for m in inv["guess_invalid"] if m) >= 20 and inv["invalid_marks"] >= 20
    seen = set()
    for ri in (1, 3, 8, 16, 24):
        F = js.Frame(c["segments_ri%d" % ri])
        bits = [8 * (F.seg_bytes[s + 1] - F.seg_bytes[s]) for s in range(len(F.seg_bytes) - 1)]
        seen |= {b // js.SUB_BITS if b % js.SUB_BITS == 0 else -1 for b in bits}
        seen |= {0 for b in bits if b < js.SUB_BITS}
    assert {0, 1, 2, 3} <= seen


def test_the_sync_model_on_the_fixture_files_of_ordinary_encoders():
    # real content: the guesses synchronise within a launch or two (the model is not pessimistic by construction)
    z = np.load(os.path.join(HERE, "golden", "jpeg_decode_cases.npz"))
    for k in range(0, 60, 7):
        m = js.sync_model(z["file_%d" % k].tobytes())
        assert m["launches"] <= 3 and m["rounds"] == 1, k


def test_restatement_equals_opencv_on_the_orthomosaic_frames():
    cv2 = pytest.importorskip("cv2")
    for colored in (False, True):
        for f in js.ortho_frames(3, 200, 150, colored, seed=int(colored)):
            for ch in ((1, 3) if colored else (1,)):
                assert np.array_equal(js.decode(f, ch)[0], imdecode(cv2, f, ch)), (colored, ch)
