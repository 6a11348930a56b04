"""The device JPEG decoder (csrc/jpeg_decode.cu) on coefficient streams no encoder writes: 16-bit IDCT lanes that wrap
and saturate, DC categories 12..15 and AC categories 11..15, 16-bit codes in a 256-symbol table, runs ending exactly at
k = 63, DC predictors past int16, extreme chroma at every sampling, and scans whose subsequences never self-synchronise.
The files are tests/jpeg_synth.py's case set; every decode is compared byte for byte with the fixture
tests/golden/jpeg_extreme_cases.npz (cv2.imread of the same files on x86) and with the restatement in
tests/jpeg_synth.py, which tests/test_jpeg_synth_cpu.py pins against OpenCV.

The last test runs this file on the emulated kernels (no GPU needed)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import jpeg_synth as js  # noqa: E402
from test_gpu_jpeg_decode import decode, ortho_case, run_both, assert_same_layers  # noqa: E402

gpu = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "jpeg_extreme_cases.npz")


def fixture():
    z = np.load(GOLDEN)
    return z, [k[5:] for k in z.files if k.startswith("file_")]


def assert_decodes(names, extra=()):
    """Decodes the named case files (and the (file, gray, bgr) of `extra`) in one batch per channel count; each must
    equal the fixture and the restatement."""
    z, _ = fixture()
    files = [z["file_" + n].tobytes() for n in names] + [e[0] for e in extra]
    for ch, key in ((1, "gray"), (3, "bgr")):
        rc, status, outs = decode(files, ch)
        assert rc == 0 and status == [0] * len(files), (ch, status)
        for k, name in enumerate(names):
            got = outs[k].image()
            assert np.array_equal(got, z["%s_%s" % (key, name)]), (name, ch)
            assert np.array_equal(got, js.decode(files[k], ch)[0]), (name, ch)
        for k, e in enumerate(extra):
            assert np.array_equal(outs[len(names) + k].image(), e[1 if ch == 1 else 2]), ("extra", k, ch)


def named(prefix):
    names = [n for n in fixture()[1] if n.startswith(prefix)]
    assert names, prefix
    return names


@gpu
@pytest.mark.parametrize("kind", ["deq_wrap", "deq_edges", "even_wrap", "odd_wrap", "pass1_sat", "shortcut", "clamp"])
def test_idct_lanes(kind):
    # each 16-bit wrap or saturation of the SIMD islow lanes in blocks of its own (which ones: test_jpeg_synth_cpu.py)
    assert_decodes(named("lanes_%s_" % kind))


@gpu
def test_extreme_huffman_categories():
    assert_decodes(named("categories_"))


@gpu
def test_runs_ending_at_coefficient_63_with_and_without_eob():
    assert_decodes(["k63_eob", "k63_zrl_tail"])


@gpu
def test_16_bit_codes_and_a_256_symbol_table():
    assert_decodes(["long_codes"])


@gpu
def test_dc_predictor_past_int16_across_subsequences_and_restarts():
    # stored modulo 2^16 from the count kernel's 64-bit sums; one file without restarts, one reset every 48 blocks
    assert_decodes(named("dc_drift_"))


@gpu
def test_extreme_chroma_at_every_sampling_and_mcu_remainder():
    assert_decodes(named("colour_"))


@gpu
def test_a_scan_whose_guesses_never_synchronise():
    # 272 subsequences in one segment, and no guess reaches a true state: the entry states become true only by the
    # decoders carrying them on, 32 subsequences per launch, so the host queues several rounds of 4 launches
    z, _ = fixture()
    m = js.sync_model(z["file_sync_never"].tobytes())
    assert m["rounds"] >= 3 and not any(x for x in m["guess_meets"] if x is not None)
    assert_decodes(["sync_never"])


@gpu
def test_guesses_that_meet_invalid_codes():
    z, _ = fixture()
    m = js.sync_model(z["file_sync_invalid"].tobytes())
    assert sum(1 for x in m["guess_invalid"] if x) >= 20
    assert_decodes(["sync_invalid"])


@gpu
def test_segments_of_whole_subsequences_and_shorter():
    # restart segments of exactly 1, 2 and 3 x 8192 bits, and of 1024 and 3072 bits
    assert_decodes(named("segments_"))


@gpu
def test_one_batch_of_every_case_and_ordinary_files():
    z = np.load(os.path.join(HERE, "golden", "jpeg_decode_cases.npz"))
    extra = [(z["file_%d" % k].tobytes(), z["gray_%d" % k], z["bgr_%d" % k]) for k in range(0, 60, 3)]
    assert_decodes(fixture()[1], extra)


@gpu
@pytest.mark.parametrize("colored", [False, True])
def test_process_jpeg_on_frames_of_extreme_content(colored):
    # the band decode (MCU rows around each frame's winners only) of frames that wrap the IDCT's lanes everywhere
    camd, poses, _ = ortho_case(colored, 0)
    files = js.ortho_frames(len(poses), camd["width"], camd["height"], colored, seed=int(colored))
    frames = [js.decode(f, 3 if colored else 1)[0] for f in files]
    a, b = run_both(camd, poses, files, colored, frames)
    assert np.isfinite(np.asarray(a["observation_index"])).sum() > 100
    assert_same_layers(a, b, colored)


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
@pytest.mark.parametrize("sched", [None, "reverse", "random:5"])
def test_this_file_passes_on_the_emulated_kernels(sched):
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_jpeg_decode_extreme.py"], sched=sched)
    assert " passed" in tail and "failed" not in tail
