"""Kernel-source logic on a box without a GPU: the product's CUDA sources compiled as plain C++ on a CPU stand-in for the
CUDA runtime (tests/emu/README.md — test infrastructure only, never a fallback of the product) and driven through the
normal Python mirror + C ABI by the GPU tests themselves, in a child pytest process with AMB_TEST_EMU=1.

  * the `gpu` tests (all but the few that create inputs with torch.cuda): the emulation reproduces what the GPU
    produced — and re-checks, on every CPU run, the CURRENT sources' kernel and host logic, also under reversed and
    pseudo-random thread scheduling orders.
This does not replace a GPU run (fibers run one after the other: no races, no memory model, no performance)."""
import os
import subprocess
import sys

import pytest

from common import ROOT


OPT_IN = ("AMB_ORTHO_DOMINANCE", "AMB_DSM_STREAM_CHUNKS", "AMB_COMPACT_MIRRORS", "AMB_DSM_PRECISION")


def run_child(marker, files, extra=(), sched=None, opt_in=None):
    env = dict(os.environ, AMB_TEST_EMU="1")
    for k in OPT_IN + ("AMB_EMU_SCHED",):
        env.pop(k, None)
    if opt_in:
        env.update(opt_in)
    if sched:
        env["AMB_EMU_SCHED"] = sched   # order in which the threads of a block take their turns (tests/emu/emu_runtime.cc)
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", marker, "-p", "no:cacheprovider"] + list(extra) + \
          [os.path.join(ROOT, "tests", f) for f in files]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    return tail


@pytest.mark.parametrize("sched", [None, "reverse", "random:5"])
def test_variant_gpu_tests_pass_on_the_emulated_kernels(sched):
    # also with the block's threads scheduled in reverse and in a fresh pseudo-random order every round: a kernel whose
    # result depended on who runs first (e.g. a missing barrier between a write and another thread's read) would differ
    tail = run_child("gpu", ["test_gpu_ortho_dominance.py", "test_gpu_compact_mirrors.py", "test_ortho_from_pcl.py",
                             "test_stereo_rectify.py", "test_gpu_dsm_adversarial.py", "test_gpu_dsm_heights.py",
                             "test_gpu_dsm_binning.py", "test_gpu_stereo_device.py"], sched=sched)
    assert " passed" in tail and "failed" not in tail


def test_validated_gpu_tests_pass_on_the_emulated_kernels_too():
    # everything except the tests that create their inputs on a real device with torch.cuda
    tail = run_child("gpu", ["test_gpu_smoke.py", "test_gpu_refsrc.py", "test_stereo_reproject.py", "test_gpu_dsm.py",
                             "test_gpu_ortho.py", "test_ortho_from_pcl.py", "test_gpu_dsm_adversarial.py",
                             "test_gpu_dsm_heights.py"],
                     extra=["-k", "not large and not full_baseline_size"])
    assert " passed" in tail and "failed" not in tail
    import re
    assert int(re.search(r"(\d+) passed", tail).group(1)) >= 90


def test_validated_gpu_tests_with_every_opt_in_variant_switched_on():
    # chunked DSM with early mirroring + one-byte mirrors, both at once, against the same oracle-backed GPU tests
    tail = run_child("gpu", ["test_gpu_compact_mirrors.py", "test_gpu_ortho.py", "test_gpu_dsm.py",
                             "test_gpu_refsrc.py", "test_gpu_smoke.py"],
                     extra=["-k", "not large and not full_baseline_size"],
                     opt_in={"AMB_DSM_STREAM_CHUNKS": "4", "AMB_COMPACT_MIRRORS": "1"})
    assert " passed" in tail and "failed" not in tail


@pytest.mark.parametrize("tool,seed,cases", [("emu_fuzz_dsm.py", 11, 6), ("emu_fuzz_ortho.py", 12, 8)])
def test_random_cases_on_the_emulated_kernels(tool, seed, cases):
    # tools/emu_fuzz_*.py: random geometry / density / cameras (from 1x1 maps up) against the oracle
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), str(seed), str(cases)], cwd=ROOT,
                       capture_output=True, text=True)
    assert r.returncode == 0 and "fails 0" in r.stdout, (r.stdout + r.stderr)[-2000:]


@pytest.mark.parametrize("colored", [False, True])
def test_cpp_shim_on_the_emulated_kernels_equals_the_reference_build_of_the_same_source(tmp_path, colored):
    # tests/cpp/shim_demo.cc built against the DROP-IN headers + the emulated kernels vs built against the reference's own
    # headers and sources (oracle/_ref): the C++ marshalling of the shim is exercised end to end without a GPU
    import numpy as np
    import test_shim as ts
    from common import ulp_diff
    from oracle import pyoracle as po
    if not po.have_reference_demo():
        pytest.skip("oracle/_ref/libamb_reference_demo.so not built (needs /root/reference)")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    libdir = os.path.dirname(build_emu.build())
    exe = str(tmp_path / "shim_demo_emu")
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-DAMB_SHIM_MINI", "-I" + os.path.join(ROOT, "aerial_mapper_b200", "shim"),
                           os.path.join(ROOT, "tests", "cpp", "shim_demo.cc"), "-o", exe, "-L" + libdir, "-lamb_emu",
                           "-Wl,-rpath," + libdir])
    scen, (rows, cols, res, xyz, camd, poses, imgs) = ts.make_scenario(tmp_path, colored)
    out = tmp_path / "layers.bin"
    r = subprocess.run([exe, str(scen), str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    emu = ts.read_layers(out, rows, cols)
    ref = ts.run_reference_demo(tmp_path, scen, rows, cols)
    assert np.array_equal(np.isnan(emu[0]), np.isnan(ref[0])) and ulp_diff(emu[0], ref[0]).max() <= 1
    same = (emu[2] == ref[2]) | (np.isnan(emu[2]) & np.isnan(ref[2]))
    assert (~same).sum() <= 2
    for k in (3, 4):
        assert (emu[k].view(np.uint32) != ref[k].view(np.uint32))[same].sum() == 0
    assert ulp_diff(emu[1][same], ref[1][same]).max() <= 1


def test_the_product_never_reaches_for_the_emulated_library():
    pkg = os.path.join(ROOT, "aerial_mapper_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".h", ".inc", ".cuh")) or f == "Makefile":
                text = open(os.path.join(dirpath, f)).read()
                assert "libamb_emu" not in text and "tests/emu/" .replace(" ", "") not in text.replace("tests/emu (", "").replace("tests/emu only", ""), f
    assert "AMB_TEST_EMU" not in open(os.path.join(ROOT, "bench.py")).read()
    assert "emu" not in open(os.path.join(ROOT, "__graft_entry__.py")).read()


def test_pageable_staging_logic_on_the_emulated_runtime(tmp_path):
    # csrc/host_staging.cu (worker pool, pinned slots, chunking, slot-wise packing of the frame rectangles) with
    # AMB_EMU_PAGEABLE=1: every caller buffer counts as pageable, so the staged paths run — same layers as the direct path
    import json
    code = r'''
import os, sys, json, ctypes as C
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
import conftest
import numpy as np
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth, _lib
rows, cols, res = 1100, 1000, 0.25            # 4.4 MB layers, 4.8 MB cloud: above the 4 MB staging threshold
xyz = synth.point_cloud(200000, rows * res / 2, cols * res / 2, seed=71, holes=3, hole_sides=(2.0, 6.0))
camd = synth.scaled_camera(0.25)
poses = synth.lawnmower_poses(2, 3, rows * res / 2, cols * res / 2, 150.0, seed=72)
imgs = [synth.procedural_image(k, camd["width"], camd["height"], 1) for k in range(len(poses))]
gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
amb.Dsm(amb.DsmSettings(), gm).process(xyz, gm)
amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm).process(poses, imgs, gm)
np.save(sys.argv[1], np.stack([gm[k] for k in ("elevation", "elevation_angle", "observation_index", "ortho")]))
out = {}
for key in ("staged_h2d_chunks", "staged_d2h_chunks", "staged_rect_slots"):
    s, n = C.c_longlong(0), C.c_longlong(0)
    _lib._lib.amb_emu_counter(key.encode(), C.byref(s), C.byref(n))
    out[key] = int(n.value)
print(json.dumps(out))
''' % (ROOT, ROOT)
    script = tmp_path / "staged.py"
    script.write_text(code)
    import numpy as np
    results = {}
    for pageable in ("1", "0"):
        env = dict(os.environ, AMB_TEST_EMU="1", AMB_EMU_PAGEABLE=pageable)
        out = tmp_path / ("layers_%s.npy" % pageable)
        r = subprocess.run([sys.executable, str(script), str(out)], cwd=ROOT, env=env, capture_output=True, text=True)
        assert r.returncode == 0, (r.stdout + r.stderr)[-2000:]
        results[pageable] = (np.load(out), json.loads(r.stdout.strip().splitlines()[-1]))
    staged, direct = results["1"], results["0"]
    assert staged[1]["staged_h2d_chunks"] >= 3 and staged[1]["staged_d2h_chunks"] >= 3 and staged[1]["staged_rect_slots"] >= 1
    assert direct[1] == {"staged_h2d_chunks": 0, "staged_d2h_chunks": 0, "staged_rect_slots": 0}
    assert np.array_equal(staged[0].view(np.uint32), direct[0].view(np.uint32))


def test_shim_resident_layers_and_repetitions_give_the_same_layers(tmp_path):
    # The drop-in classes share one backend per map geometry.  AMB_SHIM_RESIDENT_LAYERS=1 skips the upload of a layer the
    # backend itself downloaded into that buffer last: in the demo's sequence (DSM, then orthomosaic on the same map) that
    # is the elevation the orthomosaic reads — same layers as the default, host-authoritative mode.
    # A second repetition of the sequence is idempotent in both modes (same cloud -> same elevation; no frame beats its own
    # earlier observation angle), which checks that the shared backend carries no stale state from call to call.  (The
    # demo re-initialises the host layers between repetitions, which the resident mode — by its documented assumption —
    # does not see: idempotence is why the result is still the same.)
    import numpy as np
    import test_shim as ts
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    libdir = os.path.dirname(build_emu.build())
    exe = str(tmp_path / "shim_demo_emu")
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-DAMB_SHIM_MINI", "-I" + os.path.join(ROOT, "aerial_mapper_b200", "shim"),
                           os.path.join(ROOT, "tests", "cpp", "shim_demo.cc"), "-o", exe, "-L" + libdir, "-lamb_emu",
                           "-Wl,-rpath," + libdir])
    scen, (rows, cols, res, xyz, camd, poses, imgs) = ts.make_scenario(tmp_path, False)
    got = {}
    for label, env, reps in (("default", {}, "1"), ("resident", {"AMB_SHIM_RESIDENT_LAYERS": "1"}, "1"),
                             ("default_x2", {}, "2"), ("resident_x2", {"AMB_SHIM_RESIDENT_LAYERS": "1"}, "2")):
        out = tmp_path / ("layers_%s.bin" % label)
        r = subprocess.run([exe, str(scen), str(out), reps], capture_output=True, text=True,
                           env=dict(os.environ, AMB_SHIM_TRACE="1", **env))
        assert r.returncode == 0, r.stderr
        got[label] = (ts.read_layers(out, rows, cols), r.stderr)
    for label in ("resident", "default_x2", "resident_x2"):
        for k in range(4):   # elevation, elevation_angle, observation_index, ortho
            assert np.array_equal(got[label][0][k].view(np.uint32), got["default"][0][k].view(np.uint32)), (label, k)
    assert "[amb shim] Dsm::process: amb_dsm_process" in got["default"][1]   # the AMB_SHIM_TRACE step trace


def test_peer_push_producer_on_local_stand_in_segments(tmp_path):
    # The producer side of the peer-push halo exchange — dsm_partition_kernel<PUSH> + halo_publish (per-tile slot
    # reservation, both sides at once, header {count | stamp << 32}) — needs other ranks' memory on hardware.  The
    # emulated library's test hook amb_emu_self_push (tests/emu/emu_test_hooks.cc) points the two "neighbour segments" at
    # local buffers: the pushed records must be exactly the stripe's border points, and the stripe's elevation must equal
    # the one of the same points binned without a push.
    import json
    code = r'''
import os, sys, json, ctypes as C
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
import conftest
import numpy as np
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth, sharding, _lib
L = _lib._lib
L.amb_emu_self_push.restype = C.c_int
L.amb_emu_self_push.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.c_double, C.c_double, C.c_uint,
                                C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p]
rows, cols, res = 160, 224, 0.5
c0, c1 = 64, 160                      # a middle stripe: both neighbours exist; 96 columns >= reach (35 cells)
center_e = 3.25                       # dsm::Settings::center_easting: the border test uses y - center_easting
xyz_all = synth.point_cloud(90000, rows * res / 2, cols * res / 2, seed=81)
xyz_all[:, 1] += center_e
ids_all = np.arange(len(xyz_all), dtype=np.uint64) * 7 + 3          # global ids: unique, not the array positions
out = {}
def stripe_map():
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0, col_range=(c0, c1))
    return gm
gm = stripe_map()
y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
reach = L.amb_dsm_halo_reach(C.byref(gm.geometry), 1)
ys = xyz_all[:, 1] - center_e
own = (ys > y_lo) & (ys <= y_hi)
xyz = np.ascontiguousarray(xyz_all[own]); ids = np.ascontiguousarray(ids_all[own]); n = len(xyz)
assert n > 3 * 2048                  # several tiles: the per-tile bases matter
exp_up = ids[(xyz[:, 1] - center_e) > y_hi - reach]; exp_down = ids[(xyz[:, 1] - center_e) < y_lo + reach]
assert len(exp_up) > 100 and len(exp_down) > 100
def run(capacity, have_prev, have_next, stamp):
    g = stripe_map()
    amb.check(L.amb_dsm_set_density_hint(g.context(), len(xyz_all) / float(rows * cols)), g.context())
    up = np.zeros(32 * (capacity + 1), np.uint8); down = np.zeros(32 * (capacity + 1), np.uint8)
    st = L.amb_emu_self_push(g.context(), xyz.ctypes.data, ids.ctypes.data, n, 1, center_e, 0.0, capacity, have_prev, have_next,
                             stamp, up.ctypes.data, down.ctypes.data)
    assert st == 0, st
    g.sync(); g.download(("elevation",))
    return up, down, g["elevation"][:, c0:c1].copy()
def parse(seg, capacity):
    hdr = seg[:8].view(np.uint64)[0]
    count, stamp = int(hdr & 0xffffffff), int(hdr >> 32)
    rec = seg[32:32 + 32 * min(count, capacity)].view(np.float64).reshape(-1, 4)
    return count, stamp, rec, rec[:, 3].copy().view(np.uint64)
cap = 20000
up, down, elev = run(cap, 1, 1, 41)
for seg, exp, name in ((up, exp_up, "up"), (down, exp_down, "down")):
    count, stamp, rec, rid = parse(seg, cap)
    assert count == len(exp) and stamp == 41, (name, count, len(exp), stamp)
    order = np.argsort(rid)
    assert np.array_equal(rid[order], np.sort(exp)), name
    src = xyz[np.searchsorted(ids, rid[order])]          # ids are increasing in the own array
    assert np.array_equal(rec[order][:, :3], src), name    # raw (unshifted) coordinates, bit for bit
# one neighbour only: the other segment stays untouched
up1, down1, elev1 = run(cap, 0, 1, 5)
assert not up1.any() and parse(down1, cap)[0] == len(exp_down) and parse(down1, cap)[1] == 5
# a segment that is too small: the true count is published (the consumer raises the overflow flag), slots stay in range
small = 64
up2, down2, _ = run(small, 1, 1, 9)
c2, s2, rec2, rid2 = parse(up2, small)
assert c2 == len(exp_up) and s2 == 9 and len(rid2) == small and np.isin(rid2, exp_up).all()
# the push changes nothing in the binning: same elevation as the plain entry point on the same points
g0 = stripe_map()
amb.check(L.amb_dsm_set_density_hint(g0.context(), len(xyz_all) / float(rows * cols)), g0.context())
amb.check(L.amb_dsm_process_device_ids(g0.context(), xyz.ctypes.data, ids.ctypes.data, n, 1, center_e, 0.0), g0.context())
g0.sync(); g0.download(("elevation",))
ref = g0["elevation"][:, c0:c1]
assert np.array_equal(elev.view(np.uint32), ref.view(np.uint32)) and np.array_equal(elev1.view(np.uint32), ref.view(np.uint32))
print(json.dumps({"n_own": int(n), "up": int(len(exp_up)), "down": int(len(exp_down))}))
''' % (ROOT, ROOT)
    script = tmp_path / "self_push.py"
    script.write_text(code)
    for sched in (None, "reverse"):
        env = dict(os.environ, AMB_TEST_EMU="1")
        if sched:
            env["AMB_EMU_SCHED"] = sched
        r = subprocess.run([sys.executable, str(script)], cwd=ROOT, env=env, capture_output=True, text=True)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        info = json.loads(r.stdout.strip().splitlines()[-1])
        assert info["n_own"] > 6000 and info["up"] > 100 and info["down"] > 100
