"""The producers of a sharded cloud's border halo (aerial_mapper_b200/csrc/halo_push.h) against the border sets computed in
numpy, on the emulated kernels (tests/emu/README.md).  Three of them fill exchange segments and need other ranks on
hardware: the peer push of the binning's partition kernel, the compaction of the send/recv exchange (one segment per
side) and the compaction of the all-gather exchange (one segment for both sides).  The emulated library's test hook
amb_emu_halo_segments (tests/emu/emu_test_hooks.cc) points their segments at local buffers.  The fourth,
amb_dsm_extract_halo / amb_ortho_from_pcl_extract_halo, is public and runs on the same points.  Every producer must
yield exactly the stripe's border points, with their ids, their coordinates (or intensities) bit for bit and the true
count, for Dsm (y shifted by center_easting) and OrthoFromPcl (the intensity as the record's z).  With too small a
capacity the true count is still reported and the stored slots stay in range."""
import json
import os
import subprocess
import sys

import pytest

from common import ROOT

SCRIPT = r'''
import os, sys, json, ctypes as C
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
import conftest
import numpy as np
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth, sharding, _lib
L = _lib._lib
L.amb_emu_halo_segments.restype = C.c_int
L.amb_emu_halo_segments.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32,
                                    C.c_double, C.c_double, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p]
PUSH, SPLIT, ALL_GATHER = 0, 1, 2
rows, cols, res = 160, 224, 0.5
c0, c1 = 64, 160                      # a middle stripe: both neighbours exist; 96 columns >= reach (35 cells)
pcl = sys.argv[1] == "pcl"
center_e = 0.0 if pcl else 3.25       # dsm::Settings::center_easting: the border test uses y - center_easting
xyz_all = synth.point_cloud(90000, rows * res / 2, cols * res / 2, seed=81)
xyz_all[:, 1] += center_e
ids_all = np.arange(len(xyz_all), dtype=np.uint64) * 7 + 3          # global ids: unique, not the array positions
inten_all = np.random.default_rng(82).integers(-1000, 100000, len(xyz_all)).astype(np.int32)
def stripe_map():
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0, col_range=(c0, c1))
    amb.check(L.amb_dsm_set_density_hint(gm.context(), len(xyz_all) / float(rows * cols)), gm.context())
    return gm
gm = stripe_map()
y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
reach = L.amb_dsm_halo_reach(C.byref(gm.geometry), 1)
ys = xyz_all[:, 1] - center_e
own = (ys > y_lo) & (ys <= y_hi)
xyz = np.ascontiguousarray(xyz_all[own]); ids = np.ascontiguousarray(ids_all[own]); n = len(xyz)
inten = np.ascontiguousarray(inten_all[own])
assert n > 3 * 2048                  # several tiles: the per-tile bases of the push matter
up_mask = (xyz[:, 1] - center_e) > y_hi - reach
down_mask = (xyz[:, 1] - center_e) < y_lo + reach
exp_up, exp_down, exp_any = ids[up_mask], ids[down_mask], ids[up_mask | down_mask]
assert len(exp_up) > 100 and len(exp_down) > 100 and len(exp_any) < 40000
# what a record carries: raw (unshifted) x, y and z, or the intensity as z
rec_src = xyz.copy()
if pcl:
    rec_src[:, 2] = inten.astype(np.float64)
out_layer = "ortho" if pcl else "elevation"
def run(producer, capacity, have_prev=1, have_next=1, stamp=0):
    g = stripe_map()
    # (GUARD bytes beyond each segment: no producer may write there)
    up = np.zeros(32 * (capacity + 1) + GUARD, np.uint8); down = np.zeros(32 * (capacity + 1) + GUARD, np.uint8)
    st = L.amb_emu_halo_segments(g.context(), producer, xyz.ctypes.data, inten.ctypes.data if pcl else None,
                                 ids.ctypes.data, n, 1, center_e, 0.0, capacity, have_prev, have_next, stamp,
                                 up.ctypes.data, down.ctypes.data)
    assert st == 0, st
    g.sync()
    layer = None
    if producer == PUSH:
        g.download((out_layer,))
        layer = g[out_layer][:, c0:c1].copy()
    return up, down, layer
def parse(seg, capacity):
    hdr = seg[:8].view(np.uint64)[0]
    count, stamp = int(hdr & 0xffffffff), int(hdr >> 32)
    rec = seg[32:32 + 32 * min(count, capacity)].view(np.float64).reshape(-1, 4)
    return count, stamp, rec, rec[:, 3].copy().view(np.uint64) & np.uint64(0xffffffff)   # readers use the low 32 bits
def check_records(rid, rec, exp, name):
    order = np.argsort(rid)
    assert np.array_equal(rid[order], np.sort(exp) & np.uint64(0xffffffff)), name
    src = rec_src[np.searchsorted(ids & np.uint64(0xffffffff), rid[order])]   # ids are increasing in the own array
    assert np.array_equal(rec[order][:, :3].view(np.uint64), src.view(np.uint64)), name
def check_segment(seg, capacity, exp, stamp, name):
    count, s, rec, rid = parse(seg, capacity)
    assert count == len(exp) and s == stamp, (name, count, len(exp), s)
    check_records(rid, rec, exp, name)
cap, small, GUARD = 40000, 64, 4096
done = []
# the peer push, both neighbours
up, down, layer = run(PUSH, cap, 1, 1, 41)
check_segment(up, cap, exp_up, 41, "push up"); check_segment(down, cap, exp_down, 41, "push down")
# one neighbour only: the other segment stays untouched
up1, down1, layer1 = run(PUSH, cap, 0, 1, 5)
assert not up1.any()
check_segment(down1, cap, exp_down, 5, "push down, no rank - 1")
# the push changes nothing in the binning: same layer as the plain entry point on the same points
g0 = stripe_map()
if pcl:
    st = L.amb_ortho_from_pcl_process_device_ids(g0.context(), xyz.ctypes.data, inten.ctypes.data, ids.ctypes.data, n, 1, 0)
else:
    st = L.amb_dsm_process_device_ids(g0.context(), xyz.ctypes.data, ids.ctypes.data, n, 1, center_e, 0.0)
amb.check(st, g0.context())
g0.sync(); g0.download((out_layer,))
ref = g0[out_layer][:, c0:c1]
assert np.array_equal(layer.view(np.uint32), ref.view(np.uint32)) and np.array_equal(layer1.view(np.uint32), ref.view(np.uint32))
done.append("push")
# the compaction of the send/recv exchange: one segment per side (headers zeroed: stamp 0)
up, down, _ = run(SPLIT, cap)
check_segment(up, cap, exp_up, 0, "split up"); check_segment(down, cap, exp_down, 0, "split down")
done.append("split")
# the compaction of the all-gather exchange: both sides in one segment, a point on both sides once
up, down, _ = run(ALL_GATHER, cap)
check_segment(up, cap, exp_any, 0, "all-gather")
assert not down[:32].any()
done.append("all_gather")
# too small a segment: the true count is published (the consumer raises the overflow flag), slots stay in range
for producer, stamp in ((PUSH, 9), (SPLIT, 0), (ALL_GATHER, 0)):
    up2, down2, _ = run(producer, small, 1, 1, stamp)
    for seg, exp in (((up2, exp_any),) if producer == ALL_GATHER else ((up2, exp_up), (down2, exp_down))):
        c2, s2, rec2, rid2 = parse(seg, small)
        assert c2 == len(exp) and s2 == stamp and len(rid2) == small, (producer, c2, s2)
        assert np.isin(rid2, exp).all() and len(np.unique(rid2)) == small, producer
        check_records(rid2, rec2, rid2, producer)
        assert not seg[32 * (small + 1):].any(), producer        # nothing beyond the last slot
# the public SoA extraction on the same points
g = stripe_map()
for capacity in (cap, small):
    out_xyz = np.zeros((capacity + 8, 3)); out_ids = np.zeros(capacity + 8, np.uint64)
    out_int = np.zeros(capacity + 8, np.int32); count = np.zeros(1, np.uint32)
    if pcl:
        st = L.amb_ortho_from_pcl_extract_halo(g.context(), xyz.ctypes.data, inten.ctypes.data, ids.ctypes.data, n, y_lo, y_hi,
                                               reach, out_xyz.ctypes.data, out_int.ctypes.data, out_ids.ctypes.data,
                                               capacity, count.ctypes.data)
    else:
        st = L.amb_dsm_extract_halo(g.context(), xyz.ctypes.data, ids.ctypes.data, n, y_lo, y_hi, reach, center_e,
                                    out_xyz.ctypes.data, out_ids.ctypes.data, capacity, count.ctypes.data)
    amb.check(st, g.context())
    g.sync()
    k = min(len(exp_any), capacity)
    assert int(count[0]) == len(exp_any), (int(count[0]), len(exp_any))
    assert not out_ids[k:].any() and not out_xyz[k:].any() and not out_int[k:].any()   # slots stay in range
    rid = out_ids[:k]
    if capacity == cap:
        assert np.array_equal(np.sort(rid), np.sort(exp_any))
    else:
        assert np.isin(rid, exp_any).all() and len(np.unique(rid)) == k
    pos = np.searchsorted(ids, rid)
    assert np.array_equal(out_xyz[:k].view(np.uint64), xyz[pos].view(np.uint64))
    if pcl:
        assert np.array_equal(out_int[:k], inten[pos])
done.append("extract_halo")
print(json.dumps({"n_own": int(n), "up": int(len(exp_up)), "down": int(len(exp_down)), "producers": done}))
'''


@pytest.mark.parametrize("sched", [None, "reverse"])
@pytest.mark.parametrize("pass_", ["dsm", "pcl"])
def test_halo_producers_on_local_stand_in_segments(tmp_path, pass_, sched):
    script = tmp_path / "halo_producers.py"
    script.write_text(SCRIPT % (ROOT, ROOT))
    env = dict(os.environ, AMB_TEST_EMU="1")
    env.pop("AMB_EMU_SCHED", None)
    if sched:
        env["AMB_EMU_SCHED"] = sched   # order in which the threads of a block take their turns (tests/emu/emu_runtime.cc)
    r = subprocess.run([sys.executable, str(script), pass_], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert info["n_own"] > 6000 and info["up"] > 100 and info["down"] > 100
    assert info["producers"] == ["push", "split", "all_gather", "extract_halo"]
