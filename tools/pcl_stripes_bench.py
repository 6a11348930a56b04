"""OrthoFromPcl (ortho-from-pcl.cc:20-113) on the joint_10k cloud of bench.py (50 M points, 10000 x 10000 cells at
0.25 m) with seeded intensities, radius 2, plain and adaptive (the adaptive runs on the cloud with bench.py's 3000
holes of 1-8 m):
  whole     one context owning the whole map (amb_ortho_from_pcl_process);
  stripes   two column-stripe contexts on device 0, each given the whole cloud, one after the other — what every device
            of amb_multi does, so the cost of a stripe (adaptive: the second, whole-map binning) is visible on one GPU;
  multi     amb_multi_ortho_from_pcl_process over all visible GPUs ("not measured" below two devices).
Reports per configuration the median wall time of the blocking host call, the library's CUDA-event stage times of the
last step (amb_get_timings, dsm_* fields; the adaptive pass runs after dsm_total_ms and shows in the wall time only),
whether every stripe's bits equal the whole-map run, and the card's name and power limit.  One JSON line per
configuration.  Developer tool: numbers go to DESIGN.md with the card they were measured on.

    python tools/pcl_stripes_bench.py [--workload joint_10k] [--steps 5] [--warmup 2] [--radius 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import bench
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import sharding


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "devices": torch.cuda.device_count()}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    walls = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        walls.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(walls)), float(min(walls)), float(max(walls))


def stage_times(ctx):
    t = amb._lib.Timings()
    amb.check(amb.lib().amb_get_timings(ctx, C.byref(t)), ctx)
    d = t.as_dict()
    return {k: (round(v, 3) if isinstance(v, float) else v) for k, v in d.items() if k.startswith("dsm_")}


def run_contexts(g, ranges, devices, xyz, inten, radius, adaptive, steps, warmup):
    """One blocking amb_ortho_from_pcl_process per context, one after the other; returns (ortho slabs, record)."""
    L = amb.lib()
    ctxs = []
    for (c0, c1), dev in zip(ranges, devices):
        ctx = C.c_void_p()
        amb.check(L.amb_create(C.byref(g), int(dev), int(c0), int(c1), C.byref(ctx)))
        ctxs.append(ctx)
    n = len(xyz)
    px, pi = xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p)
    try:
        def step():
            for ctx in ctxs:
                amb.check(L.amb_init_layers(ctx), ctx)
                amb.check(L.amb_ortho_from_pcl_process(ctx, px, pi, n, int(radius), 1 if adaptive else 0), ctx)
        med, lo, hi = timed(step, steps, warmup)
        slabs = []
        for (c0, c1), ctx in zip(ranges, ctxs):
            s = np.empty((g.rows, c1 - c0), np.float32, order="F")
            amb.check(L.amb_download_layer(ctx, amb.LAYER_ID["ortho"], s.ctypes.data_as(C.c_void_p)), ctx)
            slabs.append(s)
        return slabs, {"wall_ms_median": round(med, 2), "wall_ms_min": round(lo, 2), "wall_ms_max": round(hi, 2),
                       "stages": [stage_times(ctx) for ctx in ctxs]}
    finally:
        for ctx in ctxs:
            L.amb_destroy(ctx)


def run_multi(g, n_gpus, xyz, inten, radius, adaptive, steps, warmup):
    L = amb.lib()
    m = C.c_void_p()
    amb.check(L.amb_multi_create(C.byref(g), int(n_gpus), C.byref(m)))
    px, pi = xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p)
    try:
        def step():
            amb.check(L.amb_multi_init_layers(m))
            st = L.amb_multi_ortho_from_pcl_process(m, px, pi, len(xyz), int(radius), 1 if adaptive else 0)
            if st != 0:
                raise amb.AmbError(st, L.amb_multi_last_error(m).decode())
        med, lo, hi = timed(step, steps, warmup)
        full = np.empty((g.rows, g.cols), np.float32, order="F")
        amb.check(L.amb_multi_download_layer(m, amb.LAYER_ID["ortho"], full.ctypes.data_as(C.c_void_p)))
        ranges = []
        for r in range(L.amb_multi_size(m)):
            ranges.append(sharding.stripe_range(g.cols, r, L.amb_multi_size(m)))
        stages = [stage_times(L.amb_multi_context(m, r)) for r in range(L.amb_multi_size(m))]
        return full, ranges, {"wall_ms_median": round(med, 2), "wall_ms_min": round(lo, 2), "wall_ms_max": round(hi, 2),
                              "stages": stages}
    finally:
        L.amb_multi_destroy(m)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="joint_10k", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--radius", type=int, default=2)
    ap.add_argument("--holes", type=int, default=3000)
    args = ap.parse_args()
    if amb.lib().amb_device_count() <= 0:
        raise SystemExit("pcl_stripes_bench: no CUDA device (the hot path has no CPU fallback)")
    wl = bench.WORKLOADS[args.workload]
    rows, cols, res, half_x, half_y, _, _ = bench.workload_inputs(wl)
    n = wl["n_points"]
    dev = torch.device("cuda:0")
    info = card()
    g = amb.Geometry()
    amb.check(amb.lib().amb_geometry_init(rows * res, cols * res, res, 0.0, 0.0, C.byref(g)))
    gen = torch.Generator(device=dev)
    gen.manual_seed(5)
    clouds = {}
    for label, holes in (("plain", None), ("holes", bench.hole_rectangles(dict(holes=args.holes, hole_sides=(1.0, 8.0)),
                                                                          half_x, half_y))):
        xyz = bench.device_point_cloud(torch, n, half_x, half_y, dev, holes=holes)
        inten = torch.randint(0, 256, (xyz.shape[0],), generator=gen, device=dev, dtype=torch.int32)
        clouds[label] = (xyz.cpu().pin_memory().numpy(), inten.cpu().pin_memory().numpy())
        del xyz, inten
    torch.cuda.empty_cache()
    half = cols // 2 + 7   # two ragged stripes
    n_dev = info["devices"]
    for adaptive in (False, True):
        xyz, inten = clouds["holes" if adaptive else "plain"]
        common = {"workload": args.workload, "points": int(len(xyz)), "radius": args.radius, "adaptive": adaptive,
                  "card": info}
        (full,), rec = run_contexts(g, [(0, cols)], [0], xyz, inten, args.radius, adaptive, args.steps, args.warmup)
        print(json.dumps(dict(common, config="whole", **rec)), flush=True)
        ranges = [(0, half), (half, cols)]
        slabs, rec = run_contexts(g, ranges, [0, 0], xyz, inten, args.radius, adaptive, args.steps, args.warmup)
        same = all(np.array_equal(s.view(np.uint32), full[:, c0:c1].view(np.uint32)) for s, (c0, c1) in zip(slabs, ranges))
        print(json.dumps(dict(common, config="stripes_on_device_0", stripes=ranges, bits_equal_whole=same, **rec)),
              flush=True)
        del slabs
        if n_dev >= 2:
            got, ranges, rec = run_multi(g, n_dev, xyz, inten, args.radius, adaptive, args.steps, args.warmup)
            same = all(np.array_equal(got[:, c0:c1].view(np.uint32), full[:, c0:c1].view(np.uint32)) for c0, c1 in ranges)
            print(json.dumps(dict(common, config="multi", n_gpus=n_dev, bits_equal_whole=same, **rec)), flush=True)
        else:
            print(json.dumps(dict(common, config="multi", n_gpus=n_dev, result="not measured (one visible GPU)")),
                  flush=True)


if __name__ == "__main__":
    main()
