"""Baseline JPEG encoding (amb_jpeg_encode_device / amb_export_jpeg, csrc/jpeg_encode.cu) against cv2.imencode, on one GPU.

    python tools/jpeg_encode_bench.py [--launches 50] [--repeats 5] [--out DIR]

Input: the orthomosaics of the joint workload's 10000 x 10000 map (bench.py joint_10k: 0.25 m cells, 250 frames of
4000 x 3000), gray `ortho` and `colored_ortho`, rendered on the analytic terrain, exported with amb_export_raster_device.
Device: amb_jpeg_encode_device of the exported band for GRAY8, BGR8 4:2:0 and BGR8 4:4:4 at quality 95, CUDA events
over --launches calls after warm-up (each call ends with the file in pinned host memory, so this is the whole encode
including its D2H copy).  Host API: GridMap.to_jpeg (export + encode + copy into a pageable buffer), best of --repeats.
cv2.imencode of the same image on this host's CPU, best of 3.  Prints the card's name and power limit and one JSON
line; writes it to --out/jpeg_encode_bench.json if given."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, synth  # noqa: E402
import bench  # noqa: E402


def best(fn, repeats):
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import cv2
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("jpeg_encode_bench: no CUDA device (nothing is measured without one)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    wl = bench.WORKLOADS["joint_10k"]
    rows, cols, res, half_x, half_y, camd, poses = bench.workload_inputs(wl)
    names = ("ortho", "colored_ortho", "elevation", "elevation_angle", "observation_index")
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res), layer_names=names).getMutable()
    gm.layers["elevation"][...] = synth.analytic_elevation(rows, cols, res)
    gm.to_device(0, names=names)
    W, H = camd["width"], camd["height"]
    for colored in (False, True):
        ch = 3 if colored else 1
        imgs = synth.procedural_images_torch(len(poses), W, H, ch, "cuda:0")
        torch.cuda.synchronize()
        amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm).process_device(
            poses, [imgs[k].data_ptr() for k in range(len(poses))], W * ch, gm)
        gm.sync()
        del imgs
        torch.cuda.empty_cache()
    ctx = gm.context()
    L = amb.lib()
    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    out = {"card": q, "width": rows, "height": cols, "quality": 95, "launches": args.launches, "cases": {}}
    for label, name, fmt, sampling in (("gray8", "ortho", "gray8", "420"), ("bgr8_420", "colored_ortho", "bgr8", "420"),
                                       ("bgr8_444", "colored_ortho", "bgr8", "444")):
        f = _lib.RASTER_FORMAT[fmt]
        ch = 3 if fmt == "bgr8" else 1
        band = torch.empty(rows * cols * ch, dtype=torch.uint8, device="cuda:0")
        amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID[name], f, band.data_ptr()), ctx)
        gm.sync()
        host_img = band.cpu().numpy().reshape((cols, rows) + ((3,) if ch == 3 else ()))
        s = api.JPEG_SAMPLING[sampling]
        cap = int(L.amb_jpeg_max_size(rows, cols, ch, 95, s, 0))
        p = C.c_void_p()
        amb.check(L.amb_host_alloc(C.byref(p), cap))
        size = C.c_size_t(0)

        def enc():
            amb.check(L.amb_jpeg_encode_device(ctx, band.data_ptr(), rows, cols, rows * ch, ch, 95, s, 0, p, cap,
                                               C.byref(size)), ctx)

        for _ in range(3):
            enc()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.launches):
            enc()
        e1.record(stream)
        e1.synchronize()
        dev_ms = e0.elapsed_time(e1) / args.launches
        ours = bytes((C.c_uint8 * size.value).from_address(p.value))
        api_ms = 1e3 * best(lambda: gm.to_jpeg(name, 95, sampling, 0, fmt=fmt), args.repeats)
        params = [cv2.IMWRITE_JPEG_QUALITY, 95]
        if ch == 3:
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == "420"
                       else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
        ref = cv2.imencode(".jpg", host_img, params)[1].tobytes()
        cv2_ms = 1e3 * best(lambda: cv2.imencode(".jpg", host_img, params), 3)
        out["cases"][label] = {"device_ms": dev_ms, "host_api_ms": api_ms, "cv2_ms": cv2_ms, "bytes": len(ours),
                               "identical": ours == ref, "speedup_device_vs_cv2": cv2_ms / dev_ms,
                               "speedup_api_vs_cv2": cv2_ms / api_ms}
        L.amb_host_free(p)
        del band
    out["cv2"] = {"version": cv2.__version__, "threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}
    line = json.dumps(out)
    print("card:", q)
    for label, r in out["cases"].items():
        print("%-9s device %.2f ms  host API %.2f ms  cv2 %.1f ms  (%.0fx / %.0fx)  %.1f MB  identical %s"
              % (label, r["device_ms"], r["host_api_ms"], r["cv2_ms"], r["speedup_device_vs_cv2"],
                 r["speedup_api_vs_cv2"], r["bytes"] / 1e6, r["identical"]))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_encode_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
