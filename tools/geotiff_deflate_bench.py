"""Deflate GeoTIFF strips (amb_deflate_strips_device / GridMap.to_geotiff, csrc/deflate_encode.cu) against host zlib, on
one GPU.

    python tools/geotiff_deflate_bench.py [--launches 50] [--repeats 5] [--out DIR]

Rasters: the joint workload's 10000 x 10000 map at 0.25 m (bench.py joint_10k) in four variants: a DSM-like F32
elevation (analytic terrain, 5 cm noise, NaN holes), the gray and colour orthomosaics of tools/jpeg_encode_bench.py
(250 frames of 4000 x 3000 rendered on the analytic terrain) and the observation_index mask (MASK8), each exported
with amb_export_raster_device, in libtiff's default 8 KiB strips.
Device: amb_deflate_strips_device of the exported band, CUDA events over --launches calls after warm-up, each ending
with the file's strips in pinned host memory.  Host API: GridMap.to_geotiff to a file in a temporary directory, best
of --repeats.  Baseline: zlib.compress at levels 1 and 6 of the same predicted strips on all of this host's threads
(zlib releases the GIL).  Every device file is checked to inflate to the predicted strips.  Prints the card's name and
power limit and one JSON line; writes it to --out/geotiff_deflate_bench.json if given."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402
import bench  # noqa: E402


def best(fn, repeats):
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def predicted_strips(img, fmt, rps):
    """The TIFF predictor of include/aerial_mapper_b200.h (amb_deflate_strips_device), strip by strip."""
    h = img.shape[0]
    if fmt == "f32":
        be = img.astype(">f4").view(np.uint8).reshape(h, img.shape[1], 4)
        b = np.ascontiguousarray(be.transpose(0, 2, 1)).reshape(h, -1)
        step = 1
    else:
        b = np.ascontiguousarray(img[:, :, ::-1] if fmt == "bgr8" else img).reshape(h, -1)
        step = 3 if fmt == "bgr8" else 1
    d = b.copy()
    d[:, step:] -= b[:, :-step]
    return [d[s:s + rps].tobytes() for s in range(0, h, rps)]


BENCH_LAYERS = (("elevation", "f32"), ("ortho", "gray8"), ("colored_ortho", "bgr8"), ("observation_index", "mask8"))


def bench_map():
    """The joint workload's 10000 x 10000 map on cuda:0 with the four rasters of this benchmark: the gray and colour
    orthomosaics of its 250 frames rendered on the analytic terrain, their observation_index, and then, in the elevation
    layer, the terrain with 5 cm noise and NaN holes (a DSM-like DEM)."""
    import torch
    wl = bench.WORKLOADS["joint_10k"]
    rows, cols, res, half_x, half_y, camd, poses = bench.workload_inputs(wl)
    names = ("ortho", "colored_ortho", "elevation", "elevation_angle", "observation_index")
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res), layer_names=names).getMutable()
    terrain = synth.analytic_elevation(rows, cols, res)
    gm.layers["elevation"][...] = terrain
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
    # the DSM-like elevation: terrain + 5 cm noise + NaN holes, uploaded after the orthomosaics were rendered on the
    # smooth terrain
    rng = np.random.default_rng(0)
    dem = (terrain + rng.normal(0.0, 0.05, terrain.shape)).astype(np.float32)
    for _ in range(300):
        i, j, r = rng.integers(0, rows), rng.integers(0, cols), int(rng.integers(4, 80))
        dem[max(0, i - r):i + r, max(0, j - r):j + r] = np.nan
    gm.layers["elevation"][...] = dem
    gm.upload(("elevation",))
    return gm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("geotiff_deflate_bench: no CUDA device (nothing is measured without one)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    gm = bench_map()
    rows, cols = gm.getSize()
    ctx = gm.context()
    L = amb.lib()
    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    threads = os.cpu_count()
    pool = ThreadPoolExecutor(threads)
    out = {"card": q, "width": rows, "height": cols, "launches": args.launches, "host_threads": threads,
           "zlib": zlib.ZLIB_RUNTIME_VERSION, "cases": {}}
    tmp = tempfile.mkdtemp()
    for name, fmt in BENCH_LAYERS:
        f = _lib.RASTER_FORMAT[fmt]
        bpp = _lib.RASTER_BPP[f]
        rps = max(1, 8192 // (rows * bpp))
        band = torch.empty(rows * cols * bpp, dtype=torch.uint8, device="cuda:0")
        amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID[name], f, band.data_ptr()), ctx)
        gm.sync()
        host = band.cpu().numpy()
        img = host.view(np.float32).reshape(cols, rows) if fmt == "f32" else \
            host.reshape((cols, rows) + ((3,) if fmt == "bgr8" else ()))
        cap = int(L.amb_deflate_max_size(rows, cols, f, rps))
        p = C.c_void_p()
        amb.check(L.amb_host_alloc(C.byref(p), cap))
        counts = np.zeros((cols + rps - 1) // rps, np.uint32)
        size = C.c_size_t(0)

        def enc():
            amb.check(L.amb_deflate_strips_device(ctx, band.data_ptr(), rows, cols, rows * bpp, f, rps, p, cap,
                                                  C.byref(size), counts.ctypes.data), ctx)

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
        strips = predicted_strips(img, fmt, rps)
        at, exact = 0, True
        for s, n in zip(strips, counts):
            exact = exact and zlib.decompress(ours[at:at + int(n)]) == s
            at += int(n)
        api_ms = 1e3 * best(lambda: gm.to_geotiff(os.path.join(tmp, "a.tif"), name, fmt=fmt), args.repeats)
        raw = sum(len(s) for s in strips)
        case = {"device_ms": dev_ms, "host_api_ms": api_ms, "raw_bytes": raw, "bytes": len(ours),
                "ratio": raw / len(ours), "decodes_exactly": exact}
        for level in (1, 6):
            t0 = time.perf_counter()
            zs = list(pool.map(lambda s: len(zlib.compress(s, level)), strips, chunksize=64))
            case["zlib%d_ms" % level] = 1e3 * (time.perf_counter() - t0)
            case["zlib%d_ratio" % level] = raw / sum(zs)
        case["size_vs_zlib1"] = len(ours) / (raw / case["zlib1_ratio"])
        case["speedup_device_vs_zlib1"] = case["zlib1_ms"] / dev_ms
        out["cases"][name] = case
        L.amb_host_free(p)
        del band
    line = json.dumps(out)
    print("card:", q)
    for name, r in out["cases"].items():
        print("%-17s device %.2f ms  host API %.1f ms  zlib-1 %.0f ms / zlib-6 %.0f ms on %d threads (%.0fx)  ratio %.3f "
              "(zlib-1 %.3f, zlib-6 %.3f)  exact %s" % (name, r["device_ms"], r["host_api_ms"], r["zlib1_ms"],
                                                       r["zlib6_ms"], threads, r["speedup_device_vs_zlib1"],
                                                       r["ratio"], r["zlib1_ratio"], r["zlib6_ratio"],
                                                       r["decodes_exactly"]))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "geotiff_deflate_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
