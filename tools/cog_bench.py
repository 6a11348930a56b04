"""Cloud-Optimized GeoTIFF tiles (amb_cog_tiles_device / GridMap.to_cog, csrc/raster_pyramid.cu + csrc/deflate_encode.cu)
against the host path, on one GPU.

    python tools/cog_bench.py [--launches 20] [--repeats 5] [--tile 512] [--out DIR]

Rasters: the four 10000 x 10000 rasters of tools/geotiff_deflate_bench.py (bench_map()).
Device: amb_cog_tiles_device of the exported band, CUDA events over --launches calls after warm-up, each ending with the
file's tiles in pinned host memory.  Host API: GridMap.to_cog to a file in a temporary directory, best of --repeats, and
its size next to GridMap.to_geotiff's strip file.  Kernel split: one call under torch.profiler in a separate run,
CUDA time summed over the reduce, tile and Deflate kernels.  Status quo, in the same call: to_raster, a numpy
restatement of the pyramid and the tiles' predictor, then zlib level 1 of the same predicted tiles on all of this
host's threads.  Every device file is checked to inflate to the restated tiles.  Prints the card's name and power limit
and one JSON line; writes it to --out/cog_bench.json if given."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, io  # noqa: E402
from geotiff_deflate_bench import BENCH_LAYERS, bench_map, best  # noqa: E402


def reduce(a, fmt):
    """One level of the convention's box filter (include/aerial_mapper_b200.h, amb_cog_tiles_device)."""
    h, w = a.shape[:2]
    h2, w2 = -(-h // 2), -(-w // 2)
    if fmt == "f32":
        p = np.full((2 * h2, 2 * w2), np.nan, np.float64)
        p[:h, :w] = a
        kids = [p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2]]
        s = np.zeros((h2, w2))
        n = np.zeros((h2, w2), np.int64)
        with np.errstate(invalid="ignore", over="ignore"):
            for v in kids:
                ok = ~np.isnan(v)
                s = np.where(ok & (n == 0), v, np.where(ok, s + v, s))
                n += ok
            out = (s / np.maximum(n, 1)).astype(np.float32)
        out[(n == 0) | np.isnan(out)] = np.uint32(0x7FC00000).view(np.float32)
        return out
    p = np.zeros((2 * h2, 2 * w2) + a.shape[2:], np.int64)
    p[:h, :w] = a
    kids = [p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2]]
    if fmt == "mask8":
        return np.maximum.reduce(kids).astype(np.uint8)
    present = np.zeros((2 * h2, 2 * w2), np.int64)
    present[:h, :w] = 1
    n = present[0::2, 0::2] + present[0::2, 1::2] + present[1::2, 0::2] + present[1::2, 1::2]
    n = n[..., None] if a.ndim == 3 else n
    return ((sum(kids) + n // 2) // n).astype(np.uint8)


def predicted_tiles(img, fmt, tile):
    """The pyramid's tiles in file order, predicted (the restatement of tests/test_cog_cpu.py)."""
    levels = [img]
    for _ in io.cog_layout(img.shape[1], img.shape[0], tile)[1:]:
        levels.append(reduce(levels[-1], fmt))
    out = []
    for lv in levels[::-1]:
        h, w = lv.shape[:2]
        th, tw = -(-h // tile), -(-w // tile)
        pad = np.zeros((th * tile, tw * tile) + lv.shape[2:], lv.dtype)
        pad[:h, :w] = lv
        if fmt == "f32":
            be = pad.astype(">f4").view(np.uint8).reshape(th * tile, tw, tile, 4).transpose(0, 1, 3, 2)
            b = np.ascontiguousarray(be).reshape(th * tile, tw, 4 * tile)
            step = 1
        else:
            src = pad[:, :, ::-1] if fmt == "bgr8" else pad
            b = np.ascontiguousarray(src).reshape(th * tile, tw, -1)
            step = 3 if fmt == "bgr8" else 1
        d = b.copy()
        d[:, :, step:] -= b[:, :, :-step]
        d = d.reshape(th, tile, tw, -1).transpose(0, 2, 1, 3)
        out += [np.ascontiguousarray(d[ty, tx]).tobytes() for ty in range(th) for tx in range(tw)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--tile", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("cog_bench: no CUDA device (nothing is measured without one)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    gm = bench_map()
    rows, cols = gm.getSize()
    ctx = gm.context()
    L = amb.lib()
    T = args.tile
    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    threads = os.cpu_count()
    pool = ThreadPoolExecutor(threads)
    out = {"card": q, "width": rows, "height": cols, "tile": T, "launches": args.launches, "host_threads": threads,
           "zlib": zlib.ZLIB_RUNTIME_VERSION, "cases": {}}
    tmp = tempfile.mkdtemp()
    for name, fmt in BENCH_LAYERS:
        f = _lib.RASTER_FORMAT[fmt]
        bpp = _lib.RASTER_BPP[f]
        band = torch.empty(rows * cols * bpp, dtype=torch.uint8, device="cuda:0")
        amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID[name], f, band.data_ptr()), ctx)
        gm.sync()
        cap = int(L.amb_cog_max_size(rows, cols, f, T))
        p = C.c_void_p()
        amb.check(L.amb_host_alloc(C.byref(p), cap))
        n_tiles = sum(-(-w // T) * -(-h // T) for w, h in io.cog_layout(rows, cols, T))
        counts = np.zeros(n_tiles, np.uint32)
        size = C.c_size_t(0)

        def enc():
            amb.check(L.amb_cog_tiles_device(ctx, band.data_ptr(), rows, cols, rows * bpp, f, T, p, cap, C.byref(size),
                                             counts.ctypes.data), ctx)

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
        cog_path, strip_path = os.path.join(tmp, "a_cog.tif"), os.path.join(tmp, "a_strips.tif")
        api_ms = 1e3 * best(lambda: gm.to_cog(cog_path, name, fmt=fmt, tile_size=T), args.repeats)
        gm.to_geotiff(strip_path, name, fmt=fmt)
        # status quo: the raster to the host, the pyramid and the predictor in numpy, zlib level 1 on every thread
        t0 = time.perf_counter()
        img = gm.to_raster(name, fmt)
        t1 = time.perf_counter()
        tiles = predicted_tiles(img, fmt, T)
        t2 = time.perf_counter()
        zs = list(pool.map(lambda s: len(zlib.compress(s, 1)), tiles, chunksize=8))
        t3 = time.perf_counter()
        at, exact = 0, len(tiles) == len(counts)
        for s, n in zip(tiles, counts):
            exact = exact and zlib.decompress(ours[at:at + int(n)]) == s
            at += int(n)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc()
            torch.cuda.synchronize()
        split = {"reduce": 0.0, "tile": 0.0, "deflate": 0.0}
        for e in prof.key_averages():
            key = "reduce" if "pyramid_reduce" in e.key else "tile" if "pyramid_tile" in e.key else \
                "deflate" if "deflate_" in e.key else None
            if key:
                split[key] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        raw = rows * cols * bpp
        case = {"device_ms": dev_ms, "host_api_ms": api_ms, "kernel_ms": split, "raw_bytes": raw, "tiles": len(counts),
                "cog_bytes": os.path.getsize(cog_path), "strip_file_bytes": os.path.getsize(strip_path),
                "decodes_exactly": exact, "status_quo_ms": {"to_raster": 1e3 * (t1 - t0), "numpy_pyramid": 1e3 * (t2 - t1),
                                                            "zlib1": 1e3 * (t3 - t2), "total": 1e3 * (t3 - t0)},
                "zlib1_bytes": sum(zs)}
        case["speedup_api_vs_status_quo"] = case["status_quo_ms"]["total"] / api_ms
        out["cases"][name] = case
        L.amb_host_free(p)
        del band
    line = json.dumps(out)
    print("card:", q)
    for name, r in out["cases"].items():
        print("%-17s device %.1f ms (reduce %.2f, tile %.2f, deflate %.1f)  to_cog %.0f ms  status quo %.0f ms  COG %.1f MB "
              "vs strips %.1f MB  exact %s" % (name, r["device_ms"], r["kernel_ms"]["reduce"], r["kernel_ms"]["tile"],
                                               r["kernel_ms"]["deflate"], r["host_api_ms"], r["status_quo_ms"]["total"],
                                               r["cog_bytes"] / 1e6, r["strip_file_bytes"] / 1e6, r["decodes_exactly"]))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cog_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
