"""JPEG-compressed Cloud-Optimized GeoTIFF tiles with a 1-bit mask (amb_cog_jpeg_tiles_device, amb_cog_mask_tiles_device
/ GridMap.to_cog(compress="jpeg", mask=...), csrc/raster_pyramid.cu + csrc/jpeg_encode.cu) against the host path, on one
GPU.

    python tools/cog_jpeg_bench.py [--launches 20] [--repeats 3] [--tile 512] [--out DIR]

Rasters: the 10000 x 10000 rasters of tools/cog_bench.py (bench_map()): ortho as gray8, colored_ortho as bgr8 at 4:2:0,
each at quality 75 and 90, and observation_index as the mask.  Device: the entry point on the exported band, CUDA events
over --launches calls after warm-up, each ending with the tiles in pinned host memory.  Kernel split: one call under
torch.profiler in a separate run, CUDA time summed over the reduce, tile, mask pack, JPEG and Deflate kernels.  Host
API: GridMap.to_cog to a file in a temporary directory, best of --repeats, with the mask and without, and the file sizes
next to the Deflate COG of the same raster.  Status quo, in the same call: to_raster, the numpy pyramid and tiles, then
cv2.imencode of every tile on all of this host's threads.  Every device tile is checked against cv2's entropy-coded
bytes for that tile.  Prints the card's name and power limit and one JSON line; writes it to --out/cog_jpeg_bench.json
if given."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, io  # noqa: E402
from cog_bench import reduce  # noqa: E402
from geotiff_deflate_bench import bench_map, best  # noqa: E402

CASES = (("ortho", "gray8", "420"), ("colored_ortho", "bgr8", "420"))
QUALITIES = (75, 90)
KERNELS = (("reduce", "pyramid_reduce"), ("tile", "pyramid_tile"), ("mask_pack", "mask_pack"), ("jpeg", "jpeg_"),
           ("deflate", "deflate_"))


def pyramid_tiles(img, fmt, tile):
    """The pyramid's T x T tiles in file order, zero outside each level (the restatement of tests/test_cog_jpeg_cpu.py)."""
    levels = [img]
    for _ in io.cog_layout(img.shape[1], img.shape[0], tile)[1:]:
        levels.append(reduce(levels[-1], fmt))
    out = []
    for lv in levels[::-1]:
        h, w = lv.shape[:2]
        th, tw = -(-h // tile), -(-w // tile)
        pad = np.zeros((th * tile, tw * tile) + lv.shape[2:], np.uint8)
        pad[:h, :w] = lv
        out += [pad[ty * tile:(ty + 1) * tile, tx * tile:(tx + 1) * tile] for ty in range(th) for tx in range(tw)]
    return out


def cv2_data(jpg):
    """The entropy-coded bytes of a whole JPEG file: after SOS, before EOI."""
    at = 2
    while jpg[at + 1] != 0xDA:
        at += 2 + int.from_bytes(jpg[at + 2:at + 4], "big")
    return jpg[at + 2 + int.from_bytes(jpg[at + 2:at + 4], "big"):-2]


def kernel_split(prof):
    split = {k: 0.0 for k, _ in KERNELS}
    for e in prof.key_averages():
        for k, pat in KERNELS:
            if pat in e.key:
                split[k] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
                break
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--tile", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("cog_jpeg_bench: no CUDA device (nothing is measured without one)")
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
    n_tiles = sum(-(-w // T) * -(-h // T) for w, h in io.cog_layout(rows, cols, T))
    out = {"card": q, "width": rows, "height": cols, "tile": T, "tiles": n_tiles, "launches": args.launches,
           "host_threads": threads, "opencv": cv2.__version__, "cases": {}}
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "a.tif")

    def timed(enc):
        for _ in range(3):
            enc()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.launches):
            enc()
        e1.record(stream)
        e1.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc()
            torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.launches, kernel_split(prof)

    counts = np.zeros(n_tiles, np.uint32)
    size = C.c_size_t(0)
    # the mask of observation_index
    mband = torch.empty(rows * cols, dtype=torch.uint8, device="cuda:0")
    amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID["observation_index"], _lib.RASTER_MASK8, mband.data_ptr()),
              ctx)
    gm.sync()
    mcap = int(L.amb_cog_mask_max_size(rows, cols, T))
    mp = C.c_void_p()
    amb.check(L.amb_host_alloc(C.byref(mp), mcap))

    def enc_mask():
        amb.check(L.amb_cog_mask_tiles_device(ctx, mband.data_ptr(), rows, cols, rows, T, mp, mcap, C.byref(size),
                                              counts.ctypes.data), ctx)

    dev_ms, split = timed(enc_mask)
    out["mask"] = {"device_ms": dev_ms, "kernel_ms": split, "bytes": size.value,
                   "valid_share": float(mband.ne(0).float().mean().item())}
    L.amb_host_free(mp)
    del mband
    for name, fmt, sampling in CASES:
        f = _lib.RASTER_FORMAT[fmt]
        bpp = _lib.RASTER_BPP[f]
        s = api.JPEG_SAMPLING[sampling]
        band = torch.empty(rows * cols * bpp, dtype=torch.uint8, device="cuda:0")
        amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID[name], f, band.data_ptr()), ctx)
        gm.sync()
        gm.to_cog(path, name, fmt=fmt, tile_size=T)
        deflate_bytes = os.path.getsize(path)
        t0 = time.perf_counter()
        img = gm.to_raster(name, fmt)
        t1 = time.perf_counter()
        tiles = pyramid_tiles(img, fmt, T)
        t2 = time.perf_counter()
        for quality in QUALITIES:
            cap = int(L.amb_cog_jpeg_max_size(rows, cols, f, T, quality, s))
            p = C.c_void_p()
            amb.check(L.amb_host_alloc(C.byref(p), cap))

            def enc():
                amb.check(L.amb_cog_jpeg_tiles_device(ctx, band.data_ptr(), rows, cols, rows * bpp, f, T, quality, s, p,
                                                      cap, C.byref(size), counts.ctypes.data), ctx)

            dev_ms, split = timed(enc)
            ours = bytes((C.c_uint8 * size.value).from_address(p.value))
            lens = counts.copy()
            L.amb_host_free(p)
            params = [cv2.IMWRITE_JPEG_QUALITY, quality]
            if fmt == "bgr8":
                params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
            t3 = time.perf_counter()
            files = list(pool.map(lambda t: cv2.imencode(".jpg", t, params)[1].tobytes(), tiles, chunksize=4))
            t4 = time.perf_counter()
            at, exact = 0, len(files) == len(lens)
            for jpg, n in zip(files, lens):
                tile = ours[at:at + int(n)]
                exact = exact and tile[-2 - len(cv2_data(jpg)):-2] == cv2_data(jpg)
                at += int(n)
            api_ms = 1e3 * best(lambda: gm.to_cog(path, name, fmt=fmt, tile_size=T, compress="jpeg", quality=quality,
                                                  sampling=sampling), args.repeats)
            jpeg_bytes = os.path.getsize(path)
            api_mask_ms = 1e3 * best(lambda: gm.to_cog(path, name, fmt=fmt, tile_size=T, compress="jpeg",
                                                       quality=quality, sampling=sampling, mask="observation_index"),
                                     args.repeats)
            case = {"device_ms": dev_ms, "kernel_ms": split, "tiles_bytes": size.value, "to_cog_ms": api_ms,
                    "to_cog_mask_ms": api_mask_ms, "cog_bytes": jpeg_bytes, "cog_mask_bytes": os.path.getsize(path),
                    "deflate_cog_bytes": deflate_bytes, "matches_cv2": exact,
                    "status_quo_ms": {"to_raster": 1e3 * (t1 - t0), "numpy_pyramid": 1e3 * (t2 - t1),
                                      "cv2_imencode": 1e3 * (t4 - t3), "total": 1e3 * (t2 - t0 + t4 - t3)}}
            case["speedup_api_vs_status_quo"] = case["status_quo_ms"]["total"] / api_ms
            out["cases"]["%s_q%d" % (name, quality)] = case
        del band, img, tiles
    line = json.dumps(out)
    print("card:", q)
    m = out["mask"]
    print("mask              device %.1f ms  %s  %.2f MB" % (m["device_ms"], m["kernel_ms"], m["bytes"] / 1e6))
    for key, r in out["cases"].items():
        print("%-17s device %.1f ms %s  to_cog %.0f ms (+mask %.0f)  status quo %.0f ms  COG %.1f MB (+mask %.1f) vs "
              "Deflate %.1f MB  matches cv2 %s" % (key, r["device_ms"], {k: round(v, 2) for k, v in r["kernel_ms"].items()},
                                                   r["to_cog_ms"], r["to_cog_mask_ms"], r["status_quo_ms"]["total"],
                                                   r["cog_bytes"] / 1e6, r["cog_mask_bytes"] / 1e6,
                                                   r["deflate_cog_bytes"] / 1e6, r["matches_cv2"]))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cog_jpeg_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
