"""Importing a Deflate GeoTIFF DEM into a map layer (GridMap.from_geotiff, csrc/deflate_decode.cu) against the host
paths, on one GPU.

    python tools/geotiff_inflate_bench.py [--repeats 3] [--out DIR] [--skip-full-read]

Cases (DEMs written by this script, zlib level 6, into a temporary directory):
  strips16   10000 x 10000 float32, predictor 3, 16-row strips, map 2500 m at 0.25 m over all of it
  tiles512   the same DEM as 512 x 512 tiles
  one_strip  the same DEM as one strip (one zlib stream: one warp inflates it)
  int16      10000 x 10000 int16, predictor 2, 16-row strips
  window     40000 x 40000 float32 at 0.5 m in 512 tiles (16 distinct tiles repeated), a 2500 m map over 1/64 of it
Per case, host clock around calls that end synchronised, best of --repeats, the file's bytes in pageable memory:
  read_geotiff   io.read_geotiff (one host thread: zlib, numpy predictor, assembly) + GridMap.from_raster
  host_threads   zlib on every host thread (zlib releases the GIL) + the numpy predictor per chunk + from_raster
  host_window    the same, but only the chunks the map's window meets (its rows and columns from
                 amb_raster_import_tables), into a window band passed to from_raster with its shifted geotransform
  device         GridMap.from_geotiff: the H2D copy of the window's chunks, inflate, unpredict, resample
and the device's own time in one more call of its own under torch.profiler (CUPTI sees every kernel and copy of the
process): device_kernels_ms, the sum of the kernels' durations, and device_h2d_ms, of the host-to-device copies.
Every path's layer is compared bit for bit.  Prints the card's name and power limit and one JSON line."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import io  # noqa: E402
from test_geotiff_inflate_cpu import make_tiff, predict  # noqa: E402


def dem(h, w, dtype, seed=0):
    rng = np.random.default_rng(seed)
    y = np.arange(h, dtype=np.float32)[:, None]
    x = np.arange(w, dtype=np.float32)[None, :]
    a = 400 + 30 * np.sin(x / 700) * np.cos(y / 900) + rng.normal(0, 0.05, (h, w)).astype(np.float32)
    return a.astype(dtype) if dtype == np.float32 else (a * 10).astype(dtype)


def compress_all(a, pred, chunk, pool):
    """make_tiff with its chunks compressed on every host thread."""
    cache = {}

    def enc(raw, k):
        return cache[k]
    t = np.asarray(a)[:, :, None]
    H, W = a.shape
    if chunk[0] == "strips":
        parts = [t[r:r + chunk[1]] for r in range(0, H, chunk[1])]
    else:
        parts = []
        for r in range(0, H, chunk[2]):
            for c in range(0, W, chunk[1]):
                p = np.zeros((chunk[2], chunk[1], 1), a.dtype)
                s = t[r:r + chunk[2], c:c + chunk[1]]
                p[:s.shape[0], :s.shape[1]] = s
                parts.append(p)
    for k, z in enumerate(pool.map(lambda p: zlib.compress(predict(p, pred), 6), parts)):
        cache[k] = z
    return enc


def window_file(path, n=40000, tile=512, gt=None):
    """A 40000 x 40000 float32 predictor-3 tiled GeoTIFF whose tiles repeat 16 distinct compressed tiles."""
    base = dem(4 * tile, 4 * tile, np.float32, seed=7)
    tiles = [zlib.compress(predict(base[r:r + tile, c:c + tile, None], 3), 6)
             for r in range(0, 4 * tile, tile) for c in range(0, 4 * tile, tile)]
    across = -(-n // tile)
    counts = [len(tiles[(k // across % 4) * 4 + k % across % 4]) for k in range(across * across)]
    layout = [(322, io._LONG, [tile]), (323, io._LONG, [tile]), (324, io._LONG, [0] * len(counts)),
              (325, io._LONG, counts)]
    tags = io._image_tags(n, n, 1, 32, 3, layout, (gt, 32632, None))
    data_at = (8 + io._ifd_size(tags) + 15) & ~15
    offs = (np.concatenate([[0], np.cumsum(counts)[:-1]]) + data_at).tolist()
    tags = io._set_tag(tags, 324, io._LONG, offs)
    head = b"II*\0" + (8).to_bytes(4, "little") + io._ifd(tags, 8)
    with open(path, "wb") as f:
        f.write(head + b"\0" * (data_at - len(head)))
        for k in range(len(counts)):
            f.write(tiles[(k // across % 4) * 4 + k % across % 4])


def host_threads(data, pool):
    t = io.tiff_layout(data)
    out = np.empty((t.height, t.width), t.dtype)

    def one(args):
        (r0, c0, rows, cols), at, n = args
        a = io._undo_predictor(zlib.decompress(data[at:at + n]), t.predictor, t.dtype, rows, cols, t.spp)
        out[r0:r0 + rows, c0:c0 + cols] = a[:t.height - r0, :t.width - c0, 0]
    list(pool.map(one, zip(t.grid, t.offsets, t.counts)))
    return out, t.georeferencing()


def window_of(gm, t, gt):
    """Rows [r0, r1) and columns [c0, c1) of the raster the map's bilinear import reads."""
    g = gm.geometry
    sc, fx = np.empty(g.rows, np.int32), np.empty(g.rows)
    sr, fy = np.empty(g.cols, np.int32), np.empty(g.cols)
    assert amb.lib().amb_raster_import_tables(C.byref(g), 0, g.cols, t.width, t.height, (C.c_double * 6)(*gt), 1,
                                              sc.ctypes.data, fx.ctypes.data, sr.ctypes.data, fy.ctypes.data) == 0
    c, r = sc >= 0, sr >= 0
    return (int(sr[r].min()), int((sr + (fy != 0))[r].max()) + 1, int(sc[c].min()), int((sc + (fx != 0))[c].max()) + 1)


def host_window(data, pool, win):
    """host_threads over the chunks that meet the window only: (window band, its geotransform, no-data)."""
    t = io.tiff_layout(data)
    r0, r1, c0, c1 = win
    out = np.empty((r1 - r0, c1 - c0), t.dtype)

    def one(args):
        (cr, cc, rows, cols), at, n = args
        if cr >= r1 or cr + rows <= r0 or cc >= c1 or cc + cols <= c0:
            return
        a = io._undo_predictor(zlib.decompress(data[at:at + n]), t.predictor, t.dtype, rows, cols, t.spp)[:, :, 0]
        ra, rb, ca, cb = max(cr, r0), min(cr + rows, r1), max(cc, c0), min(cc + cols, c1)
        out[ra - r0:rb - r0, ca - c0:cb - c0] = a[ra - cr:rb - cr, ca - cc:cb - cc]
    list(pool.map(one, zip(t.grid, t.offsets, t.counts)))
    gt, _, nd = t.georeferencing()
    return out, (gt[0] + c0 * gt[1], gt[1], 0.0, gt[3] + r0 * gt[5], 0.0, gt[5]), nd


def device_split(gm, data):
    """(kernel ms, H2D copy ms) of one from_geotiff call, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gm.from_geotiff("elevation", data)
    kern = h2d = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if "HtoD" in e.name:
            h2d += us
        elif "Memcpy" not in e.name and "Memset" not in e.name:
            kern += us
    return round(kern / 1e3, 3), round(h2d / 1e3, 3)


def fresh(side_m, res, center):
    gm = amb.AerialGridMap(amb.GridMapSettings(center[0], center[1], side_m, side_m, res)).getMutable()
    gm.to_device(0, names=("elevation",))
    return gm


def best(fn, repeats):
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-full-read", action="store_true", help="no read_geotiff of the 40000 x 40000 file")
    ap.add_argument("--cases", default="strips16,tiles512,one_strip,int16,window")
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    pool = ThreadPoolExecutor(os.cpu_count())
    tmp = tempfile.mkdtemp()
    center = (464500.0, 5272500.0)
    results = {"host_threads": os.cpu_count()}
    cases = []
    want = args.cases.split(",")
    gt = (center[0] - 1250.0, 0.25, 0.0, center[1] + 1250.0, 0.0, -0.25)
    for name, dtype, pred, chunk in (("strips16", np.float32, 3, ("strips", 16)),
                                     ("tiles512", np.float32, 3, ("tiles", 512, 512)),
                                     ("one_strip", np.float32, 3, ("strips", 10000)),
                                     ("int16", np.int16, 2, ("strips", 16))):
        if name not in want:
            continue
        a = dem(10000, 10000, dtype)
        p = os.path.join(tmp, name + ".tif")
        with open(p, "wb") as f:
            f.write(make_tiff(a, pred, chunk, encode=compress_all(a, pred, chunk, pool), gt=gt))
        cases.append((name, p, 2500.0, 0.25))
        del a
    if "window" in want:
        p = os.path.join(tmp, "window.tif")
        window_file(p, gt=(center[0] - 1250.0, 0.5, 0.0, center[1] + 1250.0, 0.0, -0.5))
        cases.append(("window", p, 2500.0, 0.5))
    for name, path, side, res in cases:
        data = open(path, "rb").read()
        r = {"file_mb": round(len(data) / 1e6, 1)}
        gm_dev = fresh(side, res, center)
        gm_dev.from_geotiff("elevation", data)                    # warm-up: scratch and modules
        r["device_s"] = best(lambda: gm_dev.from_geotiff("elevation", data), args.repeats)
        gm_dev.download(("elevation",))
        dev = np.array(gm_dev["elevation"], copy=True)
        gm_h = fresh(side, res, center)

        def threads():
            a, (g, _, nd) = host_threads(data, pool)
            gm_h.from_raster("elevation", a.astype(np.float32), g, nodata=nd)
        r["host_threads_s"] = best(threads, args.repeats)
        gm_h.download(("elevation",))
        assert np.array_equal(gm_h["elevation"].view(np.uint32), dev.view(np.uint32)), name
        t = io.tiff_layout(data)
        win = window_of(gm_h, t, t.georeferencing()[0])
        r["window_rows_cols"] = win
        gm_w = fresh(side, res, center)

        def window():
            a, g, nd = host_window(data, pool, win)
            gm_w.from_raster("elevation", a.astype(np.float32), g, nodata=nd)
        r["host_window_s"] = best(window, args.repeats)
        gm_w.download(("elevation",))
        assert np.array_equal(gm_w["elevation"].view(np.uint32), dev.view(np.uint32)), name
        try:
            r["device_kernels_ms"], r["device_h2d_ms"] = device_split(gm_dev, data)
        except Exception as e:  # the profiler is optional instrumentation: report, do not lose the case
            r["device_split_error"] = repr(e)
        if not (name == "window" and args.skip_full_read):
            gm_r = fresh(side, res, center)

            def single():
                a, g, _, nd = io.read_geotiff(path)
                gm_r.from_raster("elevation", a.astype(np.float32), g, nodata=nd)
            r["read_geotiff_s"] = best(single, 1 if name == "window" else args.repeats)
            gm_r.download(("elevation",))
            assert np.array_equal(gm_r["elevation"].view(np.uint32), dev.view(np.uint32)), name
        r["equal"] = True
        results[name] = r
        print(name, r, flush=True)
    line = json.dumps(results)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "geotiff_inflate_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
