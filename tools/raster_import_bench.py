"""Raster import (amb_import_raster*, csrc/raster_import.cu) against what a user does without it, on one GPU.

    python tools/raster_import_bench.py [--rows 10000] [--cols 10000] [--res 0.25] [--launches 50] [--out DIR]

Device: CUDA events over --launches launches after warm-up of the import from a device band: the map's own F32 raster
(aligned) with nearest and with bilinear resampling, and a 1 m DEM resampled bilinearly; against a device-to-device copy
of the same float32 layer in the same run.  Rate = (bytes of the band the import reads + 4 B written per cell) / time;
the copy's rate is 2 * 4 bytes per cell.
Host: amb_import_raster from page-locked and from pageable memory, and the status quo for the 1 m DEM: scipy's
map_coordinates(order=1) at the cell centres, the flip into the column-major layer, amb_upload_layer.  Host clock around
calls that end synchronised; best of --repeats.
Prints the card's name and power limit and one JSON line; writes it to --out/raster_import_bench.json if given."""
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
from aerial_mapper_b200 import _lib, synth  # noqa: E402

UTM = (464500.0, 5272500.0)


def best(fn, repeats):
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def status_quo(gm, band, gt):
    """scipy bilinear interpolation at the cell centres (half-pixel convention, edges clamped), then the flip into the
    column-major layer and its upload: the numpy a user would write."""
    from scipy.ndimage import map_coordinates
    g = gm.geometry
    qx, qy = synth.grid_positions(g.rows, g.cols, g.resolution, g.pos_x, g.pos_y)
    u = (qx - gt[0]) / gt[1] - 0.5
    v = (qy - gt[3]) / gt[5] - 0.5
    # cell (i, j) reads (v_j, u_i): the layer is column-major, so the [cols, rows] image of the cells is its transpose
    img = map_coordinates(band, [np.repeat(v, g.rows), np.tile(u, g.cols)], order=1, mode="nearest")
    gm["elevation"] = img.reshape(g.cols, g.rows).T
    gm.upload(("elevation",))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--cols", type=int, default=10000)
    ap.add_argument("--res", type=float, default=0.25)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("raster_import_bench: no CUDA device (nothing is measured without one)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    rows, cols, res = args.rows, args.cols, args.res
    cells = rows * cols
    gm = amb.AerialGridMap(amb.GridMapSettings(UTM[0], UTM[1], rows * res, cols * res, res),
                           layer_names=("elevation",)).getMutable()
    gm["elevation"] = synth.analytic_elevation(rows, cols, res, *UTM)
    gm.to_device(0, names=("elevation",))
    ctx = gm.context()
    L = amb.lib()
    E = _lib.LAYER_ID["elevation"]
    aligned = gm.to_raster("elevation", "f32")                       # [cols, rows]: the map's own grid
    gt_aligned = gm.geotransform()
    # a 1 m DEM over the map plus a margin, its origin a third of a pixel off the map's grid
    dem_res = 1.0
    west, north = gt_aligned[0] - 2.0 - dem_res / 3, gt_aligned[3] + 2.0 + dem_res / 3
    dw, dh = int(rows * res / dem_res) + 5, int(cols * res / dem_res) + 5
    dx = west + (np.arange(dw) + 0.5) * dem_res
    dy = north - (np.arange(dh) + 0.5) * dem_res
    dem = synth.terrain(dx[None, :], dy[:, None]).astype(np.float32)
    gt_dem = (west, dem_res, 0.0, north, 0.0, -dem_res)

    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    d_aligned = torch.from_numpy(aligned).cuda()
    d_dem = torch.from_numpy(dem).cuda()
    copy_src = torch.empty(cells * 4, dtype=torch.uint8, device="cuda:0")
    copy_dst = torch.empty(cells * 4, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    out = {"card": q, "rows": rows, "cols": cols, "res": res, "launches": args.launches, "device": {}, "host": {}}

    def timed(fn):
        for _ in range(5):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.launches):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.launches / 1e3

    def dev_import(t, band, gt, method):
        h, w = band.shape
        gtc = (C.c_double * 6)(*gt)
        return lambda: amb.check(L.amb_import_raster_device(ctx, E, t.data_ptr(), w, h, w * 4, gtc, 0, 0.0,
                                                            _lib.RESAMPLE[method]), ctx)

    cases = {"aligned_nearest": (d_aligned, aligned, gt_aligned, "nearest", 4.0 * cells),
             "aligned_bilinear": (d_aligned, aligned, gt_aligned, "bilinear", 4.0 * cells),
             "dem_1m_bilinear": (d_dem, dem, gt_dem, "bilinear", float(dem.nbytes))}
    for rnd in range(2):                                               # the copy and the imports, alternated twice
        with torch.cuda.stream(stream):
            t = timed(lambda: copy_dst.copy_(copy_src))
        out["device"].setdefault("d2d_copy", []).append({"ms": t * 1e3, "GBps": 8.0 * cells / t / 1e9})
        for name, (t_band, band, gt, method, read_bytes) in cases.items():
            t = timed(dev_import(t_band, band, gt, method))
            out["device"].setdefault(name, []).append({"ms": t * 1e3, "GBps": (read_bytes + 4.0 * cells) / t / 1e9})
    copy_rate = max(r["GBps"] for r in out["device"]["d2d_copy"])
    for name in cases:
        out["device"][name + "_vs_copy"] = max(r["GBps"] for r in out["device"][name]) / copy_rate

    # the aligned import is the layer itself, bit for bit
    gm.sync()
    want = gm["elevation"].copy(order="F")
    dev_import(d_aligned, aligned, gt_aligned, "bilinear")()
    gm.sync()
    gm.download(("elevation",))
    out["aligned_identical"] = bool(np.array_equal(gm["elevation"].view(np.uint32), want.view(np.uint32)))

    # host bands: pinned and pageable, and the status quo for the DEM
    for name, band, gt in (("aligned_bilinear", aligned, gt_aligned), ("dem_1m_bilinear", dem, gt_dem)):
        p = C.c_void_p()
        amb.check(L.amb_host_alloc(C.byref(p), band.nbytes))
        pinned = np.frombuffer((C.c_uint8 * band.nbytes).from_address(p.value), np.float32).reshape(band.shape)
        pinned[...] = band
        res_h = {}
        layers = {}
        for label, b in (("pinned", pinned), ("pageable", band)):
            gm.from_raster("elevation", b, gt)
            res_h[label + "_ms"] = 1e3 * best(lambda: gm.from_raster("elevation", b, gt), args.repeats)
            gm.download(("elevation",))
            layers[label] = gm["elevation"].copy(order="F")
        res_h["pinned_equals_pageable"] = bool(np.array_equal(layers["pinned"].view(np.uint32),
                                                              layers["pageable"].view(np.uint32)))
        if name == "dem_1m_bilinear":
            res_h["status_quo_ms"] = 1e3 * best(lambda: status_quo(gm, band, gt), max(2, args.repeats // 2))
            sq = gm["elevation"].copy(order="F")
            ulps = np.abs(sq.view(np.int32).astype(np.int64) - layers["pinned"].view(np.int32).astype(np.int64))
            res_h["status_quo_max_ulps"] = int(ulps.max())
        out["host"][name] = res_h
        L.amb_host_free(p)
    gm.sync()
    line = json.dumps(out)
    print("card:", q)
    print("d2d copy %.0f GB/s" % copy_rate)
    for name in cases:
        d = out["device"][name]
        print("%-17s device %.3f ms (%.0f GB/s, %.0f%% of the copy)" % (name, min(r["ms"] for r in d),
                                                                       max(r["GBps"] for r in d),
                                                                       100 * out["device"][name + "_vs_copy"]))
    for name, h in out["host"].items():
        print("%-17s host %s" % (name, h))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raster_import_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
