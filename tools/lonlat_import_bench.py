"""Importing a longitude/latitude DEM into a UTM map (GridMap.from_lonlat_raster / from_geotiff(map_epsg=...),
amb_import_*_lonlat, csrc/raster_import.cu) against the projected import and the host status quo, on one GPU.

    python tools/lonlat_import_bench.py [--launches 50] [--repeats 3] [--host-cols 1000] [--out DIR]

Setup: a 10000 x 10000 map at 0.25 m around the reference's Rafz origin in UTM 32N, and a synthetic 3601 x 3601
one-arc-second float32 tile (8-9 E, 47-48 N) covering it.
  per_call    amb_import_raster_lonlat_device of the tile in device memory, CUDA events over --launches back-to-back
              calls after warm-up (host preparation included where it is longer than the kernels); beside it, as the
              yardstick, amb_import_raster_device of a 1 m UTM band over the same map
  kernels     the same calls' kernel time alone, summed from torch.profiler over 10 calls of each, in a run of its own
  end_to_end  from_geotiff(map_epsg=32632) of the tile as a Deflate GeoTIFF in 512 x 512 tiles with predictor 3, host
              clock around a synchronised call, best of --repeats (copy of the window's tiles, inflate, kernel)
  host        the status quo without this feature: the inverse projection restated in numpy (float64, the same series)
              plus scipy.ndimage.map_coordinates (order 1) on the host, timed on --host-cols map columns and scaled to
              the whole map
Every path's layer is compared: the device band and the file give the same bits, and the host path agrees within
2e-3 m (map_coordinates' bilinear rule at the tile's edges and the float32 rounding differ).  Prints the card's name and
power limit and one JSON line."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, synth  # noqa: E402
from test_lonlat_import_cpu import lonlat_tiff  # noqa: E402

RAFZ = (464980.0, 5272260.0)
ARCSEC = 1.0 / 3600.0


def tile():
    n = 3601
    lon = 8.0 + (np.arange(n) + 0.5) * ARCSEC
    lat = 48.0 - (np.arange(n) + 0.5) * ARCSEC
    a = 450.0 + 120.0 * np.sin(lon[None, :] * 300.0) * np.cos(lat[:, None] * 210.0) + \
        15.0 * np.sin(lon[None, :] * 4100.0 + lat[:, None] * 2900.0)
    return a.astype(np.float32), (8.0, ARCSEC, 0.0, 48.0, 0.0, -ARCSEC)


def host_import(x, y, band, gt):
    """The status quo: the inverse series in numpy, then map_coordinates (order 1) at the pixel coordinates."""
    from scipy.ndimage import map_coordinates
    f = 1 / 298.257223563
    n = f / (2 - f)
    e2 = f * (2 - f)
    e, e2m = np.sqrt(e2), 1 - e2
    k0A = 0.9996 * 6378137 / (1 + n) * (1 + n ** 2 / 4 + n ** 4 / 64 + n ** 6 / 256)
    c = [[1 / 2, -2 / 3, 37 / 96, -1 / 360, -81 / 512, 96199 / 604800],
         [0, 1 / 48, 1 / 15, -437 / 1440, 46 / 105, -1118711 / 3870720],
         [0, 0, 17 / 480, -37 / 840, -209 / 4480, 5569 / 90720],
         [0, 0, 0, 4397 / 161280, -11 / 504, -830251 / 7257600],
         [0, 0, 0, 0, 4583 / 161280, -108847 / 3991680],
         [0, 0, 0, 0, 0, 20648693 / 638668800]]
    beta = [sum(ck * n ** (m + 1) for m, ck in enumerate(row)) for row in c]
    xi, eta = y / k0A, (x - 500000.0) / k0A
    xip, etap = xi.copy(), eta.copy()
    for k, b in enumerate(beta, 1):
        xip -= b * np.sin(2 * k * xi) * np.cosh(2 * k * eta)
        etap -= b * np.cos(2 * k * xi) * np.sinh(2 * k * eta)
    s, co, sh = np.sin(xip), np.cos(xip), np.sinh(etap)
    taup = s / np.sqrt(sh * sh + co * co)
    tau = taup / e2m
    for _ in range(2):
        tau1 = np.sqrt(1 + tau * tau)
        sig = np.sinh(e * np.arctanh(e * tau / tau1))
        taupa = np.sqrt(1 + sig * sig) * tau - sig * tau1
        tau += (taup - taupa) * (1 + e2m * tau * tau) / (e2m * tau1 * np.sqrt(1 + taupa * taupa))
    lat = np.degrees(np.arctan(tau))
    lon = 9.0 + np.degrees(np.arctan2(sh, co))
    u = (lon - gt[0]) / gt[1] - 0.5
    v = (lat - gt[3]) / gt[5] - 0.5
    return map_coordinates(band, [v.ravel(), u.ravel()], order=1, mode="nearest").reshape(x.shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-cols", type=int, default=1000)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("lonlat_import_bench: no CUDA device (nothing is measured without one)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    rows = cols = args.rows
    res = 0.25
    L = amb.lib()
    E = _lib.LAYER_ID["elevation"]

    def fresh():
        gm = amb.AerialGridMap(amb.GridMapSettings(RAFZ[0], RAFZ[1], rows * res, cols * res, res),
                               layer_names=("elevation",)).getMutable()
        gm.to_device(0, names=("elevation",))
        return gm

    band, gt = tile()
    gm = fresh()
    ctx = gm.context()
    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    d_band = torch.from_numpy(band).cuda()
    # the yardstick: a 1 m UTM band over the map, imported by the projected path
    g0 = gm.geotransform()
    dw = dh = int(rows * res) + 8
    dx = g0[0] - 4.0 + (np.arange(dw) + 0.5)
    dy = g0[3] + 4.0 - (np.arange(dh) + 0.5)
    utm = synth.terrain(dx[None, :], dy[:, None]).astype(np.float32)
    gt_utm = (g0[0] - 4.0, 1.0, 0.0, g0[3] + 4.0, 0.0, -1.0)
    d_utm = torch.from_numpy(utm).cuda()
    torch.cuda.synchronize()
    gtc, gtu = (C.c_double * 6)(*gt), (C.c_double * 6)(*gt_utm)
    calls = {
        "lonlat_bilinear": lambda: L.amb_import_raster_lonlat_device(ctx, E, d_band.data_ptr(), 3601, 3601, 4 * 3601,
                                                                    gtc, 0, 0.0, 1, 32632),
        "lonlat_nearest": lambda: L.amb_import_raster_lonlat_device(ctx, E, d_band.data_ptr(), 3601, 3601, 4 * 3601,
                                                                   gtc, 0, 0.0, 0, 32632),
        "projected_bilinear": lambda: L.amb_import_raster_device(ctx, E, d_utm.data_ptr(), dw, dh, 4 * dw, gtu, 0, 0.0,
                                                                 1),
    }

    def timed(fn):
        for _ in range(5):
            amb.check(fn(), ctx)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.launches):
            amb.check(fn(), ctx)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.launches

    out = {"card": card, "rows": rows, "cols": cols, "res": res, "launches": args.launches, "per_call_ms": {},
           "kernels_ms": {}}
    for rnd in range(2):        # alternated twice
        for name, fn in calls.items():
            out["per_call_ms"].setdefault(name, []).append(timed(fn))
    # the device's own time per call, in a run of its own under torch.profiler: the sum of the call's kernels (for the
    # longitude/latitude calls the table prologue and the import kernel), so host preparation is not in it
    from torch.profiler import ProfilerActivity, profile
    n_prof = 10
    for name, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                amb.check(fn(), ctx)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            t_us = getattr(e, "device_time_total", None)
            if t_us is None:
                t_us = e.cuda_time_total
            if "kernel" in e.key and t_us > 0:
                kern[e.key.split("(")[0][-48:]] = t_us / n_prof / 1e3
        out["kernels_ms"][name] = {"total": sum(kern.values()), "by_kernel": kern}
    cells = rows * cols
    k_ms = out["kernels_ms"]["lonlat_bilinear"]["total"]
    out["lonlat_bilinear_cells_per_s"] = cells / (k_ms * 1e-3)
    # HBM floor: the layer's 4 bytes per cell written (the tile's window and the tables are a few MB, read from L2)
    out["hbm_floor_ms"] = 4.0 * cells / 3.35e12 * 1e3
    out["kernel_over_hbm_floor"] = k_ms / out["hbm_floor_ms"]

    # the device band's layer
    amb.check(calls["lonlat_bilinear"](), ctx)
    gm.sync()
    gm.download(("elevation",))
    want = gm["elevation"].copy(order="F")

    # end to end from a Deflate-tiled GeoTIFF
    t0 = time.perf_counter()
    b = lonlat_tiff(band, gt, ("tiles", 512, 512), 3)
    out["file_MB"] = len(b) / 1e6
    out["file_write_s"] = time.perf_counter() - t0
    e2e = []
    for _ in range(args.repeats):
        g2 = fresh()
        g2.sync()
        t0 = time.perf_counter()
        g2.from_geotiff("elevation", b, map_epsg=32632)
        g2.sync()
        e2e.append(time.perf_counter() - t0)
    out["end_to_end_s"] = e2e
    g2.download(("elevation",))
    got = g2["elevation"]
    out["file_equals_device_band_bits"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))

    # host status quo on the first --host-cols columns, scaled
    hc = min(args.host_cols, cols)
    x = np.array([gm.getPosition((i, 0))[0] for i in range(rows)])[:, None] * np.ones((1, hc))
    y = np.array([gm.getPosition((0, j))[1] for j in range(hc)])[None, :] * np.ones((rows, 1))
    t0 = time.perf_counter()
    host = host_import(x, y, band, gt)
    t_host = time.perf_counter() - t0
    out["host_s_measured"] = t_host
    out["host_cols"] = hc
    out["host_s_whole_map"] = t_host * cols / hc
    out["host_max_abs_diff_m"] = float(np.abs(host - want[:, :hc]).max())
    assert out["file_equals_device_band_bits"], "the file and the device band gave different layers"
    assert out["host_max_abs_diff_m"] < 2e-3, out["host_max_abs_diff_m"]
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lonlat_import_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
