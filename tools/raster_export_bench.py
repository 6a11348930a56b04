"""Raster export (amb_export_raster*, csrc/raster_export.cu) against what a user does without it, on one GPU.

    python tools/raster_export_bench.py [--rows 10000] [--cols 10000] [--launches 50] [--out DIR]

Device: every format's export into a device buffer, CUDA events over --launches launches after warm-up, against a
device-to-device copy of the same float32 layer in the same run.  Rate = cells * (4 + bytes per pixel) / time (the
bytes the export reads and writes); the copy's rate is 2 * 4 bytes per cell.
Host: amb_export_raster into page-locked and into pageable memory, against the status quo: amb_download_layer of the
float32 layer, then the conversion and flip in numpy.  Host clock around calls that end synchronised; best of --repeats.
Prints the card's name and power limit and one JSON line; writes it to --out/raster_export_bench.json if given."""
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
from aerial_mapper_b200 import _lib  # noqa: E402

FORMATS = ("f32", "gray8", "bgr8", "mask8")
LAYER = {"f32": "elevation", "gray8": "ortho", "bgr8": "colored_ortho", "mask8": "observation_index"}


def status_quo(gm, name, fmt):
    """float32 download + host conversion and flip to the same raster (the numpy a user would write)."""
    gm.download((name,))
    a = gm[name].T[:, ::-1]
    if fmt == "f32":
        return np.ascontiguousarray(a)
    if fmt == "gray8":
        return np.clip(np.rint(np.nan_to_num(a, nan=0.0)), 0, 255).astype(np.uint8)
    if fmt == "mask8":
        return np.where(np.isnan(a), 0, 255).astype(np.uint8)
    bits = np.ascontiguousarray(a).view(np.uint32)
    return np.stack([(bits >> s) & 0xFF for s in (0, 8, 16)], axis=-1).astype(np.uint8)


def best(fn, repeats):
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--cols", type=int, default=10000)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("raster_export_bench: no CUDA device (nothing is measured without one)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    rows, cols = args.rows, args.cols
    cells = rows * cols
    rng = np.random.default_rng(1)
    gm = amb.AerialGridMap(amb.GridMapSettings(464500.0, 5272500.0, float(rows), float(cols), 1.0),
                           layer_names=tuple(LAYER.values())).getMutable()
    gray = rng.integers(0, 256, cells).astype(np.float32)
    gm["ortho"] = gray.reshape(rows, cols, order="F")
    elev = (400.0 + rng.standard_normal(cells)).astype(np.float32)
    elev[rng.random(cells) < 0.1] = np.nan
    gm["elevation"] = elev.reshape(rows, cols, order="F")
    gm["colored_ortho"] = rng.integers(0, 1 << 24, cells, dtype=np.uint32).view(np.float32).reshape(rows, cols, order="F")
    gm["observation_index"] = np.where(rng.random(cells) < 0.2, np.nan, 3.0).astype(np.float32).reshape(rows, cols,
                                                                                                          order="F")
    del gray, elev
    gm.to_device(0, names=tuple(LAYER.values()))
    ctx = gm.context()
    L = amb.lib()
    stream = torch.cuda.ExternalStream(L.amb_stream(ctx), device="cuda:0")
    dst = torch.empty(cells * 4 + 64, dtype=torch.uint8, device="cuda:0")
    src_copy = torch.empty(cells * 4, dtype=torch.uint8, device="cuda:0")
    out = {"card": q, "rows": rows, "cols": cols, "launches": args.launches, "device": {}, "host": {}}

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

    # device: the copy and the four formats, alternated twice
    for rnd in range(2):
        with torch.cuda.stream(stream):
            t = timed(lambda: dst[:cells * 4].copy_(src_copy))
        out["device"].setdefault("d2d_copy", []).append({"ms": t * 1e3, "GBps": 8.0 * cells / t / 1e9})
        for fmt in FORMATS:
            f = _lib.RASTER_FORMAT[fmt]
            bpp = _lib.RASTER_BPP[f]
            t = timed(lambda: amb.check(L.amb_export_raster_device(ctx, _lib.LAYER_ID[LAYER[fmt]], f, dst.data_ptr()), ctx))
            out["device"].setdefault(fmt, []).append({"ms": t * 1e3, "GBps": (4.0 + bpp) * cells / t / 1e9})
    copy_rate = max(r["GBps"] for r in out["device"]["d2d_copy"])
    for fmt in FORMATS:
        out["device"][fmt + "_vs_copy"] = max(r["GBps"] for r in out["device"][fmt]) / copy_rate

    # host: pinned and pageable destinations against download + numpy
    for fmt in FORMATS:
        f = _lib.RASTER_FORMAT[fmt]
        bpp = _lib.RASTER_BPP[f]
        p = C.c_void_p()
        amb.check(L.amb_host_alloc(C.byref(p), cells * bpp))
        pinned = np.frombuffer((C.c_uint8 * (cells * bpp)).from_address(p.value), np.uint8)
        pageable = np.empty(cells * bpp, np.uint8)
        pageable[:] = 0  # touched: page faults are not part of the export
        name = LAYER[fmt]
        res = {}
        for label, buf in (("pinned", pinned), ("pageable", pageable)):
            amb.check(L.amb_export_raster(ctx, _lib.LAYER_ID[name], f, buf.ctypes.data), ctx)
            res[label + "_ms"] = 1e3 * best(lambda: amb.check(L.amb_export_raster(ctx, _lib.LAYER_ID[name], f,
                                                                                   buf.ctypes.data), ctx), args.repeats)
        ref = status_quo(gm, name, fmt)
        res["status_quo_ms"] = 1e3 * best(lambda: status_quo(gm, name, fmt), max(2, args.repeats // 2))
        res["identical"] = bool(pinned.tobytes() == ref.tobytes() and pageable.tobytes() == ref.tobytes())
        out["host"][fmt] = res
        L.amb_host_free(p)
    gm.sync()
    line = json.dumps(out)
    print("card:", q)
    for fmt in FORMATS:
        d, h = out["device"][fmt], out["host"][fmt]
        print("%-6s device %.3f ms (%.0f GB/s, %.0f%% of the copy's %.0f GB/s)  host pinned %.1f ms  pageable %.1f ms  "
              "download+numpy %.1f ms  identical %s" % (fmt, min(r["ms"] for r in d), max(r["GBps"] for r in d),
                                                        100 * out["device"][fmt + "_vs_copy"], copy_rate,
                                                        h["pinned_ms"], h["pageable_ms"], h["status_quo_ms"],
                                                        h["identical"]))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raster_export_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
