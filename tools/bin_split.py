"""Split the DSM binning stage by kernel and set each kernel against the HBM bandwidth this card reaches.

    python tools/bin_split.py [--calls 20] [--warmup 3] [--trace DIR]

Workload: tools/prof_run.py's DSM driver (bench.py's dsm_c2 cloud: 50 M points over 10000^2 cells at 0.25 m, seeded in
HBM).  Two runs in one process:

1. Plain device copies timed with CUDA events: a 1.2 GB read-only reduction, a 1.6 GB write-only fill and a 1.6 GB
   copy.  They give the bandwidth the card actually reaches (nothing is written to MEASURED_PEAKS.json).
2. `--calls` warmed-up Dsm calls under torch.profiler (CUDA activities only).  Per binning kernel: mean device time
   per call and the algorithmic bytes of DESIGN §4.0's byte model, computed from the shapes:
     memsets          the bucket counts G (4 B per bucket) + the bucket flags (1 B per bucket) + the stage counters
     P1 partition     24 B read + 32 B written per point, + the uint16 run-start table
     scan_reduce      G read once;  scan_apply: G read and written;  scan_spine: the block sums
     P2 fine_scatter  32 B read + 32 B written per point, + the run-start table read (summed over its launches, one
                      per band)
   plus the stage's span on the device (first memset start -> last P2 end), which includes the launch gaps and, since
   the gather runs beside P2 (tools/overlap_trace.py), part of the gather.

Prints the card's name and power limit, one JSON line per copy, one per kernel and one for the stage.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import prof_run  # noqa: E402  (puts ROOT on sys.path)
import torch  # noqa: E402

ROWS, COLS, RES, N = 10000, 10000, 0.25, 50_000_000
PART_TILE = 2048          # kPartTile (dsm_partition.inc)
WINDOW = 48 << 20         # default bytes per coarse destination (dsm_kernels.cu)
MAX_COARSE = 256
KERNELS = ("memsets", "dsm_partition_kernel", "scan_reduce_kernel", "scan_spine_kernel", "scan_apply_kernel",
           "dsm_fine_scatter_kernel")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def plan_shapes(rows, cols, res, n, radius=1):
    """Bucket lattice and coarse destinations as amb_dsm's host plan derives them for a whole-map context."""
    def round_up(a, b):
        return (a + b - 1) // b * b
    lam, thr = 1.0, []
    while True:
        thr.append(lam * radius)
        lam *= 1.1
        if lam * radius > 7.0:
            break
    P = int((max(thr) ** 0.5) / res + 0.5 + 1e-6)
    W = int((float(radius) ** 0.5) / res + 0.5 + 1e-6)
    P = max(P, W)
    per_cell = n / (rows * cols)
    B = 1
    while B < 16 and per_cell * (2.0 * B) ** 2 <= 48.0:
        B *= 2
    Pa = round_up(P, B)
    tile_j1 = (cols - 1) // 32
    KR = round_up(round_up(rows, 32) + 2 * Pa, B) // B
    KC = round_up((tile_j1 + 1) * 32 + Pa + Pa, B) // B
    nbk = KR * KC
    g_elems = (nbk + 2 + 3) // 4 * 4
    S = max(1, min(min(-(-n * 32 // WINDOW), MAX_COARSE), KC))
    kj_per = -(-KC // S)
    S = -(-KC // kj_per)
    n_tiles = -(-n // PART_TILE)
    return {"B": B, "buckets": nbk, "g_elems": g_elems, "S": S, "n_tiles": n_tiles,
            "scan_blocks": -(-(g_elems // 4) // 1024)}


def byte_model(sh, n):
    g = 4 * sh["g_elems"]
    offs = 2 * (sh["S"] + 1) * sh["n_tiles"]
    return {"memsets": g + sh["buckets"] + 20,
            "dsm_partition_kernel": 24 * n + 32 * n + offs,
            "scan_reduce_kernel": g,
            "scan_spine_kernel": 8 * sh["scan_blocks"],
            "scan_apply_kernel": 2 * g,
            "dsm_fine_scatter_kernel": 32 * n + 32 * n + offs}


def copy_bandwidth(reps=20):
    """GB/s of a read-only reduction, a write-only fill and a copy, each over >= 1.2 GB, timed with CUDA events."""
    dev = torch.device("cuda:0")
    src = torch.ones(150_000_000, dtype=torch.float64, device=dev)        # 1.2 GB
    a = torch.empty(200_000_000, dtype=torch.float64, device=dev)         # 1.6 GB
    b = torch.empty_like(a)
    a.fill_(1.0)
    out = {}
    cases = (("read_1.2GB_sum", src.numel() * 8, lambda: src.sum()),
             ("write_1.6GB_fill", a.numel() * 8, lambda: b.fill_(2.0)),
             ("copy_1.6GB", 2 * a.numel() * 8, lambda: b.copy_(a)))
    for name, nbytes, fn in cases:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = {"bytes": nbytes, "ms": round(ms, 4), "GB_s": round(nbytes / ms / 1e6, 1)}
    del src, a, b
    torch.cuda.empty_cache()
    return out


def _ev(e):
    """(name, start_ns, duration_ns, is_device) of a kineto event, across torch versions."""
    name = e.name()
    start = e.start_ns() if hasattr(e, "start_ns") else e.start_us() * 1000
    dur = e.duration_ns() if hasattr(e, "duration_ns") else e.duration_us() * 1000
    dev = str(e.device_type()).endswith("CUDA")
    return name, start, dur, dev


def kernel_key(name):
    if name.startswith("Memset"):
        return "memset"
    for k in KERNELS[1:]:
        if k in name:
            return k
    return None


def split_stage(events):
    """Per binning call: device ms per kernel kind, and the stage span (first memset start -> last P2 end)."""
    dev = sorted((ev for ev in map(_ev, events) if ev[3]), key=lambda ev: ev[1])
    calls = []
    for i, (name, start, dur, _) in enumerate(dev):
        if kernel_key(name) != "dsm_partition_kernel":
            continue
        call = {k: 0.0 for k in KERNELS}
        first = start
        j = i - 1
        while j >= 0 and kernel_key(dev[j][0]) == "memset":   # the stage's memsets lie right before P1
            call["memsets"] += dev[j][2] / 1e6
            first = dev[j][1]
            j -= 1
        j = i
        while j < len(dev):   # P2 is one launch per band, interleaved with the gather: up to the next call's memsets
            k = kernel_key(dev[j][0])
            if k == "memset" or (k == "dsm_partition_kernel" and j > i):
                break
            if k is not None:
                call[k] += dev[j][2] / 1e6
            if k == "dsm_fine_scatter_kernel":
                call["stage_span"] = (dev[j][1] + dev[j][2] - first) / 1e6
            j += 1
        if "stage_span" in call:
            calls.append(call)
    return calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", default=None, help="also write the chrome trace into this directory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bin_split.py: no CUDA device — these are GPU timings")

    print(json.dumps({"gpu": gpu_info()}), flush=True)
    bw = copy_bandwidth()
    for k, v in bw.items():
        print(json.dumps({"copy": k, **v}), flush=True)
    peak = max(v["GB_s"] for v in bw.values())

    xyz, gm, d = prof_run.dsm_setup(ROWS, COLS, RES, N)
    for _ in range(args.warmup):
        d.process_device(xyz.data_ptr(), N, gm)
    gm.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.calls):
            d.process_device(xyz.data_ptr(), N, gm)
        gm.sync()
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace, "bin_split.pt.trace.json"))
    calls = split_stage(prof.profiler.kineto_results.events())
    if len(calls) != args.calls:
        raise SystemExit(f"bin_split.py: found {len(calls)} binning stages in the trace, expected {args.calls}")

    sh = plan_shapes(ROWS, COLS, RES, N)
    model = byte_model(sh, N)
    print(json.dumps({"shapes": sh, "points": N, "calls": len(calls), "peak_GB_s": peak,
                      "peak_source": "max of the copies above"}), flush=True)
    total_ms = 0.0
    for k in KERNELS:
        ms = sum(c[k] for c in calls) / len(calls)
        lo, hi = min(c[k] for c in calls), max(c[k] for c in calls)
        total_ms += ms
        gbs = model[k] / ms / 1e6 if ms > 0 else None
        print(json.dumps({"kernel": k, "bytes": model[k], "ms": round(ms, 4), "ms_min": round(lo, 4),
                          "ms_max": round(hi, 4), "GB_s": round(gbs, 1) if gbs else None,
                          "frac_of_copy_peak": round(gbs / peak, 3) if gbs else None}), flush=True)
    span = sum(c["stage_span"] for c in calls) / len(calls)
    alg = sum(model.values())
    print(json.dumps({"stage": "binning", "bytes": alg, "kernels_ms": round(total_ms, 4), "span_ms": round(span, 4),
                      "gaps_ms": round(span - total_ms, 4), "GB_s_over_span": round(alg / span / 1e6, 1),
                      "frac_of_copy_peak": round(alg / span / 1e6 / peak, 3)}), flush=True)


if __name__ == "__main__":
    main()
