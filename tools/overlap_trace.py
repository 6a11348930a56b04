"""How far the DSM's fine scatter (P2) and its gather overlap: per-kernel start and end times from torch.profiler.

    python tools/overlap_trace.py [--calls 10] [--warmup 3] [--out DIR] [--label NAME]

Workload: tools/prof_run.py's DSM driver (bench.py's dsm_c2 cloud: 50 M points over 10000^2 cells at 0.25 m, seeded in
HBM).  `--calls` warmed-up Dsm calls run under torch.profiler (CUDA activities only).  Per call, from the device
intervals of its kernels:
  p1_ms           dsm_partition_kernel
  p2_busy_ms      time during which at least one dsm_fine_scatter_kernel launch runs (union of its intervals)
  gather_busy_ms  the same for the gather launches (dsm_gather_kernel_f32 / dsm_gather_kernel)
  overlap_ms      time during which both run
  span_ms         first P2 or gather start -> last P2 or gather end: what the two cost together
  serial_ms       p2_busy_ms + gather_busy_ms: what they would cost one after the other
  fill_ms         mark + order + warp-per-cell kernels (device time)
  call_ms         first binning kernel start -> last kernel end of the call
Prints the card's name, power limit and clocks, one JSON line per call and the means, and with --out writes every kernel
interval of every call to DIR/overlap_<label>.json.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bin_split  # noqa: E402  (gpu_info, kineto event access)
import prof_run  # noqa: E402
import torch  # noqa: E402

KINDS = (("p1", "dsm_partition_kernel"), ("p2", "dsm_fine_scatter_kernel"), ("gather", "dsm_gather_kernel"),
         ("fill", "dsm_mark_buckets_kernel"), ("fill", "dsm_bucket_order_kernel"), ("fill", "dsm_cell_kernel"),
         ("scan", "scan_"))


def kind(name):
    for k, key in KINDS:
        if key in name:
            return k
    return None


def union(iv):
    """Merged [start, end) intervals."""
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def length(iv):
    return sum(b - a for a, b in iv)


def intersect(x, y):
    i = j = 0
    tot = 0
    while i < len(x) and j < len(y):
        a, b = max(x[i][0], y[j][0]), min(x[i][1], y[j][1])
        tot += max(0, b - a)
        if x[i][1] < y[j][1]:
            i += 1
        else:
            j += 1
    return tot


def split_calls(events):
    """Device kernels of the trace, grouped into calls: a call starts at its dsm_partition_kernel."""
    dev = sorted(((name, start, start + dur) for name, start, dur, is_dev in map(bin_split._ev, events) if is_dev
                  and kind(name)), key=lambda e: e[1])
    calls = []
    for name, a, b in dev:
        k = kind(name)
        if k == "p1" and (not calls or any(kind(n) == "fill" for n, _, _ in calls[-1])):
            calls.append([])
        if calls:
            calls[-1].append((name, a, b))
    return calls


def measure(call):
    ns = 1e-6
    iv = {k: [(a, b) for n, a, b in call if kind(n) == k] for k in ("p1", "p2", "gather", "fill", "scan")}
    p2, ga = union(iv["p2"]), union(iv["gather"])
    both = union(iv["p2"] + iv["gather"])
    return {"p1_ms": length(union(iv["p1"])) * ns, "p2_busy_ms": length(p2) * ns, "gather_busy_ms": length(ga) * ns,
            "overlap_ms": intersect(p2, ga) * ns, "span_ms": (both[-1][1] - both[0][0]) * ns,
            "serial_ms": (length(p2) + length(ga)) * ns, "fill_ms": sum(b - a for a, b in iv["fill"]) * ns,
            "call_ms": (max(b for _, _, b in call) - min(a for _, a, _ in call)) * ns,
            "p2_launches": len(iv["p2"]), "gather_launches": len(iv["gather"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="write the kernel intervals into this directory")
    ap.add_argument("--label", default="this_build")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("overlap_trace.py: no CUDA device — these are GPU timings")
    print(json.dumps({"gpu": bin_split.gpu_info(), "label": args.label,
                      "env": {k: v for k, v in os.environ.items() if k.startswith("AMB_")}}), flush=True)

    n = bin_split.N
    xyz, gm, d = prof_run.dsm_setup(bin_split.ROWS, bin_split.COLS, bin_split.RES, n)
    for _ in range(args.warmup):
        d.process_device(xyz.data_ptr(), n, gm)
    gm.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.calls):
            d.process_device(xyz.data_ptr(), n, gm)
        gm.sync()
    calls = split_calls(prof.profiler.kineto_results.events())
    if len(calls) != args.calls:
        raise SystemExit(f"overlap_trace.py: found {len(calls)} calls in the trace, expected {args.calls}")
    rows = [measure(c) for c in calls]
    for r in rows:
        print(json.dumps({k: round(v, 4) for k, v in r.items()}), flush=True)
    mean = {k: round(sum(r[k] for r in rows) / len(rows), 4) for k in rows[0]}
    mean["span_ms_min"] = round(min(r["span_ms"] for r in rows), 4)
    mean["span_ms_max"] = round(max(r["span_ms"] for r in rows), 4)
    print(json.dumps({"label": args.label, "mean": mean}), flush=True)
    if not args.out:
        return
    os.makedirs(args.out, exist_ok=True)
    t0 = calls[0][0][1]
    with open(os.path.join(args.out, f"overlap_{args.label}.json"), "w") as f:
        json.dump({"label": args.label, "mean": mean,
                   "calls": [[(name, (a - t0) * 1e-6, (b - t0) * 1e-6) for name, a, b in c] for c in calls]}, f)


if __name__ == "__main__":
    main()
