"""JPEG frames decoded on the device (amb_jpeg_decode_device, amb_ortho_process_jpeg, csrc/jpeg_decode.cu) against
cv2.imread, on one GPU.

    python tools/jpeg_decode_bench.py [--frames 250] [--batch 25] [--out DIR]

Inputs: --frames frames of 4000 x 3000 (the joint_10k camera of bench.py) in two sets, each encoded by cv2.imencode at
quality 95 in 4:2:0 and 4:2:2, without restart markers and with a restart interval of one MCU row:
  synth       the procedural frames of aerial_mapper_b200.synth, noise-like: the worst case for Huffman decoding
  ortho_cut   4000 x 3000 windows of the colour orthomosaic rendered at the joint_10k geometry: realistic content
Reported per set and encoding:
  device      amb_jpeg_decode_device of all frames, --batch frames per call (files in pageable host memory, their H2D
              copy included), CUDA events around all calls, BGR output; checked against cv2.imread on a sample
  cv2_threads cv2.imdecode of the same files on every host thread (a thread pool over the frames), IMREAD_COLOR
  profile     (one encoding, a run of its own) the kernels' share of one batch under torch.profiler
End to end at the joint_10k geometry (gray orthomosaic from the synth frames at 4:2:0, written to a temporary
directory): io.read_jpeg_files + OrthoBackwardGrid.process_jpeg against io.load_images_from_file + process, outputs
checked identical.  Prints the card's name and power limit and one JSON line; writes it to --out/jpeg_decode_bench.json
if given."""
import argparse
import concurrent.futures as cf
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import aerial_mapper_b200 as amb  # noqa: E402
from aerial_mapper_b200 import _lib, api, synth  # noqa: E402
from aerial_mapper_b200 import io as amb_io  # noqa: E402
import bench  # noqa: E402


def encode(img, sampling, restart):
    import cv2
    flag = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if sampling == "420" else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, flag,
                                       cv2.IMWRITE_JPEG_RST_INTERVAL, restart])
    assert ok
    return b.tobytes()


def frame_sets(n, W, H):
    """{name: callable k -> BGR uint8 [H, W, 3]}"""
    import torch
    wl = bench.WORKLOADS["joint_10k"]
    rows, cols, res, half_x, half_y, camd, poses = bench.workload_inputs(wl)
    names = ("colored_ortho", "elevation", "elevation_angle", "observation_index")
    gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res), layer_names=names).getMutable()
    gm.layers["elevation"][...] = synth.analytic_elevation(rows, cols, res)
    gm.to_device(0, names=names)
    imgs = synth.procedural_images_torch(len(poses), W, H, 3, "cuda:0")
    torch.cuda.synchronize()
    amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=True), gm).process_device(
        poses, [imgs[k].data_ptr() for k in range(len(poses))], W * 3, gm)
    gm.sync()
    ctx = gm.context()
    band = torch.empty(rows * cols * 3, dtype=torch.uint8, device="cuda:0")
    amb.check(amb.lib().amb_export_raster_device(ctx, _lib.LAYER_ID["colored_ortho"], _lib.RASTER_BGR8,
                                                 band.data_ptr()), ctx)
    gm.sync()
    ortho = band.view(cols, rows, 3)
    rng = np.random.default_rng(5)
    offs = [(int(rng.integers(0, cols - H)), int(rng.integers(0, rows - W))) for _ in range(n)]
    return {"synth": lambda k: imgs[k % len(poses)].cpu().numpy(),
            "ortho_cut": lambda k: ortho[offs[k][0]:offs[k][0] + H, offs[k][1]:offs[k][1] + W].contiguous().cpu().numpy()}


def device_decode(files, batch, W, H, download=True):
    """ms of amb_jpeg_decode_device over all files, `batch` per call, into a reused device buffer; the last batch's
    outputs (on the host, if `download`)."""
    import torch
    ctx = api._jpeg_context(0)
    out = torch.empty((batch, H, W, 3), dtype=torch.uint8, device="cuda:0")
    L = amb.lib()
    calls = []
    for b0 in range(0, len(files), batch):
        chunk = files[b0:b0 + batch]
        bufs = [C.create_string_buffer(f, len(f)) for f in chunk]
        n = len(chunk)
        calls.append((bufs, (C.c_void_p * n)(*[C.cast(x, C.c_void_p).value for x in bufs]),
                      (C.c_size_t * n)(*[len(f) for f in chunk]), n))
    ptrs = (C.c_void_p * batch)(*[out[k].data_ptr() for k in range(batch)])
    steps = (C.c_size_t * batch)(*([W * 3] * batch))
    status = (C.c_int * batch)()

    def run():
        for _, fp, fs, n in calls:
            amb.check(L.amb_jpeg_decode_device(ctx, fp, fs, n, 3, ptrs, steps, status), ctx)
    run()   # warm-up: scratch allocated, modules loaded
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(torch.cuda.current_stream())
    run()
    e1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (out[:calls[-1][3]].cpu().numpy() if download else None)


def host_decode(files, threads):
    import cv2
    t0 = time.perf_counter()
    with cf.ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
    return (time.perf_counter() - t0) * 1e3


def profile(files, W, H):
    """ms per decode call of each kernel (and copy) of one batch, under torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        device_decode(files, len(files), W, H, download=False)   # two calls: warm-up and timed
    split = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0))
        if t <= 0:
            continue
        key = e.key.replace("amb::(anonymous namespace)::", "").split("(")[0].split("<")[0].strip()
        split[key] = split.get(key, 0.0) + t / 1e3 / 2
    torch.cuda.synchronize()
    return {k: round(v, 3) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}


def end_to_end(files, camd, poses, W, H):
    wl = bench.WORKLOADS["joint_10k"]
    rows, cols, res = wl["rows"], wl["cols"], wl["res"]
    names = ("ortho", "elevation", "elevation_angle", "observation_index")
    res_ms, layers = {}, {}
    with tempfile.TemporaryDirectory() as d:
        prefix = os.path.join(d, "frame_")
        for k, f in enumerate(files):
            with open("%s%d.jpg" % (prefix, k), "wb") as fh:
                fh.write(f)
        for arm in ("device_jpeg", "cv2_imread"):
            gm = amb.AerialGridMap(amb.GridMapSettings(0.0, 0.0, rows * res, cols * res, res),
                                   layer_names=names).getMutable()
            gm.layers["elevation"][...] = synth.analytic_elevation(rows, cols, res)
            gm.to_device(0, names=names)
            o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm)
            t0 = time.perf_counter()
            if arm == "device_jpeg":
                o.process_jpeg(poses, amb_io.read_jpeg_files(prefix, len(poses)), gm)
            else:
                o.process(poses, amb_io.load_images_from_file(prefix, len(poses)), gm)
            gm.sync()
            res_ms[arm] = (time.perf_counter() - t0) * 1e3
            written = ("ortho", "elevation_angle", "observation_index")
            gm.download(written)
            layers[arm] = {n: np.asarray(gm[n]).copy() for n in written}
    same = all(np.array_equal(layers["device_jpeg"][n].view(np.uint32), layers["cv2_imread"][n].view(np.uint32))
               for n in layers["device_jpeg"])
    return {"ms": {k: round(v, 1) for k, v in res_ms.items()}, "outputs_identical": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=250)
    ap.add_argument("--batch", type=int, default=25)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import cv2
    if amb.lib().amb_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("jpeg_decode_bench: no CUDA device (nothing is measured without one)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    wl = bench.WORKLOADS["joint_10k"]
    _, _, _, _, _, camd, poses = bench.workload_inputs(wl)
    W, H = camd["width"], camd["height"]
    threads = os.cpu_count() or 1
    sets = frame_sets(args.frames, W, H)
    out = {"card": card, "frames": args.frames, "width": W, "height": H, "quality": 95, "host_threads": threads,
           "cases": {}}
    profiled = False
    for set_name, frame in sets.items():
        for sampling in ("420", "422"):
            for restart in (0, W // 16):
                with cf.ThreadPoolExecutor(threads) as ex:   # (input preparation, not measured)
                    files = list(ex.map(lambda k: encode(frame(k), sampling, restart), range(args.frames)))
                dev_ms, last = device_decode(files, args.batch, W, H)
                k0 = len(files) - len(last)
                ok = all(np.array_equal(last[j], cv2.imdecode(np.frombuffer(files[k0 + j], np.uint8), cv2.IMREAD_COLOR))
                         for j in range(0, len(last), max(1, len(last) // 4)))
                host_ms = host_decode(files, threads)
                case = {"mean_file_bytes": int(np.mean([len(f) for f in files])), "device_ms": round(dev_ms, 1),
                        "device_ms_per_frame": round(dev_ms / len(files), 2), "cv2_all_threads_ms": round(host_ms, 1),
                        "speedup": round(host_ms / dev_ms, 2), "checked_equal": bool(ok)}
                if not profiled:
                    case["profile_ms_per_batch"] = profile(files[:args.batch], W, H)
                    profiled = True
                key = "%s_%s_rst%d" % (set_name, sampling, restart)
                out["cases"][key] = case
                print(key, json.dumps(case), flush=True)
                del files
    with cf.ThreadPoolExecutor(threads) as ex:
        gray_files = list(ex.map(lambda k: encode(sets["synth"](k), "420", 0), range(len(poses))))
    out["end_to_end_joint_10k_gray"] = end_to_end(gray_files, camd, poses, W, H)
    print("card:", card)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_decode_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
