"""Workload driver for ncu captures (never a bench number): device-resident inputs, N repetitions of one stage."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth


def dsm_setup(rows, cols, res, n):
    """bench.py's dsm_c2-style cloud seeded in HBM, a device-resident map and a Dsm: (xyz, gm, dsm)."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(2)
    half_x, half_y = rows * res / 2, cols * res / 2
    xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
    xyz[:, 0] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * half_x
    xyz[:, 1] = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * half_y
    xyz[:, 2] = 100 + 10 * torch.sin(0.01 * xyz[:, 0]) * torch.cos(0.01 * xyz[:, 1]) + \
        0.05 * torch.randn(n, generator=g, device=dev, dtype=torch.float64)
    torch.cuda.synchronize()
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    gm.to_device(0, names=())
    return xyz, gm, amb.Dsm(amb.DsmSettings(), gm)


def dsm(rows, cols, res, n, reps):
    xyz, gm, d = dsm_setup(rows, cols, res, n)
    for r in range(reps):
        d.process_device(xyz.data_ptr(), n, gm)
        gm.sync()
        print(json.dumps({k: v for k, v in gm.timings().items() if k.startswith("dsm")}), flush=True)


def ortho(rows, cols, res, lines, per_line, agl, reps, colored=False):
    dev = torch.device("cuda:0")
    half_x, half_y = rows * res / 2, cols * res / 2
    camd = dict(synth.C3_CAMERA)
    poses = synth.lawnmower_poses(lines, per_line, half_x, half_y, agl, 4)
    n = len(poses)
    ch = 3 if colored else 1
    imgs = synth.procedural_images_torch(n, camd["width"], camd["height"], ch, dev)
    torch.cuda.synchronize()
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    gm.layers["elevation"][...] = synth.analytic_elevation(rows, cols, res)
    gm.to_device(0)
    o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm)
    ptrs = [imgs[k].data_ptr() for k in range(n)]
    for r in range(reps):
        amb.lib().amb_init_layers(gm.context())
        gm.upload(("elevation",))
        o.process_device(poses, ptrs, camd["width"] * ch, gm)
        gm.sync()
        print(json.dumps({k: v for k, v in gm.timings().items() if k.startswith("ortho")}), flush=True)


if __name__ == "__main__":
    what = sys.argv[1]
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    if what == "dsm":
        dsm(10000, 10000, 0.25, 50000000, reps)
    elif what == "dsm_small":
        dsm(4000, 4000, 0.25, 8000000, reps)
    elif what == "ortho":
        ortho(8000, 8000, 0.5, 10, 25, 600.0, reps)
