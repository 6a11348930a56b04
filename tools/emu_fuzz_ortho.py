"""Randomised cases of the orthomosaic kernels, plain and with the dominance cull on the CPU EMULATION of the kernel source (tests/emu) against the oracle:
sizes from 1x1, every distortion model / radius / density / offset the generators below draw, the map at the origin or at
UTM coordinates (northern and southern hemisphere).  No GPU involved.

    python tools/emu_fuzz_ortho.py <seed> <cases>      # exits non-zero on any mismatch
"""
import ctypes as C, sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ["AMB_TEST_EMU"] = "1"
import numpy as np
import conftest
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from oracle import pyoracle as po
from common import ulp_diff, fresh_layers
from scipy.spatial.transform import Rotation as R
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
# map positions from their own stream, so that a seed draws the same scenes as before positions were drawn
pos_rng = np.random.default_rng([int(sys.argv[1]) if len(sys.argv) > 1 else 0, 1])
POSITIONS = ((0.0, 0.0), (4.6e5 + 123.0, 5.2e6 + 457.0), (4.6e5 + 321.0, 9.9e6 + 211.0))
fails = 0
checked = 0
t0 = time.time()
N = int(sys.argv[2]) if len(sys.argv) > 2 else 30
for it in range(N):
    rows, cols = int(rng.integers(1, 200)), int(rng.integers(1, 200))
    res = float(rng.choice([0.25, 0.5, 1.0, 2.0]))
    dist_type = int(rng.integers(0, 3))
    dist = {0: (0, 0, 0, 0), 1: (-0.05, 0.01, 1e-4, 1e-4), 2: (0.01, -0.002, 0.0005, -0.0001)}[dist_type]
    if dist_type == 1 and rng.random() < 0.3:
        dist = (float(rng.uniform(-0.2, 0.1)), float(rng.uniform(-0.02, 0.05)), float(rng.normal(0, 1e-3)), float(rng.normal(0, 1e-3)))
    colored = bool(rng.integers(0, 2))
    scale = float(rng.choice([0.03, 0.06, 0.1]))
    camd = synth.scaled_camera(scale, dist_type=dist_type, dist=dist)
    if rng.random() < 0.5:
        q = np.r_[1.0, rng.normal(0, 0.1, 3)]; camd["q_C_B"] = tuple(q / np.linalg.norm(q)); camd["t_C_B"] = tuple(rng.normal(0, 0.3, 3))
    agl = float(rng.choice([20.0, 60.0, 150.0, 400.0]))
    lines, per = int(rng.integers(1, 5)), int(rng.integers(1, 7))
    poses = synth.lawnmower_poses(lines, per, rows * res / 2, cols * res / 2, agl, int(rng.integers(0, 1000)), jitter_pos=agl / 50,
                                  jitter_rp_deg=float(rng.choice([1.0, 5.0, 20.0])))
    pos = POSITIONS[int(pos_rng.integers(0, len(POSITIONS)))]
    poses[:, 0] += pos[0]
    poses[:, 1] += pos[1]
    ch = 3 if colored else 1
    imgs = [synth.procedural_image(k, camd["width"], camd["height"], ch) for k in range(len(poses))]
    elev = synth.analytic_elevation(rows, cols, res)
    elev += (rng.choice([0.0, 5.0, 40.0]) * np.sin(np.arange(rows)[:, None] / 3.0) * np.cos(np.arange(cols)[None, :] / 4.0)).astype(np.float32)
    if rng.random() < 0.5:
        m = rng.random((rows, cols)) < 0.05; elev[m] = np.nan
    prior = rng.random() < 0.3
    outs = []
    for dom in ("0", "1"):
        os.environ["AMB_ORTHO_DOMINANCE"] = dom
        gm = amb.AerialGridMap(amb.GridMapSettings(pos[0], pos[1], rows * res, cols * res, res)).getMutable()
        if gm.getSize() != (rows, cols): break
        gm["elevation"] = elev
        if prior:
            gm["elevation_angle"][...] = np.float32(1.2)   # an earlier batch already saw most cells steeply
        o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm)
        try:
            o.process(poses, imgs, gm)
        except amb.AmbError as e:
            print("it", it, "AmbError", e); break
        outs.append(gm)
    if len(outs) < 2:
        print('case', it, 'skipped: only', len(outs), 'runs', gm.getSize(), (rows, cols)); continue
    checked += 1
    L = fresh_layers(rows, cols, elev)
    if prior: L["elevation_angle"][...] = np.float32(1.2)
    st, _ = po.ortho_process(po.make_geometry(rows, cols, res, pos[0], pos[1]), L, po.make_camera(**camd), poses, imgs, colored=colored, num_threads=-1)
    key = "colored_ortho" if colored else "ortho"
    for nm, g in zip(("plain", "dom"), outs):
        ok = st == 0 and np.array_equal(g["observation_index"], L["observation_index"], equal_nan=True) and \
            np.array_equal(g[key].view(np.uint32), L[key].view(np.uint32)) and ulp_diff(g["elevation_angle"], L["elevation_angle"]).max() <= 1
        if not ok:
            fails += 1
            print("MISMATCH", nm, "it", it, (rows, cols, res, pos, dist_type, dist, colored, scale, agl, lines, per, prior), "st", st)
print("done", N, "cases,", checked, "checked, fails", fails, "%.0fs" % (time.time() - t0))
sys.exit(1 if fails or checked < N // 2 else 0)
