"""The orthomosaic's exact-decision guards at UTM map coordinates (csrc/ortho_kernels.cu: the per-tile bound `delta` on
|fast path - reference| in camera coordinates, and the pixel / camera-plane / angle guards scaled by it).

At a map position of 5e6 m the fused fast path (pre-multiplied rotation, FMA) and the reference's operation sequence
(quaternion rotation, un-contracted) round 5e6 m quantities differently: keypoints differ by up to ~1e-8 px and sin^2 of
the observation angle by up to ~6e-11 at f = 3000 px and 30 m above the ground, ten times the fixed guards that suffice
near the map origin.  Every scenario of tests/test_gpu_ortho_adversarial.py runs here at the origin, at common.UTM and at
a southern-hemisphere northing, with full-resolution focal lengths 30 .. 600 m above the ground, through every path:
host frames (SELECT + texel gather) and resident frames, the dominance cull on and off, brute force, a ragged stripe
context, and two process() calls whose frames tie across the calls (the running best read from the layer).

Bar: observation_index and the ortho / colored_ortho bits equal the CPU oracle's in every cell, elevation_angle within
1 ulp, no spurious CHECK(alpha > 0) error; where oracle/_ref is built, also the reference's own ortho-backward-grid.cc.
The last test runs this file on the emulated kernels (tests/emu), so every CPU run checks the kernel logic too."""
import os

import numpy as np
import pytest

from common import UTM, fresh_layers, ulp_diff
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

gpu = pytest.mark.gpu
EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")

NADIR = (0.0, 1.0, 0.0, 0.0)   # qw qx qy qz: rotation by pi about x, every product of the rotation exact
SOUTH = (4.6e5 + 321.0, 9.9e6 + 211.0)                     # a southern-hemisphere northing
POSITIONS = {"origin": (0.0, 0.0), "utm": UTM, "south": SOUTH}
DIST = {0: (0.0, 0.0, 0.0, 0.0), 1: (-0.05, 0.01, 1e-4, 1e-4), 2: (0.01, -0.002, 0.0005, -0.0001), 3: (0.9, 0.0, 0.0, 0.0)}
# every path through the kernels: (frames on the host or resident, AMB_ORTHO_DOMINANCE, brute force, stripe context)
PATHS = (("host", "1", False, False), ("device", "1", False, False), ("host", "0", False, False),
         ("host", "1", True, False), ("device", "0", False, True))


def camera(width, height, cu, cv, f, dist_type=0):
    return dict(width=width, height=height, fu=f, fv=f, cu=cu, cv=cv, dist_type=dist_type, dist=DIST[dist_type])


def mismatches(a, b):
    return int((~((a == b) | (np.isnan(a) & np.isnan(b)))).sum())


def _device_images(imgs):
    if EMULATED:                    # tests/emu: host memory is device memory
        return imgs, [im.ctypes.data for im in imgs]
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(im)).cuda() for im in imgs]
    return d, [t.data_ptr() for t in d]


def gpu_run(path, pos, rows, cols, res, elev, camd, batches, colored=False, prior=None):
    """The CUDA orthomosaic over `batches` (a list of (poses, images), one process() call each) on `path`; returns the
    layers over the whole map (a stripe path runs every stripe in its own context and stitches them).  prior: the
    elevation_angle layer before the first call (an earlier batch's running best), default 0."""
    where, dominance, brute, stripes = path
    old = os.environ.get("AMB_ORTHO_DOMINANCE")
    os.environ["AMB_ORTHO_DOMINANCE"] = dominance
    try:
        out = {k: np.empty((rows, cols), np.float32, order="F")
               for k in ("elevation_angle", "observation_index", "ortho", "colored_ortho")}
        cuts = (0, cols // 3 + 1, 2 * cols // 3 + 3, cols) if stripes else (0, cols)   # ragged stripes
        for c0, c1 in zip(cuts[:-1], cuts[1:]):
            gm = amb.AerialGridMap(amb.GridMapSettings(pos[0], pos[1], rows * res, cols * res, res)).getMutable()
            gm["elevation"] = elev
            if prior is not None:
                gm["elevation_angle"] = prior
            if stripes:
                gm.context(0, (c0, c1))
            o = amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(colored_ortho=colored), gm)
            o.brute_force = brute
            if where == "device":
                gm.to_device(0)
            frames = []   # device frames: alive until the asynchronous kernels that read them have finished (gm.sync)
            for poses, imgs in batches:
                if where == "device":
                    keep, ptrs = _device_images(imgs)
                    frames.append(keep)
                    o.process_device(poses, ptrs, camd["width"] * (3 if colored else 1), gm)
                else:
                    o.process(poses, imgs, gm)
            if where == "device":
                gm.sync()         # raises a deferred CHECK(alpha > 0) failure of process_device
                gm.download()
            del frames
            for k in out:
                out[k][:, c0:c1] = gm[k][:, c0:c1]
        return out
    finally:
        if old is None:
            os.environ.pop("AMB_ORTHO_DOMINANCE", None)
        else:
            os.environ["AMB_ORTHO_DOMINANCE"] = old


def oracle_run(pos, rows, cols, res, elev, camd, batches, colored=False, refsrc=False, prior=None):
    L = fresh_layers(rows, cols, elev)
    if prior is not None:
        L["elevation_angle"][...] = prior
    g = po.make_geometry(rows, cols, res, pos[0], pos[1])
    run = po.refsrc_ortho_process if refsrc else po.ortho_process
    for poses, imgs in batches:
        st, _ = run(g, L, po.make_camera(**camd), poses, imgs, colored=colored)
        assert st == 0
    return L


def compare(gm, L, colored=False):
    """(observation_index mismatches, output-layer mismatches, max elevation_angle ulps)"""
    key = "colored_ortho" if colored else "ortho"
    return (mismatches(gm["observation_index"], L["observation_index"]),
            int((gm[key].view(np.uint32) != L[key].view(np.uint32)).sum()),
            int(ulp_diff(gm["elevation_angle"], L["elevation_angle"]).max()))


def run_all(pos, rows, cols, res, elev, camd, batches, paths=PATHS, colored=False, check_refsrc=False, prior=None):
    """Every path against the oracle (and the reference's own sources); returns the oracle's layers."""
    batches = [(np.asarray(p, np.float64).reshape(-1, 7), imgs) for p, imgs in batches]
    L = oracle_run(pos, rows, cols, res, elev, camd, batches, colored, prior=prior)
    bad = []
    for path in paths:
        c = compare(gpu_run(path, pos, rows, cols, res, elev, camd, batches, colored, prior), L, colored)
        if c[0] or c[1] or c[2] > 1:
            bad.append((path, c))
    assert not bad, "mismatches against the oracle (path, (observation_index, ortho, elevation_angle ulps)): %s" % bad
    if check_refsrc and po.have_refsrc():
        R = oracle_run(pos, rows, cols, res, elev, camd, batches, colored, refsrc=True, prior=prior)
        key = "colored_ortho" if colored else "ortho"
        assert mismatches(R["observation_index"], L["observation_index"]) == 0
        assert np.array_equal(R[key].view(np.uint32), L[key].view(np.uint32))
    return L


def images(n, camd, colored=False):
    return [synth.procedural_image(k, camd["width"], camd["height"], 3 if colored else 1) for k in range(n)]


def flat(rows, cols, z):
    return np.full((rows, cols), z, np.float32, order="F")


# Exact geometry: f = 3072 px and a flight height h in {32, 128, 512} m with res = h / 1024, so a cell is exactly 3 px
# and the nadir camera's keypoints are 3 * (cells from the camera) + c exactly, at any map position (the subtraction of
# two lattice coordinates of the same magnitude is exact, 1/h is a power of two).
EXACT_H = (32.0, 128.0, 512.0)
F_EXACT = 3072.0


@gpu
@pytest.mark.parametrize("h", EXACT_H)
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_every_keypoint_on_a_half_integer(where, h):
    pos, rows, cols, res = POSITIONS[where], 48, 40, h / 1024.0
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    # half a cell (1.5 px) off the lattice in x and y: every keypoint is an integer + 0.5
    pose = [qx[20] + 0.5 * res, qy[17] + 0.5 * res, 64.0 + h, *NADIR]
    camd = camera(96, 72, 48.0, 36.0, F_EXACT)
    L = run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [([pose], images(1, camd))], check_refsrc=True)
    assert (~np.isnan(L["observation_index"])).sum() > 500


@gpu
@pytest.mark.parametrize("h", EXACT_H)
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_keypoints_exactly_on_the_raster_edges(where, h):
    pos, rows, cols, res = POSITIONS[where], 48, 40, h / 1024.0
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    pose = [qx[24], qy[20], 64.0 + h, *NADIR]            # on the lattice: kx runs over ..., -3, 0, 3, ..., 93, 96, ...
    camd = camera(96, 72, 48.0, 36.0, F_EXACT)
    L = run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [([pose], images(1, camd))], check_refsrc=True)
    assert (~np.isnan(L["observation_index"])).sum() == 32 * 24      # kx == 0 in, kx == W out; the same along y


@gpu
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_camera_plane_at_the_minimum_depth(where):
    pos, rows, cols, res = POSITIONS[where], 16, 16, 1.0 / 32.0
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    camd = camera(32, 32, 16.0, 16.0, F_EXACT)
    for tz, visible in ((1e-10, False), (np.nextafter(1e-10, 1.0), True), (-1e-10, False), (0.0, False)):
        pose = [qx[7], qy[9], tz, *NADIR]                # elevation 0: camera z of the cell below is exactly tz
        L = run_all(pos, rows, cols, res, flat(rows, cols, 0.0), camd, [([pose], images(1, camd))])
        assert (~np.isnan(L["observation_index"][7, 9])) == visible


@gpu
@pytest.mark.parametrize("h", EXACT_H)
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_exact_angle_tie_follows_the_float32_rounded_running_best(where, h):
    pos, rows, cols, res = POSITIONS[where], 40, 40, h / 1024.0
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    # two cameras mirrored about the column of cells x = qx[20]: the same alpha for every cell of that column
    p0 = [qx[20] - 8 * res, qy[20], 64.0 + h, *NADIR]
    p1 = [qx[20] + 8 * res, qy[20], 64.0 + h, *NADIR]
    camd = camera(96, 96, 48.0, 48.0, F_EXACT)
    imgs = images(2, camd)
    col = run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [([p0, p1], imgs)])["observation_index"][20, :]
    assert (~np.isnan(col)).sum() > 20 and (col == 0).any() and (col == 1).any()
    # the same tie split over two process() calls: the second call's frame against the running best in the layer
    L = run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [([p0], imgs[:1]), ([p1], imgs[1:])])
    col2 = L["observation_index"][20, :]
    assert np.array_equal(np.isnan(col), np.isnan(col2)) and (col2 == 0).any()


# Full-resolution focal length at 30, 100 and 600 m above the ground: f = 3000 px, res = h / 2000 (1.5 px per cell), so
# cameras on the cell lattice put keypoints on integers and half-integers and on the raster edges; quaternions perturbed
# by 3e-14 .. 3e-10 (keypoints moved by ~1e-10 .. 1e-6 px), positions by 0 .. 2 ulps.
HEIGHTS = (30.0, 100.0, 600.0)


def perturbed_scenes(rng, pos, rows, cols, res, h, n_scenes):
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    for trial in range(n_scenes):
        eps = 10.0 ** rng.uniform(-13.5, -9.5)
        poses = []
        for k in range(2 + trial % 2):
            t = [qx[rng.integers(12, rows - 12)] + 0.5 * res * rng.integers(0, 2),
                 qy[rng.integers(12, cols - 12)] + 0.5 * res * rng.integers(0, 2), 64.0 + h]
            t = [v + np.spacing(v) * rng.integers(-2, 3) for v in t]
            q = np.array(NADIR) + eps * rng.standard_normal(4)
            poses.append([*t, *(q / np.linalg.norm(q))])
        if trial % 4 == 3:   # a frame whose camera plane passes within rounding of a cell: z ~ 1e-10
            poses.append([qx[5], qy[5], 64.0 + 1e-10 * (1.0 + 1e-3 * rng.standard_normal()), *NADIR])
        if trial % 4 == 2:   # mirrored partner with a perturbed attitude: near-ties of the observation angle
            q = np.array(NADIR) + eps * rng.standard_normal(4)
            poses.append([2 * qx[rows // 2] - poses[0][0], poses[0][1], poses[0][2], *(q / np.linalg.norm(q))])
        yield poses


@gpu
@pytest.mark.parametrize("dist_type", [0, 1, 2, 3])
@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_poses_perturbed_across_the_boundaries(where, h, dist_type):
    """Whatever the oracle decides for keypoints within 1e-10 .. 1e-6 px of raster edges and half-integers, camera
    planes at the minimum depth and near-ties of the observation angle, every CUDA path decides."""
    pos, rows, cols, res = POSITIONS[where], 48, 48, h / 2000.0
    rng = np.random.default_rng(7000 + 10 * dist_type + int(h))
    camd = camera(64, 48, 32.0, 24.0, 3000.0, dist_type)
    n = 6 if EMULATED else 16
    for s, poses in enumerate(perturbed_scenes(rng, pos, rows, cols, res, h, n)):
        imgs = images(len(poses), camd, colored=s % 3 == 1)
        paths = PATHS if s < 2 else (PATHS[s % len(PATHS)],)
        run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [(poses, imgs)], paths=paths,
                colored=s % 3 == 1, check_refsrc=s == 0)


@gpu
@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_running_best_from_the_layer_ties_across_calls(where, h):
    """Mirrored cameras split over two process() calls: the second call's frames tie the first call's angles to within
    1e-10 in sin^2, decided against the float32 running best read from the layer (the 1e-11 band and its scaling)."""
    pos, rows, cols, res = POSITIONS[where], 48, 48, h / 2000.0
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    rng = np.random.default_rng(900 + int(h))
    camd = camera(64, 48, 32.0, 24.0, 3000.0, 1)
    for trial in range(3 if EMULATED else 8):
        eps = 10.0 ** rng.uniform(-13.5, -10.5)
        first, second = [], []
        for k in range(2):
            i, j = rng.integers(16, rows - 16), rng.integers(12, cols - 12)
            d = (1 + rng.integers(0, 6)) * res
            q0 = np.array(NADIR) + eps * rng.standard_normal(4)
            q1 = np.array(NADIR) + eps * rng.standard_normal(4)
            first.append([qx[i] - d, qy[j], 64.0 + h, *(q0 / np.linalg.norm(q0))])
            second.append([qx[i] + d, qy[j], 64.0 + h, *(q1 / np.linalg.norm(q1))])
        imgs = images(4, camd)
        L = run_all(pos, rows, cols, res, flat(rows, cols, 64.0), camd, [(first, imgs[:2]), (second, imgs[2:])],
                    paths=PATHS if trial == 0 else (PATHS[trial % len(PATHS)],), check_refsrc=trial == 0)
        assert (L["observation_index"] == 0).any() or (L["observation_index"] == 1).any()


def oblique_scene(pos, h, dist_type, seed):
    """A frame that sees its cells 35 degrees off its optical axis (principal point far left of a narrow 192 x 144
    raster, f = 3000 px, h metres above flat ground, yawed and rolled so that no rotation product is exact), and a
    running best in the layer equal to the float32 nearest to each cell's reference angle.  Off the axis the observation
    angle moves with the camera coordinates (|d sin^2 / d x_c| ~ 1 / n instead of ~1e-3 / n near the axis), so at UTM
    the fast path's sin^2 misses the reference's by more than the fixed 1e-11 band, and the cells whose reference angle
    lies within ~1e-10 of a float32 (a few per thousand) are decided against the layer inside the band's scaling.
    A second frame far away only joins the frame list of brute force (the multi-candidate loop).
    Returns (pos, rows, cols, res, elevation, camera, batches, prior layer, cells within 1e-10 of their layer value)."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    rows = cols = 256
    res = 0.012 * h / 30.0                                   # about one cell per pixel
    f = 3000.0
    camd = dict(width=192, height=144, fu=f, fv=f, cu=-f * 0.7, cv=72.0, dist_type=dist_type, dist=DIST[dist_type])
    yaw, roll = rng.uniform(0.2, 1.2), rng.uniform(-0.05, 0.05)
    q = synth._quat_mul(synth._quat_mul(synth._axis_angle((0, 0, 1), yaw), np.array(NADIR)),
                        synth._axis_angle((1, 0, 0), roll))
    q /= np.linalg.norm(q)
    R_G_C = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()
    d = R_G_C @ np.array([(96.0 - camd["cu"]) / f, 0.0, 1.0])      # ray of the raster's centre pixel
    qx, qy = synth.grid_positions(rows, cols, res, *pos)
    ground = np.array([qx[rows // 2], qy[cols // 2], 64.0])
    c = ground - (-h / d[2]) * d                                  # the camera h metres above the ground, on that ray
    pose = [c[0], c[1], c[2], *q]
    far = [c[0] + 900.0, c[1] - 700.0, c[2], *q]                  # sees none of the map
    cam = po.make_camera(**camd)
    prior = np.zeros((rows, cols), np.float32, order="F")
    near = 0
    for i in range(rows):
        for j in range(cols):
            x, y, z = po.transform_to_camera(cam, np.asarray(pose), np.array([qx[i], qy[j], 64.0]))
            alpha = np.arcsin(abs(z) / np.sqrt(x * x + y * y + z * z))
            prior[i, j] = np.float32(alpha)
            near += abs(alpha - float(prior[i, j])) < 1e-10
    imgs = images(2, camd)
    return pos, rows, cols, res, flat(rows, cols, 64.0), camd, [([pose, far], imgs)], prior, near


@gpu
@pytest.mark.parametrize("dist_type", [0, 1])
@pytest.mark.parametrize("h", (30.0, 100.0))
@pytest.mark.parametrize("where", sorted(POSITIONS))
def test_oblique_rays_against_the_running_best_in_the_layer(where, h, dist_type):
    """The sin^2 band against a running best read from the layer, where it has to grow with the coordinates: rays
    35 degrees off the axis, a layer holding the float32 nearest to every cell's reference angle."""
    for seed in range(2):
        pos, rows, cols, res, elev, camd, batches, prior, near = oblique_scene(POSITIONS[where], h, dist_type, seed)
        L = run_all(pos, rows, cols, res, elev, camd, batches, prior=prior, check_refsrc=seed == 0)
        assert near > 20                                         # cells within 1e-10 of their layer value
        won = L["observation_index"] == 0
        assert won.sum() > 2000 and (~won & (L["elevation_angle"] == prior)).sum() > 2000   # both outcomes, often


@gpu
@pytest.mark.skipif(EMULATED, reason="250 frames of 4000x3000: minutes on the emulated kernels")
def test_full_size_c3_stripe_at_utm():
    """BASELINE config C3 (8000^2 cells at 0.5 m, 250 frames of 4000x3000, 600 m) placed at UTM coordinates, on a
    24-column stripe: host frames in a stripe context against the oracle restricted to the same cells."""
    rows = cols = 8000
    res = 0.5
    c0, c1 = 3988, 4012
    camd = dict(synth.C3_CAMERA)
    poses = synth.lawnmower_poses(10, 25, rows * res / 2, cols * res / 2, 600.0, seed=4, center=UTM)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"]) for k in range(len(poses))]
    qx, qy = synth.grid_positions(rows, cols, res, *UTM)
    elev_stripe = np.asfortranarray(synth.terrain(qx[:, None] - UTM[0], qy[None, c0:c1] - UTM[1]).astype(np.float32))
    gm = amb.AerialGridMap(amb.GridMapSettings(UTM[0], UTM[1], rows * res, cols * res, res),
                           layer_names=("ortho", "elevation", "elevation_angle", "observation_index")).getMutable()
    gm.layers["elevation"][:, c0:c1] = elev_stripe
    gm.context(0, (c0, c1))
    amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm).process(poses, imgs, gm)
    L = {"elevation": np.full((rows, cols), np.nan, np.float32, order="F"),
         "elevation_angle": np.zeros((rows, cols), np.float32, order="F"),
         "observation_index": np.full((rows, cols), np.nan, np.float32, order="F"),
         "ortho": np.full((rows, cols), 255.0, np.float32, order="F")}
    L["elevation"][:, c0:c1] = elev_stripe
    st, _ = po.ortho_process(po.make_geometry(rows, cols, res, *UTM), L, po.make_camera(**camd), poses, imgs,
                             cell_range=(rows * c0, rows * c1))
    assert st == 0
    a, b = gm["observation_index"][:, c0:c1], L["observation_index"][:, c0:c1]
    assert mismatches(a, b) == 0
    assert np.array_equal(gm["ortho"][:, c0:c1].view(np.uint32), L["ortho"][:, c0:c1].view(np.uint32))
    assert ulp_diff(gm["elevation_angle"][:, c0:c1], L["elevation_angle"][:, c0:c1]).max() <= 1
    assert (~np.isnan(b)).all() and len(np.unique(b)) > 20


# ---- the same tests on the emulated kernels (no GPU needed) ----------------------------------------------------------
def test_this_file_passes_on_the_emulated_kernels():
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_gpu_ortho_utm.py"])
    assert " passed" in tail and "failed" not in tail
