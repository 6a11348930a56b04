"""Orthomosaic decisions that sit EXACTLY on (or within rounding of) their boundaries — the cases the fused fast path of
ortho_kernel_dom cannot decide with FMA-contracted arithmetic and hands to the exact re-evaluation (csrc/ortho_kernels.cu:
kGuardPx / kGuardZ, exact_to_camera / exact_project).  Every scenario is compared with the CPU oracle and, when
oracle/_ref is built, with the reference's own ortho-backward-grid.cc: observation_index and pixels must be identical.

Geometry with exact arithmetic: a nadir camera (quaternion (0, 1, 0, 0): rotation by pi about x, every product exact),
no distortion, flight height 256 m above a constant elevation and f = 512 px, so a keypoint is 2*dx + cu exactly:
  * every keypoint on a half-integer  -> round-half-away-from-zero (ortho-backward-grid.cc:186-193)
  * keypoints exactly on kx == 0 / kx == W / ky == 0 / ky == H  -> the visibility predicate's >= and < (:164-171)
  * camera z exactly 1e-10 and one ulp above  -> kMinimumDepth (aslam PinholeCamera)
  * two frames with exactly equal observation angles  -> the strict `>` against the float32-rounded running best (:180-181)
and the same scenes with the pose perturbed by 1e-16 .. 1e-9 relative, which moves keypoints across those boundaries by
amounts far below the fast path's own rounding error."""
import numpy as np
import pytest

from common import fresh_layers, ulp_diff
import aerial_mapper_b200 as amb
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

NADIR = (0.0, 1.0, 0.0, 0.0)   # qw qx qy qz


def camera(width, height, cu, cv, f=512.0):
    return dict(width=width, height=height, fu=f, fv=f, cu=cu, cv=cv, dist_type=0, dist=(0.0, 0.0, 0.0, 0.0))


def run_both(rows, cols, res, elev, camd, poses, check_refsrc=True):
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 7)
    imgs = [synth.procedural_image(k, camd["width"], camd["height"]) for k in range(len(poses))]
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    gm["elevation"] = elev
    amb.OrthoBackwardGrid(amb.NCamera(**camd), amb.OrthoSettings(), gm).process(poses, imgs, gm)
    L = fresh_layers(rows, cols, elev)
    st, _ = po.ortho_process(po.make_geometry(rows, cols, res), L, po.make_camera(**camd), poses, imgs)
    assert st == 0
    a, b = gm["observation_index"], L["observation_index"]
    mism = ~((a == b) | (np.isnan(a) & np.isnan(b)))
    assert mism.sum() == 0, "observation_index differs from the oracle in %d cells" % int(mism.sum())
    assert np.array_equal(gm["ortho"].view(np.uint32), L["ortho"].view(np.uint32))
    assert ulp_diff(gm["elevation_angle"], L["elevation_angle"]).max() <= 1
    if check_refsrc and po.have_refsrc():
        R = fresh_layers(rows, cols, elev)
        st, _ = po.refsrc_ortho_process(po.make_geometry(rows, cols, res), R, po.make_camera(**camd), poses, imgs)
        assert st == 0
        rb = R["observation_index"]
        assert (~((a == rb) | (np.isnan(a) & np.isnan(rb)))).sum() == 0
        assert np.array_equal(gm["ortho"].view(np.uint32), R["ortho"].view(np.uint32))
    return gm, L


def flat(rows, cols, z):
    return np.full((rows, cols), z, np.float32, order="F")


def test_every_keypoint_on_a_half_integer():
    rows, cols, res = 48, 40, 0.5
    qx, qy = synth.grid_positions(rows, cols, res)
    # camera 0.25 m off the cell lattice in x and y: dx = 0.25 * odd -> kx = 2 dx + cu = integer + 0.5 for every cell
    pose = [qx[20] + 0.25, qy[17] + 0.25, 64.0 + 256.0, *NADIR]
    camd = camera(64, 48, 30.0, 22.0)
    gm, L = run_both(rows, cols, res, flat(rows, cols, 64.0), camd, [pose])
    seen = ~np.isnan(L["observation_index"])
    assert seen.sum() > 500      # the frame covers a good part of the map: all of those pixels were rounded at x.5


def test_keypoints_exactly_on_the_raster_edges():
    rows, cols, res = 64, 64, 0.5
    qx, qy = synth.grid_positions(rows, cols, res)
    pose = [qx[30], qy[33], 64.0 + 256.0, *NADIR]       # on the lattice: kx = 2 dx + cu is an integer for every cell
    camd = camera(40, 36, 20.0, 18.0)                   # kx runs over ..., -1, 0, 1, ..., 39, 40, 41, ... exactly
    gm, L = run_both(rows, cols, res, flat(rows, cols, 64.0), camd, [pose])
    seen = ~np.isnan(L["observation_index"])
    # exactly W x H cells see the frame: kx in [0, W) and ky in [0, H), with kx == 0 in and kx == W out
    assert seen.sum() == 40 * 36


def test_camera_plane_at_the_minimum_depth():
    rows, cols, res = 16, 16, 1.0
    qx, qy = synth.grid_positions(rows, cols, res)
    camd = camera(32, 32, 16.0, 16.0)
    for tz, visible in ((1e-10, False), (np.nextafter(1e-10, 1.0), True), (-1e-10, False), (0.0, False)):
        pose = [qx[7], qy[9], tz, *NADIR]               # elevation 0: camera z of the cell below is exactly tz
        gm, L = run_both(rows, cols, res, flat(rows, cols, 0.0), camd, [pose])
        assert (~np.isnan(L["observation_index"][7, 9])) == visible
        assert (~np.isnan(gm["observation_index"][7, 9])) == visible


def test_exact_angle_tie_follows_the_float32_rounded_running_best():
    rows, cols, res = 40, 40, 0.5
    qx, qy = synth.grid_positions(rows, cols, res)
    # two cameras mirrored about the column of cells x = qx[20]: |dx| equal, same alpha for every cell of that column
    p0 = [qx[20] - 4.0, qy[20], 64.0 + 256.0, *NADIR]
    p1 = [qx[20] + 4.0, qy[20], 64.0 + 256.0, *NADIR]
    camd = camera(64, 64, 32.0, 32.0)
    gm, L = run_both(rows, cols, res, flat(rows, cols, 64.0), camd, [p0, p1])
    col = L["observation_index"][20, :]
    # the running best is the FLOAT32-rounded angle (:181): the second frame of an exact tie wins exactly where that
    # rounding went down (alpha > (double)(float)alpha), and loses where it went up — both happen along the column
    assert (~np.isnan(col)).sum() > 20 and (col == 0).any() and (col == 1).any()
    col2 = run_both(rows, cols, res, flat(rows, cols, 64.0), camd, [p1, p0])[1]["observation_index"][20, :]
    assert np.array_equal(col, col2)          # mirrored frames: the same pattern whichever comes first


@pytest.mark.parametrize("dist_type", [0, 1, 2, 3])
def test_poses_perturbed_across_the_boundaries(dist_type):
    """Keypoints within ~1e-13..1e-6 px of raster edges and half-integers, camera planes within 1e-12 m of the minimum
    depth, near-ties of the observation angle: whatever the oracle decides, the CUDA path decides."""
    rng = np.random.default_rng(100 + dist_type)
    rows, cols, res = 40, 36, 0.5
    qx, qy = synth.grid_positions(rows, cols, res)
    dist = {0: (0, 0, 0, 0), 1: (-0.05, 0.01, 1e-4, 1e-4), 2: (0.01, -0.002, 0.0005, -0.0001), 3: (0.9, 0, 0, 0)}[dist_type]
    for trial in range(24):
        camd = camera(40, 36, 20.0, 18.0)
        camd.update(dist_type=dist_type, dist=dist)
        eps = 10.0 ** rng.uniform(-16, -9)
        poses = []
        for k in range(3):
            on_lattice = [qx[rng.integers(10, 30)] + 0.25 * rng.integers(0, 2), qy[rng.integers(10, 26)] + 0.25 * rng.integers(0, 2),
                          64.0 + 256.0]
            t = [v * (1.0 + eps * rng.standard_normal()) for v in on_lattice]
            q = np.array(NADIR) + eps * rng.standard_normal(4)
            q /= np.linalg.norm(q)
            poses.append([*t, *q])
        if trial % 4 == 3:   # a frame whose camera plane passes within rounding of a cell: z ~ 1e-10
            poses.append([qx[5], qy[5], 64.0 + 1e-10 * (1.0 + 1e-3 * rng.standard_normal()), *NADIR])
        if trial % 4 == 2:   # mirrored pair with a perturbed partner: a near-tie instead of an exact one
            poses.append([poses[0][0] + 8.0 * (1.0 + eps), poses[0][1], poses[0][2], *NADIR])
        run_both(rows, cols, res, flat(rows, cols, 64.0), camd, poses, check_refsrc=(trial % 6 == 0))
