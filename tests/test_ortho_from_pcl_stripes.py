"""ortho::OrthoFromPcl::process (ortho-from-pcl.cc:20-113) on the layouts the DSM and the orthomosaic already have: a
context owning one column stripe, a cloud that arrives sharded by stripe (border halos with their intensities), several
GPUs of one process (amb_multi_ortho_from_pcl_process and the drop-in header under AMB_SHIM_GPUS=N), and one process
per GPU with the exchange inside the library.  In every case a stripe must be bit-identical to the same columns of the
undivided map, adaptive interpolation included where the stripe holds the whole cloud.

The `gpu` tests also run on the emulated kernels (tests/emu) through the last tests of this file."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from common import ROOT, ulp_diff
from aerial_mapper_b200 import synth
from oracle import pyoracle as po

EMULATED = os.environ.get("AMB_TEST_EMU", "0") not in ("", "0")

ROWS, COLS, RES = 100, 150, 0.5
STRIPES = [(0, 45), (45, 58), (58, 150)]   # ragged: none is a multiple of the tile width, the middle one is narrow


def make_cloud(n, half_x, half_y, seed):
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(-half_x, half_x, n), rng.uniform(-half_y, half_y, n), rng.uniform(0, 5, n)]
    inten = rng.integers(0, 256, n).astype(np.int32)
    return xyz, inten


def border_y(c, rows=ROWS, cols=COLS, res=RES):
    """y of the border between columns c - 1 and c (column 0 is the max-y side)."""
    _, qy = synth.grid_positions(rows, cols, res)
    return 0.5 * (qy[c - 1] + qy[c])


def grid_map(rows=ROWS, cols=COLS, res=RES, col_range=None):
    import aerial_mapper_b200 as amb
    gm = amb.AerialGridMap(amb.GridMapSettings(0, 0, rows * res, cols * res, res)).getMutable()
    if col_range is not None:
        gm.context(0, col_range)
    return gm


def run_pcl(xyz, inten, radius, adaptive=False, col_range=None, rows=ROWS, cols=COLS, res=RES):
    import aerial_mapper_b200 as amb
    gm = grid_map(rows, cols, res, col_range)
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius,
                                              use_adaptive_interpolation=adaptive)).process(xyz, inten, gm)
    return gm


def assert_stripe_bits(stripe, full, c0, c1):
    assert np.array_equal(stripe[:, c0:c1].view(np.uint32), full[:, c0:c1].view(np.uint32)), (c0, c1)


# ---- 1. stripe contexts ---------------------------------------------------------------------------------------------
def stripe_scene(radius, seed):
    xyz, inten = make_cloud(16000, ROWS * RES / 2 + 2.0, COLS * RES / 2 + 2.0, seed)
    qx, qy = synth.grid_positions(ROWS, COLS, RES)
    xyz[5, :2] = (qx[30], qy[45])     # perfect matches on the two sides of a stripe border
    xyz[6, :2] = (qx[71], qy[57])
    inten[5], inten[6] = 17, 230
    # a cluster on the border between the first two stripes: its tiles stage far more points than the shared-memory
    # stage holds, so they go whole to the warp-per-cell kernel
    rng = np.random.default_rng(seed + 1)
    k = 12000
    cl = np.c_[rng.uniform(-2.0, 2.0, k), border_y(45) + rng.uniform(-1.5, 1.5, k), np.zeros(k)]
    xyz = np.r_[xyz, cl]
    inten = np.r_[inten, rng.integers(0, 256, k).astype(np.int32)]
    return xyz, inten


@pytest.mark.gpu
@pytest.mark.parametrize("radius,seed", [(1, 3), (2, 4), (10, 5)])
def test_stripe_contexts_equal_the_undivided_map(radius, seed):
    xyz, inten = stripe_scene(radius, seed)
    whole = run_pcl(xyz, inten, radius)
    full = whole["ortho"]
    assert whole.timings()["dsm_cells_empty"] > 0          # the cluster's tiles took the warp-per-cell path
    assert full[30, 45] == 17.0 and full[71, 57] == 230.0    # perfect matches
    for c0, c1 in STRIPES:
        gm = run_pcl(xyz, inten, radius, col_range=(c0, c1))
        assert_stripe_bits(gm["ortho"], full, c0, c1)


# ---- 2. a sharded cloud, simulated on one device ----------------------------------------------------------------------
@pytest.mark.gpu
def test_sharded_cloud_with_intensity_halos_equals_the_undivided_map():
    """Owner masks, amb_ortho_from_pcl_extract_halo, a hand gather of what the all-gather would deliver, then
    process_device(.., d_ids=) per stripe (three ranks one after the other on one device)."""
    import torch
    import aerial_mapper_b200 as amb
    from aerial_mapper_b200 import sharding
    radius, world = 2, len(STRIPES)
    xyz_np, inten_np = stripe_scene(radius, 21)
    full = run_pcl(xyz_np, inten_np, radius)["ortho"]
    dev = torch.device("cpu" if EMULATED else "cuda:0")   # emulated kernels: host memory is device memory
    device_sync = (lambda: None) if EMULATED else torch.cuda.synchronize
    xyz = torch.from_numpy(xyz_np).to(dev)
    inten = torch.from_numpy(inten_np).to(dev)
    ids = torch.arange(xyz.shape[0], dtype=torch.int64, device=dev)
    ranks = []
    for r, (c0, c1) in enumerate(STRIPES):
        gm = grid_map()
        gm.to_device(0, col_range=(c0, c1), names=("ortho",))
        y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
        m = sharding.owner_mask(xyz[:, 1], y_lo, y_hi, r, world)   # no centre shift in OrthoFromPcl
        hx = sharding.HaloExchange(torch, world, r, 20000, xyz[m], ids[m], dev, local_intensities=inten[m])
        reach = amb.lib().amb_dsm_halo_reach(C.byref(gm.geometry), radius)
        amb.check(amb.lib().amb_dsm_set_density_hint(gm.context(), xyz.shape[0] / float(ROWS * COLS)), gm.context())
        hx.extract(gm.context(), y_lo, y_hi, reach)
        ranks.append((gm, hx, c0, c1))
    assert sum(hx.n_local for _, hx, _, _ in ranks) == xyz.shape[0]   # the stripes partition the cloud
    device_sync()
    for gm, _, _, _ in ranks:
        gm.sync()
    gathered = torch.stack([hx.send for _, hx, _, _ in ranks])
    device_sync()
    o = amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius))
    for gm, hx, c0, c1 in ranks:
        hx.gathered.copy_(gathered)
        device_sync()
        assert (hx.counts() <= hx.cap).all() and (hx.counts() > 0).all()
        hx.assemble()
        o.process_device(hx.big_xyz.data_ptr(), hx.big_intensities.data_ptr(), hx.n_total, gm,
                         d_ids=hx.big_ids.data_ptr())
        gm.sync()
        gm.download(("ortho",))
        assert_stripe_bits(gm["ortho"], full, c0, c1)
    adaptive = amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius, use_adaptive_interpolation=True))
    with pytest.raises(amb.AmbError) as ei:     # no rank of a sharded cloud holds the whole cloud
        adaptive.process_sharded_device(0, 0, 0, 0, ranks[0][0], 1000)
    assert ei.value.status == -8


# ---- 3. adaptive interpolation on stripes (each stripe context gets the whole cloud) ------------------------------------
def adaptive_scene(kind, seed):
    if kind == "single":                      # one point, in the last stripe: every cell of every stripe takes it
        qx, qy = synth.grid_positions(ROWS, COLS, RES)
        return np.array([[qx[40] + 0.13, qy[120] + 0.21, 3.0]]), np.array([99], np.int32)
    xyz, inten = make_cloud(9000, ROWS * RES / 2 - 0.01, COLS * RES / 2 - 0.01, seed)
    keep = np.ones(len(xyz), bool)
    # holes centred on stripe borders: 4 m wide needs 10 r, 10 m wide 100 r, 24 m wide 1000 r (radius 1)
    for cx, c, side in ((19.0, 45, 4.0), (-19.0, 45, 10.0), (0.0, 58, 24.0)):
        cy = border_y(c)
        keep &= ~((np.abs(xyz[:, 0] - cx) < side / 2) & (np.abs(xyz[:, 1] - cy) < side / 2))
    return xyz[keep], inten[keep]


def adaptive_levels(xyz, radius):
    """Per cell: the adaptive level the reference's loop stops at (0 = primary ball non-empty)."""
    from scipy.spatial import cKDTree
    qx, qy = synth.grid_positions(ROWS, COLS, RES)
    q = np.c_[np.repeat(qx[:, None], COLS, 1).ravel(), np.repeat(qy[None, :], ROWS, 0).ravel()]
    d2 = cKDTree(xyz[:, :2]).query(q)[0] ** 2
    lvl = np.zeros(len(q), int)
    t = float(radius)
    while (d2 >= t).any() and lvl.max() < 9:
        lvl[d2 >= t] += 1
        t *= 10
    return lvl


@pytest.mark.gpu
@pytest.mark.parametrize("kind,radius,seed", [("holes", 1, 31), ("single", 2, 0)])
def test_adaptive_interpolation_on_stripes_equals_the_undivided_map(kind, radius, seed):
    xyz, inten = adaptive_scene(kind, seed)
    if kind == "holes":
        assert {1, 2, 3} <= set(np.unique(adaptive_levels(xyz, radius)))   # 10 r, 100 r and 1000 r all occur
    whole = run_pcl(xyz, inten, radius, adaptive=True)
    full = whole["ortho"]
    assert np.isfinite(full).all() and (full != 255.0).all()
    if kind == "single":
        assert (full == 99.0).all()
    if po.have_ref():   # the reference's own cell loop (nanoflann) with its 10^k radius growth
        ref = np.full((ROWS, COLS), 255.0, np.float32, order="F")
        assert po.ortho_from_pcl_process(po.make_geometry(ROWS, COLS, RES), ref, xyz, inten, radius=radius,
                                         adaptive=True, use_ref=True) == 0
        assert ulp_diff(full, ref).max() <= 1
    for c0, c1 in STRIPES:
        gm = run_pcl(xyz, inten, radius, adaptive=True, col_range=(c0, c1))
        gm.sync()
        assert_stripe_bits(gm["ortho"], full, c0, c1)


# ---- 4. restrictions ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_adaptive_stripe_with_a_point_beyond_the_bin_grid_restores_the_layer():
    import aerial_mapper_b200 as amb
    xyz, inten = make_cloud(3000, ROWS * RES / 2 - 0.01, COLS * RES / 2 - 0.01, 41)
    xyz[17, 1] = COLS * RES / 2 + 40.0       # far beyond the map + apron, on the side of another stripe
    c0, c1 = STRIPES[1]
    gm = grid_map(col_range=(c0, c1))
    gm["ortho"] = np.arange(ROWS * COLS, dtype=np.float32).reshape(ROWS, COLS) % 251   # a recognisable layer
    before = gm["ortho"].copy(order="F")
    with pytest.raises(amb.AmbError) as ei:
        amb.OrthoFromPcl(amb.OrthoFromPclSettings(use_adaptive_interpolation=True)).process(xyz, inten, gm)
    assert ei.value.status == -8                               # AMB_ERR_UNSUPPORTED
    gm.download(("ortho",))
    assert np.array_equal(gm["ortho"], before)                 # the stripe got its content back


# ---- 5. amb_multi_ortho_from_pcl_process ----------------------------------------------------------------------------
def multi_pcl(xyz, inten, radius, adaptive, n_gpus):
    import aerial_mapper_b200 as amb
    L = amb.lib()
    g = amb.Geometry()
    amb.check(L.amb_geometry_init(ROWS * RES, COLS * RES, RES, 0.0, 0.0, C.byref(g)))
    m = C.c_void_p()
    amb.check(L.amb_multi_create(C.byref(g), int(n_gpus), C.byref(m)))
    try:
        xyz = np.ascontiguousarray(xyz, np.float64)
        inten = np.ascontiguousarray(inten, np.int32)
        st = L.amb_multi_ortho_from_pcl_process(m, xyz.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p),
                                                len(xyz), int(radius), 1 if adaptive else 0)
        assert st == 0, L.amb_multi_last_error(m)
        out = np.empty((ROWS, COLS), np.float32, order="F")
        amb.check(L.amb_multi_download_layer(m, amb.LAYER_ID["ortho"], out.ctypes.data_as(C.c_void_p)))
        return out, L.amb_multi_size(m)
    finally:
        L.amb_multi_destroy(m)


@pytest.mark.gpu
@pytest.mark.parametrize("adaptive", [False, True])
def test_multi_gpu_entry_point_equals_a_single_context(adaptive, gpu_count):
    # every visible device takes a stripe (one stripe on a one-GPU box: the entry point against the single context)
    xyz, inten = adaptive_scene("holes", 51) if adaptive else stripe_scene(2, 52)
    single = run_pcl(xyz, inten, 2, adaptive=adaptive)["ortho"]
    got, stripes = multi_pcl(xyz, inten, 2, adaptive, max(gpu_count, 1))
    assert stripes == max(gpu_count, 1)
    assert np.array_equal(got.view(np.uint32), single.view(np.uint32))


# ---- 6. the drop-in header ------------------------------------------------------------------------------------------
def build_pcl_demo(tmp_path):
    if EMULATED:   # the same source against the emulated kernels
        sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
        import build_emu
        libdir, name = os.path.dirname(build_emu.build()), "amb_emu"
    else:
        import aerial_mapper_b200 as amb
        amb.lib()
        libdir, name = os.path.join(ROOT, "aerial_mapper_b200"), "aerial_mapper_b200"
    exe = str(tmp_path / "pcl_shim_demo")
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Wextra", "-Werror", "-DAMB_SHIM_MINI",
                           "-I" + os.path.join(ROOT, "aerial_mapper_b200", "shim"),
                           os.path.join(ROOT, "tests", "cpp", "pcl_shim_demo.cc"), "-o", exe, "-L" + libdir, "-l" + name,
                           "-Wl,-rpath," + libdir])
    return exe


def write_pcl_scenario(path, xyz, inten, radius, adaptive):
    with open(path, "wb") as f:
        np.array([ROWS * RES, COLS * RES, RES, 0.0, 0.0], np.float64).tofile(f)
        np.array([len(xyz), radius, 1 if adaptive else 0], np.int64).tofile(f)
        np.ascontiguousarray(xyz, np.float64).tofile(f)
        np.ascontiguousarray(inten, np.int32).tofile(f)


@pytest.mark.gpu
@pytest.mark.parametrize("adaptive", [False, True])
def test_drop_in_header_equals_the_python_mirror_on_one_and_two_gpus(tmp_path, adaptive, gpu_count):
    exe = build_pcl_demo(tmp_path)
    xyz, inten = adaptive_scene("holes", 61) if adaptive else stripe_scene(2, 62)
    scen = tmp_path / "pcl_scenario.bin"
    write_pcl_scenario(scen, xyz, inten, 2, adaptive)
    mirror = run_pcl(xyz, inten, 2, adaptive=adaptive)["ortho"]
    for gpus in ((1, 2) if gpu_count >= 2 else (1,)):   # AMB_SHIM_GPUS=2 needs two devices (amb_multi_create)
        out = tmp_path / ("ortho_%d.bin" % gpus)
        r = subprocess.run([exe, str(scen), str(out)], capture_output=True, text=True,
                           env=dict(os.environ, AMB_SHIM_GPUS=str(gpus)))
        assert r.returncode == 0, r.stderr
        got = np.fromfile(out, np.float32).reshape(COLS, ROWS).T
        assert np.array_equal(got.view(np.uint32), mirror.view(np.uint32)), gpus


# ---- 7. one process per GPU, the exchange inside the library --------------------------------------------------------
def _rank_worker(rank, world, port, tmp, mode):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    import aerial_mapper_b200 as amb
    from aerial_mapper_b200 import sharding
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)   # carries the library's NCCL id only
    radius = 2
    xyz_np, inten_np = stripe_scene(radius, 71)
    c0, c1 = sharding.stripe_range(COLS, rank, world)
    gm = grid_map()
    gm.to_device(rank, col_range=(c0, c1), names=("ortho",))
    ctx = gm.context()
    sharding.init_comm(ctx, dist, rank, world)
    amb.check(amb.lib().amb_comm_set_exchange(ctx, int(mode)), ctx)
    amb.check(amb.lib().amb_dsm_set_density_hint(ctx, len(xyz_np) / float(ROWS * COLS)), ctx)
    y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
    m = sharding.owner_mask(xyz_np[:, 1], y_lo, y_hi, rank, world)
    dev = torch.device("cuda", rank)
    xyz = torch.from_numpy(np.ascontiguousarray(xyz_np[m])).to(dev)
    inten = torch.from_numpy(np.ascontiguousarray(inten_np[m])).to(dev)
    ids = torch.from_numpy(np.flatnonzero(m).astype(np.int64)).to(dev)
    torch.cuda.synchronize(dev)
    o = amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius))
    for _ in range(2):   # a second step: the peer-push segments alternate by step parity
        o.process_sharded_device(xyz.data_ptr(), inten.data_ptr(), ids.data_ptr(), int(m.sum()), gm, 20000)
        gm.sync()
    gm.download(("ortho",))
    np.savez(os.path.join(tmp, "pcl_rank%d.npz" % rank), c0=c0, c1=c1, ortho=gm["ortho"][:, c0:c1],
             exchange=amb.lib().amb_comm_last_exchange(ctx))
    dist.barrier()
    del gm
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,expect", [(0, (4, 2)), (3, (2,)), (1, (1,))])
def test_one_process_per_gpu_every_exchange_mode_equals_the_undivided_map(tmp_path, mode, expect):
    if EMULATED:
        pytest.skip("NCCL and torch.cuda need real devices")
    import torch
    import torch.multiprocessing as mp
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs at least two CUDA devices")
    full = run_pcl(*stripe_scene(2, 71), 2)["ortho"]
    port = 32500 + (os.getpid() % 2000) + mode
    mp.spawn(_rank_worker, args=(world, port, str(tmp_path), mode), nprocs=world, join=True)
    for r in range(world):
        z = np.load(os.path.join(str(tmp_path), "pcl_rank%d.npz" % r))
        assert int(z["exchange"]) in expect, (mode, int(z["exchange"]))   # 0 (automatic): peer push where peers map
        assert_stripe_bits_slab(z["ortho"], full, int(z["c0"]), int(z["c1"]))


def assert_stripe_bits_slab(slab, full, c0, c1):
    assert np.array_equal(slab.view(np.uint32), full[:, c0:c1].view(np.uint32)), (c0, c1)


# ---- 8. the gpu tests above on the emulated kernels (no GPU needed) -------------------------------------------------
def test_the_gpu_tests_of_this_file_pass_on_the_emulated_kernels():
    from test_emulated_kernels import run_child
    tail = run_child("gpu", ["test_ortho_from_pcl_stripes.py"])
    assert " passed" in tail and "failed" not in tail


# ---- 9. two gloo ranks, the sharded OrthoFromPcl through sharding.HaloExchange on the emulated kernels ----------------
def _emu_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["AMB_TEST_EMU"] = "1"
    import torch
    import torch.distributed as dist
    import conftest  # noqa: F401  (swaps in tests/emu/_build/libamb_emu.so)
    import aerial_mapper_b200 as amb
    from aerial_mapper_b200 import sharding
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    radius = 2
    xyz_np, inten_np = stripe_scene(radius, 81)
    c0, c1 = sharding.stripe_range(COLS, rank, world)
    if rank == 0:   # the undivided map on the same emulated kernels
        np.save(os.path.join(tmp, "emu_pcl_full.npy"), run_pcl(xyz_np, inten_np, radius)["ortho"])
    gm = grid_map()
    gm.to_device(0, col_range=(c0, c1), names=("ortho",))
    xyz = torch.from_numpy(xyz_np)
    inten = torch.from_numpy(inten_np)
    ids = torch.arange(xyz.shape[0], dtype=torch.int64)
    y_lo, y_hi = sharding.stripe_y_interval(gm.geometry, c0, c1)
    m = sharding.owner_mask(xyz[:, 1], y_lo, y_hi, rank, world)
    hx = sharding.HaloExchange(torch, world, rank, 20000, xyz[m], ids[m], torch.device("cpu"),
                               local_intensities=inten[m])
    reach = amb.lib().amb_dsm_halo_reach(C.byref(gm.geometry), radius)
    amb.check(amb.lib().amb_dsm_set_density_hint(gm.context(), xyz.shape[0] / float(ROWS * COLS)), gm.context())
    hx.extract(gm.context(), y_lo, y_hi, reach)
    hx.exchange(dist)
    assert (hx.counts() <= hx.cap).all() and (hx.counts() > 0).all()
    hx.assemble()
    amb.OrthoFromPcl(amb.OrthoFromPclSettings(interpolation_radius=radius)).process_device(
        hx.big_xyz.data_ptr(), hx.big_intensities.data_ptr(), hx.n_total, gm, d_ids=hx.big_ids.data_ptr())
    gm.sync()
    gm.download(("ortho",))
    np.savez(os.path.join(tmp, "emu_pcl_rank%d.npz" % rank), c0=c0, c1=c1, n_local=hx.n_local,
             ortho=gm["ortho"][:, c0:c1])
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_cloud_on_two_gloo_ranks_on_the_emulated_kernels(tmp_path):
    import torch.multiprocessing as mp
    world = 2
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_emu_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    xyz, inten = stripe_scene(2, 81)
    full = np.full((ROWS, COLS), 255.0, np.float32, order="F")    # the oracle's undivided map
    assert po.ortho_from_pcl_process(po.make_geometry(ROWS, COLS, RES), full, xyz, inten, radius=2, num_threads=-1) == 0
    undivided = np.load(os.path.join(str(tmp_path), "emu_pcl_full.npy"))
    assert np.array_equal(undivided == 255.0, full == 255.0) and ulp_diff(undivided, full).max() <= 1
    n_local = 0
    for r in range(world):
        z = np.load(os.path.join(str(tmp_path), "emu_pcl_rank%d.npz" % r))
        c0, c1 = int(z["c0"]), int(z["c1"])
        n_local += int(z["n_local"])
        assert_stripe_bits_slab(z["ortho"], undivided, c0, c1)
    assert n_local == len(xyz)                                    # the stripes partition the cloud
