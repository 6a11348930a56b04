"""Column-stripe sharding of the map across ranks (SURVEY.md §8e) — host-side logic only.

Every grid cell is independent in both stages of the path, so the map shards with no data-path collective:
rank r owns the contiguous column stripe [c0, c1) of the column-major layers (a contiguous slab of rows*(c1-c0)
floats per layer) and computes it from the shared inputs.  One all-gather per step of the finished stripes gives
every rank the full map.  The functions below are backend-agnostic (torch tensors: NCCL on GPUs, gloo on CPU).
"""
import numpy as np


def stripe_width(cols, world):
    """Equal stripe width for a single equal-count all-gather (the last stripes may be partly or wholly padding)."""
    return (cols + world - 1) // world


def stripe_range(cols, rank, world):
    """Columns [c0, c1) owned by `rank` (c0 == c1 for a rank that owns nothing)."""
    w = stripe_width(cols, world)
    c0 = min(rank * w, cols)
    c1 = min(c0 + w, cols)
    return c0, c1


def pack_slabs(torch, slabs, rows, width, out):
    """Copy each layer's slab (1-D tensor of rows*(c1-c0) floats) into `out` [n_layers, rows*width] (zero padded)."""
    for k, t in enumerate(slabs):
        n = t.numel()
        out[k, :n].copy_(t)
        if n < rows * width:
            out[k, n:].zero_()
    return out


def all_gather_stripes(torch, dist, packed, world):
    """One collective: gathered[r] = rank r's packed slabs."""
    gathered = torch.empty((world,) + tuple(packed.shape), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(gathered.view(-1), packed.view(-1))
    return gathered


def unpack_full(gathered, rows, cols, world, n_layers):
    """gathered [world, n_layers, rows*width] -> list of n_layers numpy float32 arrays (rows, cols), F order."""
    width = stripe_width(cols, world)
    g = gathered.cpu().numpy().reshape(world, n_layers, width, rows)  # slab memory is column-major: [col][row]
    out = []
    for k in range(n_layers):
        full = np.empty((rows, cols), dtype=np.float32, order="F")
        for r in range(world):
            c0, c1 = stripe_range(cols, r, world)
            if c1 > c0:
                full[:, c0:c1] = g[r, k, :c1 - c0, :].T
        out.append(full)
    return out


# ---------------------------------------------------------------------------------------------------------------
# Sharded point cloud: each rank holds the points of its own stripe; ONE all-gather of the border halos per step.
def stripe_y_interval(geometry, c0, c1):
    """(y_lo, y_hi]: the y-range covered by the cells of columns [c0, c1) (amb_stripe_y_interval)."""
    import ctypes as C
    from ._lib import check, lib
    lo, hi = C.c_double(), C.c_double()
    check(lib().amb_stripe_y_interval(C.byref(geometry), int(c0), int(c1), C.byref(lo), C.byref(hi)))
    return lo.value, hi.value


def owner_mask(y_shifted, y_lo, y_hi, rank, world):
    """Points (by y - center_easting) owned by `rank`: its interval, plus everything beyond the map on the outer
    ranks (points outside the map still reach the border cells).  Column 0 is the max-y side (grid_map)."""
    m = (y_shifted > y_lo) & (y_shifted <= y_hi)
    if rank == 0:
        m = m | (y_shifted > y_hi)
    if rank == world - 1:
        m = m | (y_shifted <= y_lo)
    return m


def init_comm(ctx, dist, rank, world, device=None):
    """Make `ctx` (one context per rank) a member of an NCCL communicator owned by the LIBRARY (amb_comm_init): rank 0
    draws the unique id, torch.distributed only carries its 128 bytes to the other ranks.  Afterwards
    amb_dsm_process_sharded_device runs the halo exchange on the context's own stream."""
    import ctypes as C
    import torch
    from ._lib import check, lib
    buf = (C.c_ubyte * 128)()
    if rank == 0:
        check(lib().amb_comm_unique_id(C.cast(buf, C.c_void_p)))
    t = torch.tensor(list(buf), dtype=torch.uint8)
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, 0)
    raw = bytes(t.cpu().tolist())
    idb = (C.c_ubyte * 128).from_buffer_copy(raw)
    check(lib().amb_comm_init(ctx, int(rank), int(world), C.cast(idb, C.c_void_p)), ctx)


class HaloExchange(object):
    """Per-rank state of the border-halo exchange (torch tensors on the rank's device).

    send buffer (float64): [xyz: 3*cap | ids: cap (uint64 bits) | count: 1]; one all-gather fills `gathered`
    [world, 4*cap + 1]; assemble() lays out the DSM input `big_xyz` / `big_ids` = [all halos | local points] with
    this rank's own halo slot and every unused slot set to NaN (amb's binning drops NaN points).
    With `local_intensities` (OrthoFromPcl) the send buffer carries them too, as int32 bits in ceil(cap/2) more
    float64 slots after the count, and assemble() also lays out `big_intensities` beside `big_xyz` / `big_ids`."""

    def __init__(self, torch, world, rank, cap, local_xyz, local_ids, device, local_intensities=None):
        self.torch, self.world, self.rank, self.cap = torch, world, rank, int(cap)
        n = local_xyz.shape[0]
        self.n_local = n
        self.with_intensities = local_intensities is not None
        row = 4 * self.cap + 1 + ((self.cap + 1) // 2 if self.with_intensities else 0)
        self.send = torch.empty(row, dtype=torch.float64, device=device)
        self.gathered = torch.empty((world, row), dtype=torch.float64, device=device)
        self.big_xyz = torch.empty((world * self.cap + n, 3), dtype=torch.float64, device=device)
        self.big_ids = torch.empty(world * self.cap + n, dtype=torch.int64, device=device)
        self.big_xyz[world * self.cap:] = local_xyz
        self.big_ids[world * self.cap:] = local_ids
        self.local_xyz = self.big_xyz[world * self.cap:]
        self.local_ids = self.big_ids[world * self.cap:]
        self.big_intensities = self.local_intensities = None
        if self.with_intensities:
            self.big_intensities = torch.zeros(world * self.cap + n, dtype=torch.int32, device=device)
            self.big_intensities[world * self.cap:] = local_intensities
            self.local_intensities = self.big_intensities[world * self.cap:]
        self.n_total = world * self.cap + n

    def use_stream(self, stream):
        """Run the torch-side plumbing (fills, copies, the NCCL call) on `stream` — pass
        torch.cuda.ExternalStream(amb_stream(ctx)) so that everything is ordered on the library's own stream and no
        host synchronisation is needed between the compaction kernel, the all-gather and the DSM kernels."""
        self.stream = stream

    def _on_stream(self):
        import contextlib
        st = getattr(self, "stream", None)
        return self.torch.cuda.stream(st) if st is not None else contextlib.nullcontext()

    def extract(self, ctx, y_lo, y_hi, reach, center_easting=0.0):
        """Fill the send buffer with this rank's border points (hand-written compaction kernel, ctx's stream)."""
        import ctypes as C
        from ._lib import check, lib
        shared = getattr(self, "stream", None) is not None
        with self._on_stream():
            self.send.fill_(float("nan"))
        if not shared:
            self._host_sync()
        base = self.send.data_ptr()
        if self.with_intensities:   # OrthoFromPcl: no centre shift
            check(lib().amb_ortho_from_pcl_extract_halo(ctx, C.c_void_p(self.local_xyz.data_ptr()),
                                                        C.c_void_p(self.local_intensities.data_ptr()),
                                                        C.c_void_p(self.local_ids.data_ptr()), self.n_local,
                                                        float(y_lo), float(y_hi), float(reach), C.c_void_p(base),
                                                        C.c_void_p(base + 8 * (4 * self.cap + 1)),
                                                        C.c_void_p(base + 8 * 3 * self.cap), self.cap,
                                                        C.c_void_p(base + 8 * 4 * self.cap)), ctx)
        else:
            check(lib().amb_dsm_extract_halo(ctx, C.c_void_p(self.local_xyz.data_ptr()),
                                             C.c_void_p(self.local_ids.data_ptr()), self.n_local, float(y_lo),
                                             float(y_hi), float(reach), float(center_easting), C.c_void_p(base),
                                             C.c_void_p(base + 8 * 3 * self.cap), self.cap,
                                             C.c_void_p(base + 8 * 4 * self.cap)), ctx)
        if not shared:
            check(lib().amb_sync(ctx), ctx)

    def exchange(self, dist):
        with self._on_stream():
            dist.all_gather_into_tensor(self.gathered.view(-1), self.send)  # the one collective of the DSM stage

    def assemble(self):
        cap, w = self.cap, self.world
        with self._on_stream():
            self.big_xyz[:w * cap] = self.gathered[:, :3 * cap].reshape(w * cap, 3)
            self.big_ids[:w * cap] = self.gathered[:, 3 * cap:4 * cap].reshape(-1).view(self.torch.int64)
            if self.with_intensities:
                packed = self.gathered[:, 4 * cap + 1:].contiguous().view(self.torch.int32)   # [w, 2 * ceil(cap/2)]
                self.big_intensities[:w * cap] = packed[:, :cap].reshape(-1)
            self.big_xyz[self.rank * cap:(self.rank + 1) * cap] = float("nan")  # own halo: already local
        if getattr(self, "stream", None) is None:
            self._host_sync()

    def _host_sync(self):
        """Wait for the torch-side work on the current stream (nothing to wait for with host tensors)."""
        if self.send.is_cuda:
            self.torch.cuda.current_stream().synchronize()

    def counts(self):
        """Halo sizes reported by every rank (host read; > cap means a truncated halo)."""
        c = self.gathered[:, 4 * self.cap].contiguous().view(self.torch.int64).cpu().numpy()
        return (c & 0xffffffff).astype(np.int64)
