"""Multi-GPU execution (SURVEY.md 8e; the reference has no distributed layer at all).

Mode R (replicas): one process per GPU, the field replicated in every GPU's HBM, particles sharded
contiguously by rank.  Particles do not interact on this path, so the step loop needs NO collective;
``torch.distributed`` only assembles results / timings (NCCL on GPUs, gloo in the CPU tests).

Mode D (domain decomposition, config 5): the rectilinear field is cut into X-slabs (+ halo columns), one per
GPU; a particle is advanced by the rank that owns its longitude and MIGRATES when it leaves the slab.  A curvilinear field is cut
into COLUMN slabs instead (``DecomposedFieldSet.from_curvilinear``): every rank holds the whole horizontal grid and its spatial hash,
only U, V, W are cut, and a particle belongs to the rank that owns the cell column its search finds.
Two transports:

* **peer memory (default over NCCL, one box)** -- ``connect_p2p``: every rank owns an inbox in its HBM that its
  peers map through CUDA IPC; the ADVECTION KERNEL ITSELF stores a leaving particle's 48-byte record into the new
  owner's inbox over NVLink (one system-scope atomic claims the slot), so the exchange overlaps the advection of
  the stayers and there is no classify / pack pass and no all-to-all.  Per round the host does one tiny
  all-reduce (the barrier that also decides termination) and ``migrate_p2p_finish`` (compact + append).
* **collectives (gloo tests, fallback)** -- device-side classify/pack kernels (``csrc/engine.cu``) -> count
  matrix all-gather -> 48-byte records exchanged with ``all_to_all_single`` -> device-side compact+append.

Trajectories are bit-identical to a single-GPU run either way because every particle-step sees the same grid
values (the slab is a slice of the global axis; ``ei`` stays global).

Time-slab streaming composes with mode D (``DecomposedFieldSet(..., time_window=W)``): every rank keeps W time levels of ITS slab
in HBM and all ranks slide their windows in lock-step -- to the earliest time any particle anywhere waits at, and only once a
round moved nobody (an arrival then always finds the levels it left with) -- so the host side of a rank reads only its own
columns of each level (``_SlabLevels``), and the next level is copied while the kernel runs, as on one GPU.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from .plan import KernelPlan, batch_facts, evaluated_mask


def shard_bounds(n: int, world: int) -> list[tuple[int, int]]:
    """Contiguous, balanced [lo, hi) ranges: the first n % world ranks get one extra particle."""
    base, extra = divmod(int(n), int(world))
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def shard_particles(pdata: dict, rank: int, world: int) -> dict:
    """This rank's slice of a particle SoA dict (copies, C-contiguous)."""
    lo, hi = shard_bounds(len(pdata["x"]), world)[rank]
    return {k: np.ascontiguousarray(v[lo:hi]) for k, v in pdata.items()}


def gather_particles(local: dict, dist, dst: int = 0):
    """Concatenate every rank's SoA on ``dst`` in rank order (deleted particles already compacted
    locally, so shards may have shrunk).  Returns the merged dict on ``dst`` and None elsewhere."""
    world = dist.get_world_size()
    rank = dist.get_rank()
    bucket = [None] * world if rank == dst else None
    dist.gather_object(local, bucket, dst=dst)
    if rank != dst:
        return None
    return {k: np.concatenate([b[k] for b in bucket], axis=0) for k in local}


def allreduce_max(value: float, dist, device="cpu") -> float:
    import torch

    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allreduce_sum(value: float, dist, device="cpu") -> float:
    import torch

    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


# --------------------------------------------------------------------------------------------------
# mode D
# --------------------------------------------------------------------------------------------------
RECORD_BYTES = 48  # PB_MIGRATION_RECORD_BYTES
RESUME_BYTES = 24  # PB_MIGRATION_RESUME_BYTES


def slab_plan(lon, world: int, halo_cells: int) -> list[dict]:
    """Cut the global X axis (node coordinates ``lon``) into ``world`` slabs of whole cells.

    Returns per rank: ``bounds`` (world+1 owned-interval edges, shared by all ranks), the inclusive local
    node range [lo, hi] = owned cells +- halo, ``xi_offset`` = lo, and whether each local edge is a
    global edge."""
    lon = np.asarray(lon)
    nx = lon.size
    ncell = nx - 1
    if world > ncell:
        raise ValueError(f"cannot cut {ncell} cells into {world} slabs")
    edges = [round(r * ncell / world) for r in range(world + 1)]
    bounds = np.asarray(lon[edges], dtype=np.float64)
    plans = []
    for r in range(world):
        lo = max(0, edges[r] - halo_cells)
        hi = min(nx - 1, edges[r + 1] + halo_cells)
        plans.append(dict(rank=r, bounds=bounds, lo=lo, hi=hi, xi_offset=lo, left_global=lo == 0, right_global=hi == nx - 1,
                          own_cells=(edges[r], edges[r + 1])))  # fmt: skip
    return plans


def column_slab_plan(nx_nodes: int, world: int, halo_cells: int) -> list[dict]:
    """Cut the cell columns 0 .. nx_nodes - 2 of a curvilinear grid into ``world`` slabs.

    Returns per rank: ``col_edges`` (world+1 cell-column edges, shared by all ranks: rank r owns the cells whose column i has
    col_edges[r] <= i < col_edges[r+1]), the inclusive local node-column range [lo, hi] = owned cells +- halo, ``xi_offset`` = lo,
    and whether each local edge is a global edge."""
    nx = int(nx_nodes)
    ncell = nx - 1
    if world > ncell:
        raise ValueError(f"cannot cut {ncell} cell columns into {world} slabs")
    edges = np.asarray([round(r * ncell / world) for r in range(world + 1)], dtype=np.int64)
    plans = []
    for r in range(world):
        lo = max(0, int(edges[r]) - halo_cells)
        hi = min(nx - 1, int(edges[r + 1]) + halo_cells)
        plans.append(dict(rank=r, col_edges=edges, lo=lo, hi=hi, xi_offset=lo, left_global=lo == 0, right_global=hi == nx - 1,
                          own_cells=(int(edges[r]), int(edges[r + 1]))))  # fmt: skip
    return plans


def route_counts(x, bounds) -> np.ndarray:
    """Host restatement of the device classify kernel: owner rank of each x (used by the CPU tests)."""
    b = np.asarray(bounds)
    return np.clip(np.searchsorted(b[1:-1], x, side="right"), 0, len(b) - 2)


class _SlabLevels:
    """The X-slab of a (T, Z, Y, X) array-like, cut ONE TIME LEVEL AT A TIME: what a time-windowed FieldSet indexes
    (``data[level]``).  The parent may be an ``np.memmap`` or any lazy loader -- a rank never reads another rank's columns."""

    def __init__(self, parent, sl: slice):
        self._parent, self._sl = parent, sl
        T, Z, Y, X = parent.shape
        self.shape = (T, Z, Y, len(range(*sl.indices(X))))
        self.dtype = np.dtype(parent.dtype)

    def __len__(self):
        return self.shape[0]

    def __getitem__(self, level):
        return np.ascontiguousarray(np.asarray(self._parent[level])[..., self._sl])


class DecomposedFieldSet:
    """This rank's X-slab of a rectilinear FieldSet, resident on ``device`` (``time_window=W``: only W time levels of it).
    ``interp_method`` and ``padding`` are those of ``FieldSet.from_arrays``: an A-grid with XLinear_Velocity ("linear"), XFreeslip,
    XPartialslip or nearest-node sampling, or a C-grid with CGrid_Velocity and its SGRID padding."""

    def __init__(self, *, lon, lat, U, V, W=None, depth=None, time=None, mesh="spherical", rank, world, halo_cells=4,
                 device=0, time_window=None, interp_method="linear", padding=("low", "low", "high")):  # fmt: skip
        from .fieldset import FieldSet

        if np.ndim(lon) != 1 or np.ndim(lat) != 1:
            raise NotImplementedError("domain decomposition cuts rectilinear grids (1-D lon / lat) into longitude slabs; on a "
                                      "curvilinear grid a slab is not a range of longitudes: use "
                                      "DecomposedFieldSet.from_curvilinear (column slabs)")  # fmt: skip
        self.rank, self.world, self.device = rank, world, device
        self.plan = slab_plan(lon, world, halo_cells)[rank]
        lo, hi = self.plan["lo"], self.plan["hi"]
        sl = slice(lo, hi + 1)
        if time_window is None:
            cut = lambda a: np.ascontiguousarray(np.asarray(a)[..., sl])  # noqa: E731
        else:
            cut = lambda a: _SlabLevels(a, sl)  # noqa: E731
        self.fs = FieldSet.from_arrays(lon=np.ascontiguousarray(np.asarray(lon)[sl]), lat=lat, depth=depth, time=time,
                                       U=cut(U), V=cut(V), W=None if W is None else cut(W), mesh=mesh, time_window=time_window,
                                       interp_method=interp_method, padding=padding,
                                       xdim=np.asarray(lon).size - 1)  # fmt: skip  (GLOBAL cell count: ei stays global)
        self._attach()

    def add_context(self, name, value):
        """``FieldSet.add_context`` (``dres``, ``RK45_tol``, ``RK45_min_dt``, ``RK45_max_dt``, ...)."""
        self.fs.add_context(name, value)

    @classmethod
    def from_curvilinear(cls, *, lon, lat, U, V, W=None, depth=None, time=None, mesh="spherical", rank, world, halo_cells=4, device=0,
                         time_window=None, interp_method="cgrid_velocity", padding=("low", "low", "high")):  # fmt: skip
        """This rank's COLUMN SLAB of a curvilinear FieldSet: ``lon`` / ``lat`` are the (ny, nx) node coordinates, U, V (, W) global
        (T, Z, Y, X) fields.  Every rank holds the whole horizontal grid -- coordinates, cell projections and the spatial hash,
        built exactly as on one GPU, so that every search finds the single-GPU cell -- and only the node columns of its owned
        cells +- ``halo_cells`` of the fields (``column_slab_plan``).  A particle is advanced by the rank that owns the column of
        the cell its search finds.  ``interp_method``: "cgrid_velocity" (CGrid_Velocity, SGRID ``padding``) or "linear"
        (XLinear_Velocity).  Grids whose faces overlap (duplicated wrap columns, a north fold) are not supported."""
        from .fieldset import FieldSet

        if np.ndim(lon) != 2 or np.ndim(lat) != 2:
            raise ValueError("from_curvilinear takes (ny, nx) node coordinates; rectilinear grids: DecomposedFieldSet(...)")
        plan = column_slab_plan(np.shape(lon)[1], world, halo_cells)[rank]
        sl = slice(plan["lo"], plan["hi"] + 1)
        if time_window is None:
            cut = lambda a: np.ascontiguousarray(np.asarray(a)[..., sl])  # noqa: E731
        else:
            cut = lambda a: _SlabLevels(a, sl)  # noqa: E731
        fs = FieldSet.from_arrays(lon=lon, lat=lat, depth=depth, time=time, U=cut(U), V=cut(V), W=None if W is None else cut(W),
                                  mesh=mesh, time_window=time_window, interp_method=interp_method, padding=padding)  # fmt: skip
        return cls.from_slab(fs, plan, rank=rank, world=world, device=device)

    @classmethod
    def from_slab(cls, fs, plan, *, rank, world, device):
        """Wrap a FieldSet that already holds ONLY this rank's slab, e.g. when every rank generates / reads just its own columns:
        on a rectilinear grid a slab of lon built with the GLOBAL ``xdim`` (``plan`` from ``slab_plan``), on a curvilinear grid
        the whole (ny, nx) lon / lat with fields of the node columns [lo, hi] (``plan`` from ``column_slab_plan``)."""
        self = cls.__new__(cls)
        self.rank, self.world, self.device, self.plan, self.fs = rank, world, device, plan, fs
        self._attach()
        return self

    @property
    def columns(self) -> bool:
        """Column slabs of a curvilinear grid (``from_curvilinear``)."""
        return "col_edges" in self.plan

    def add_field(self, name, data, interp_method="linear", time_window=None):
        """``FieldSet.add_field`` of a GLOBAL (T, Z, Y, X) field on the velocity grid (e.g. Kh_zonal / Kh_meridional of
        AdvectionDiffusionM1 / EM), cut to this rank's columns -- one time level at a time when it streams (``time_window``)."""
        if self.columns:
            raise NotImplementedError("column slabs of a curvilinear grid hold U, V and W only")
        sl = slice(self.plan["lo"], self.plan["hi"] + 1)
        slab = np.ascontiguousarray(np.asarray(data)[..., sl]) if time_window is None else _SlabLevels(data, sl)
        return self.fs.add_field(name, slab, interp_method=interp_method, time_window=time_window)

    def _attach(self):
        self.engine = self.fs.engine(self.device)
        if self.columns:
            self.engine.decomp_set_columns(self.world, self.rank, self.plan["col_edges"], self.plan["xi_offset"], self.plan["left_global"],
                                           self.plan["right_global"])  # fmt: skip
        else:
            self.engine.decomp_set(self.world, self.rank, self.plan["bounds"], self.plan["xi_offset"], self.plan["left_global"],
                                   self.plan["right_global"])  # fmt: skip


def _engine_memory_device(index: int):
    """torch device of the buffers handed to the engine's pack / unpack kernels: the engine's GPU.  (Where torch sees no CUDA
    device the engine can only be the host simulation of the test suite, oracle/hostsim, whose "device" memory is host memory.)"""
    import torch

    return torch.device(f"cuda:{index}") if torch.cuda.is_available() else torch.device("cpu")


def _sync(device):
    if device.type == "cuda":
        import torch

        torch.cuda.synchronize(device)


def _exchange(eng, counts, dist, device, resume=False):
    """One migration round: every rank's per-destination counts -> ONE all-gather (each rank then knows what it sends, what it
    receives and whether anybody moves at all) -> records packed on the device -> all_to_all -> unpack.
    Returns (#records moving on ALL ranks, #received here).  ``resume``: the engine carries each particle's resumable state
    (AdvectionRK45, AdvectionDiffusionM1 / EM): a second buffer of 24-byte records goes along, split like the records.

    NCCL: the count matrix and the records stay on the device (records never touch the host).  gloo (CPU tests / two
    ranks sharing one GPU): the same device-side pack/unpack kernels, records staged through the host."""
    import torch

    world = dist.get_world_size()
    rank = dist.get_rank()
    n_out = int(counts.sum())
    nccl = dist.get_backend() == "nccl"
    mine = torch.as_tensor(counts, dtype=torch.int64, device=device if nccl else "cpu")
    matrix = torch.empty(world * world, dtype=torch.int64, device=mine.device)  # [src * world + dst]
    dist.all_gather_into_tensor(matrix, mine)
    m = matrix.cpu().numpy().reshape(world, world)
    total = int(m.sum())
    if total == 0:
        return 0, 0
    rc = m[:, rank]
    n_in = int(rc.sum())
    sizes = (RECORD_BYTES, RESUME_BYTES) if resume else (RECORD_BYTES,)
    sendbufs = [torch.empty(max(n_out, 1) * b, dtype=torch.uint8, device=device) for b in sizes]
    if resume:
        eng.migrate_pack_resume(sendbufs[0].data_ptr(), sendbufs[1].data_ptr(), n_out)
    else:
        eng.migrate_pack(sendbufs[0].data_ptr(), n_out)  # synchronises the engine stream before NCCL touches the buffer
    if nccl:
        recvbufs = [torch.empty(max(n_in, 1) * b, dtype=torch.uint8, device=device) for b in sizes]
        for sendbuf, recvbuf, b in zip(sendbufs, recvbufs, sizes, strict=True):
            dist.all_to_all_single(recvbuf[: n_in * b], sendbuf[: n_out * b], output_split_sizes=[int(c) * b for c in rc],
                                   input_split_sizes=[int(c) * b for c in counts])  # fmt: skip
        _sync(device)
    else:
        recvbufs = []
        for sendbuf, b in zip(sendbufs, sizes, strict=True):
            host = sendbuf[: n_out * b].cpu().numpy()
            offs = np.concatenate(([0], np.cumsum(counts))) * b
            chunks = [host[offs[r] : offs[r + 1]].tobytes() for r in range(world)]
            everyone = [None] * world
            dist.all_gather_object(everyone, chunks)
            got = b"".join(everyone[src][rank] for src in range(world))
            assert len(got) == n_in * b
            recvbufs.append(torch.frombuffer(bytearray(got) if got else bytearray(b), dtype=torch.uint8).to(device))
        _sync(device)
    if resume:
        eng.migrate_unpack_resume(recvbufs[0].data_ptr(), recvbufs[1].data_ptr(), n_in)
    else:
        eng.migrate_unpack(recvbufs[0].data_ptr(), n_in)
    return total, n_in


def connect_p2p(dfs: DecomposedFieldSet, dist, capacity_records: int) -> bool:
    """Set up in-kernel migration over peer memory for ``dfs`` (every rank calls it): allocate the inbox, all-gather the CUDA-IPC
    handles, map the peers.  ``capacity_records``: arrivals one rank can take per round (a full inbox only delays the overflow by
    a round).  Returns True when EVERY rank is connected -- from then on ``run_decomposed_resident`` uses the peer-memory rounds;
    if any rank could not allocate or map (no peer access between two devices, IPC disabled in a container ...) all ranks agree
    to stay on the collective transport and the reason is kept in ``dfs.p2p_error``."""
    from ._lib import EngineError

    err, handle = "", b""
    try:
        handle, _ = dfs.engine.migrate_p2p_init(capacity_records)
    except EngineError as e:
        err = str(e)
    everyone = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, (handle, err))
    errors = [e for _, e in everyone if e]
    if not errors:
        try:
            dfs.engine.migrate_p2p_connect(handles=[h for h, _ in everyone])
        except EngineError as e:
            err = str(e)
    flags = [None] * dist.get_world_size()
    dist.all_gather_object(flags, err)
    errors += [e for e in flags if e]
    dfs.p2p = not errors
    dfs.p2p_error = errors[0] if errors else ""
    if errors:
        dfs.engine.p2p_disable()
    return dfs.p2p


def _carries_resume(plan) -> bool:
    """AdvectionRK45 and AdvectionDiffusionM1 / EM: a lane stopped mid-call continues on its new owner with its dt, next_dt and
    iteration count, which travel with the particle."""
    return plan.kind in ("rk45", "advdiff")


def _first_eval_hint(dfs, plan, first, slid) -> bool:
    """Column slabs: ``hint_all_zero`` of a round's launch -- the whole set's (``plan.hint_all_zero``, one all-reduce) where a
    launch of the single-GPU call would pass it.  AdvectionRK45 passes it to every launch (its lanes count their iterations across
    rounds and skip the hint at their first only); the fixed-step kernel, whose count restarts in every launch, gets it where a
    single-GPU launch starts: the call's first round and, on a time-windowed field, the first round after a slide."""
    if not dfs.columns or not plan.hint_all_zero:
        return False
    return plan.kind == "rk45" or first or slid


def _advect_args(eng, plan, dt, endtime, first, seed, rng_call, rounds, hint=False):
    """The arguments of a round's launch.  AdvectionDiffusionM1 / EM: the iteration count travels with the particle and keys its
    Wiener increments -- the single-GPU run's stream, unchanged by where the rounds cut the call (no round number in the call index).

    Fused DiffusionUniformKh: the Wiener increments are keyed by (seed; particle id, iteration of the launch, call index).  Every
    migration round is a new launch on every rank (the round count is global), so the round number joins the call index and no
    particle ever draws the same increment twice, wherever it migrates.  (The stream differs from a single-GPU run's, whose
    iterations are not cut into rounds: statistically equivalent, not bit-identical -- the advection-only path is.)
    The fixed-step kernel restarts its iteration count in every launch, so the first-evaluation time bit reaches the first
    iteration of every round.  That is the single-GPU rule: the bit changes a value only on the first time level (tau == 0), where
    a particle is before its first step -- a lane the first round only routed to its owner, or one that waited for the window."""
    if plan.kind == "fixed":
        rng_call = (int(rng_call) << 20) + rounds
    return plan.launch_args(eng, dt, endtime, seed=seed, rng_call=rng_call, resume=not first, batch_levels=plan.batch_levels,
                            hint_all_zero=hint, next_dt_dtype=plan.next_dt_dtype)  # fmt: skip


def _advect_round(dfs, args, sign):
    """One launch on the resident particles; with a time-windowed field the next level's H2D copy is started under the kernel."""
    eng = dfs.engine
    if dfs.fs.time_window is None:
        return eng.advect(args)
    eng.advect_async(args)
    dfs.fs.prefetch_next(dfs.device, sign)
    return eng.last_report()


def _slide_in_lockstep(dfs, rep, sign, dist, device) -> bool:
    """Time-windowed field, called after a round in which NO particle moved between ranks: every unfinished particle anywhere now
    waits for a time level that is not resident.  All ranks slide to the same window -- the one the earliest (latest, backward in
    time) waiting particle needs -- so that a particle that migrates later finds, on its new owner, the levels it left with.
    Returns False when nobody waits (the call is complete)."""
    import torch

    waits = rep["n_wait_window"] > 0
    t = (rep["wait_t_min"] if sign > 0 else -rep["wait_t_max"]) if waits else np.inf
    v = torch.tensor([t], dtype=torch.float64, device=device if dist.get_backend() == "nccl" else "cpu")
    dist.all_reduce(v, op=dist.ReduceOp.MIN)
    t = float(v.item())
    if not np.isfinite(t):
        return False
    w = dfs.fs._win[dfs.device]
    before = (w["first"], w["n"])
    dfs.fs.slide_window(dfs.device, sign * t, sign)
    if (w["first"], w["n"]) == before:
        raise RuntimeError(f"time window of {dfs.fs.time_window} levels cannot cover one step: widen time_window")
    return True


def run_decomposed_p2p(dfs: DecomposedFieldSet, plan, dt: float, endtime: float, dist, max_rounds=100000, seed=0, rng_call=1):
    """The rounds of one ``Kernel.execute`` with in-kernel migration: advect (leavers are delivered to their new owners by the
    kernel itself) -> all-reduce of (#movers, halo flag) = the barrier that orders every rank's kernel before anybody reads an
    inbox -> ``migrate_p2p_finish`` -> resume ... until nobody moved."""
    import time

    import torch

    eng = dfs.engine
    device = _engine_memory_device(dfs.device)
    sign = 1 if dt > 0 else -1
    stats = dict(rounds=0, migrated=0, particle_steps=0, kernel_ms=0.0, exchange_ms=0.0, transport="peer memory (in-kernel)")
    slid = False
    for _ in range(max_rounds):
        hint = _first_eval_hint(dfs, plan, stats["rounds"] == 0, slid)
        if dfs.columns and (stats["rounds"] == 0 or slid):
            _route_columns(dfs, plan, hint, dist, device, stats)
        rep = _advect_round(dfs, _advect_args(eng, plan, dt, endtime, stats["rounds"] == 0, seed, rng_call, stats["rounds"], hint), sign)
        stats["max_iters_done"] = max(stats.get("max_iters_done", 0), rep["max_iters_done"])
        t0 = time.perf_counter()
        flags = torch.tensor([float(rep["n_migrate"]), float(rep["max_state"] == 99)], dtype=torch.float64,
                             device=device if dist.get_backend() == "nccl" else "cpu")
        dist.all_reduce(flags, op=dist.ReduceOp.SUM)
        moved, halo = (int(v) for v in flags.cpu().tolist())
        eng.migrate_p2p_finish()
        stats["exchange_ms"] += 1e3 * (time.perf_counter() - t0)
        stats["rounds"] += 1
        stats["migrated"] += int(rep["n_migrate"])
        stats["particle_steps"] += rep["particle_steps"]
        stats["kernel_ms"] += rep["kernel_ms"]
        if halo:
            stats["halo_violation"] = True
            raise RuntimeError("halo violation: a stage position left the owned+halo columns; increase halo_cells or reduce dt")
        slid = moved == 0
        if moved == 0 and not (dfs.fs.time_window is not None and _slide_in_lockstep(dfs, rep, sign, dist, device)):
            break
    _finish_call(dfs, plan, dt, endtime, dist, device, stats)
    return stats


def _route_columns(dfs, plan, hint, dist, device, stats):
    """Column slabs: the set goes to the owners of its cells, with the hint rule of the coming launch, before a launch that skips
    the hint at the first evaluation (the call's first and, time-windowed, the first after a slide).  A lane the kernel delivered
    before that evaluation would arrive where the next launch no longer skips the hint, as the single-GPU launch does."""
    counts = dfs.engine.migrate_classify_columns(hint)
    _exchange(dfs.engine, counts, dist, device, resume=_carries_resume(plan))
    stats["migrated"] += int(counts.sum())


def _finish_call(dfs, plan, dt, endtime, dist, device, stats):
    """AdvectionRK45: the batch-level dt clamp of the particles that left the loop early needs the call's iteration count over
    every rank and round -- once, on every rank, after the last round."""
    if plan.kind == "rk45":
        dfs.engine.rk45_finalize(dt, endtime, int(allreduce_max(stats.get("max_iters_done", 0), dist, _collective_device(dist, device))))


def _collective_device(dist, device):
    return device if dist.get_backend() == "nccl" else "cpu"


def run_decomposed_resident(dfs: DecomposedFieldSet, plan, dt: float, endtime: float, dist, max_rounds=100000, seed=0, rng_call=1):
    """The rounds of one ``Kernel.execute`` over a domain-decomposed field on the particles RESIDENT in the rank's engine (uploaded
    with ``upload_decomposed`` or restored from a snapshot): advect until every particle reached ``endtime`` or left the slab ->
    classify / count -> exchange -> resume ... until nobody moves.  Nothing crosses PCIe except the count matrix.  Returns stats."""
    import time

    if getattr(dfs, "p2p", False):
        return run_decomposed_p2p(dfs, plan, dt, endtime, dist, max_rounds=max_rounds, seed=seed, rng_call=rng_call)
    eng = dfs.engine
    device = _engine_memory_device(dfs.device)
    sign = 1 if dt > 0 else -1
    stats = dict(rounds=0, migrated=0, particle_steps=0, kernel_ms=0.0, exchange_ms=0.0, transport="collectives (all_to_all_single)")
    first = True
    rep = None
    for _ in range(max_rounds):
        t0 = time.perf_counter()
        # (column slabs: by the column of the cell each particle's next search finds, with the hint rule of the next launch)
        counts = eng.migrate_classify_columns(_first_eval_hint(dfs, plan, first, False)) if dfs.columns else eng.migrate_count()
        total, _ = _exchange(eng, counts, dist, device, resume=_carries_resume(plan))
        stats["exchange_ms"] += 1e3 * (time.perf_counter() - t0)
        stats["migrated"] += int(counts.sum())
        slid = total == 0 and not first
        if slid and not (dfs.fs.time_window is not None and _slide_in_lockstep(dfs, rep, sign, dist, device)):
            break
        hint = _first_eval_hint(dfs, plan, first, slid)
        if dfs.columns and slid:  # (the count above used the rule of a launch that does not skip the hint)
            _route_columns(dfs, plan, hint, dist, device, stats)
        rep = _advect_round(dfs, _advect_args(eng, plan, dt, endtime, first, seed, rng_call, stats["rounds"], hint), sign)
        first = False
        stats["rounds"] += 1
        stats["particle_steps"] += rep["particle_steps"]
        stats["kernel_ms"] += rep["kernel_ms"]
        stats["max_iters_done"] = max(stats.get("max_iters_done", 0), rep["max_iters_done"])
        if rep["max_state"] == 99:  # every rank raises in the same round or the next count exchange would hang: agree first
            stats["halo_violation"] = True
        if allreduce_max(float(rep["max_state"] == 99), dist, device) > 0:
            raise RuntimeError("halo violation: a stage position left the owned+halo columns; increase halo_cells or reduce dt")
    _finish_call(dfs, plan, dt, endtime, dist, device, stats)
    return stats


def decomposed_plan(dfs: DecomposedFieldSet, kernels, pdata: dict | None = None):
    """The kernel list lowered for mode D: one of the fused fixed-step schemes (optionally with DiffusionUniformKh),
    ``[AdvectionRK45, DeleteParticle]`` (``pdata`` must then hold ``next_dt``) or ``[AdvectionDiffusionM1 | EM, DeleteParticle]``."""
    # (the particle variables stand in for the ParticleClass: RK45 needs next_dt)
    pclass = SimpleNamespace(variables=[SimpleNamespace(name=k, dtype=v.dtype) for k, v in (pdata or {}).items()])
    plan = KernelPlan(kernels, dfs.fs, pclass)
    if plan.stepwise:
        raise NotImplementedError("domain-decomposed execution runs one built-in kernel -- a fixed-step advection scheme (optionally "
                                  "with DiffusionUniformKh), AdvectionRK45 or AdvectionDiffusionM1 / EM -- followed by DeleteParticle; "
                                  "user kernels and other mixes run on one GPU")  # fmt: skip
    if not plan.delete_on_error:
        raise NotImplementedError("domain-decomposed execution needs the DeleteParticle handler (errors cannot be replayed "
                                  "step-exactly across ranks)")  # fmt: skip
    return plan


def upload_decomposed(dfs: DecomposedFieldSet, pdata: dict, dt: float, plan=None):
    """Make ``pdata`` this rank's resident set.  AdvectionRK45 keeps every particle's dt and next_dt (the reference never resets dt
    in RK45 mode); the kernels that continue a lane on another rank get their resumable-state columns."""
    from .statuscodes import StatusCode

    pdata["state"][:] = StatusCode.Evaluate
    rk45 = plan is not None and plan.kind == "rk45"
    if not rk45:
        pdata["dt"][:] = dt
    dfs.engine.upload_particles(pdata, np.ascontiguousarray(pdata["ei"][:, -1]))
    if plan is not None and _carries_resume(plan):
        dfs.engine.upload_resume(len(pdata["x"]), dt=pdata["dt"] if rk45 else None, next_dt=pdata["next_dt"] if rk45 else None)


def download_decomposed(dfs: DecomposedFieldSet, dt: float, ngrids=1, plan=None) -> dict:
    """This rank's resident set (deleted particles dropped); with AdvectionRK45 each particle's own dt and next_dt."""
    from .statuscodes import StatusCode

    out = dfs.engine.download_all(ngrids=ngrids)
    if plan is not None and plan.kind == "rk45":
        out["dt"][:], ndt, _ = dfs.engine.download_resume(len(out["x"]))
        out["next_dt"] = ndt.astype(plan.next_dt_dtype)
    else:
        out["dt"][:] = dt
    keep = out["state"] != StatusCode.Delete
    return {k: v[keep] for k, v in out.items()}


def _global_batch_facts(dfs, pdata, dt, endtime, dist, device) -> tuple[bool, int]:
    """The reference's batch-level decisions of the call's first evaluation (plan.batch_facts) over the WHOLE set -- every rank's
    shard, one all-reduce: ``hint_all_zero`` (curvilinear grids: every evaluated particle's hinted xi is 0) and the batch-level bits
    -- so that the first-iteration rules of the kernels are the single-GPU ones."""
    import torch

    hint_all_zero, bits = batch_facts(dfs.fs, pdata, pdata["ei"][:, -1], dt, endtime)
    v = torch.tensor([float(bits & 1), float(bits & 2), float(not hint_all_zero)], dtype=torch.float64,
                     device=_collective_device(dist, device))  # fmt: skip
    dist.all_reduce(v, op=dist.ReduceOp.MAX)
    return v[2].item() == 0, int(v[0].item() > 0) | (2 if v[1].item() > 0 else 0)


def execute_decomposed(dfs: DecomposedFieldSet, pdata: dict, kernels, dt: float, endtime: float, dist, max_rounds=100000, seed=0,
                       rng_call=1):
    """``Kernel.execute`` over a domain-decomposed field: ``pdata`` is ANY shard of the particle set (it is
    routed to the owners first).  Returns (local particle dict after the call, stats)."""
    plan = decomposed_plan(dfs, kernels, pdata)
    upload_decomposed(dfs, pdata, dt, plan)
    if dfs.columns and allreduce_sum(len(pdata["x"]), dist, _collective_device(dist, _engine_memory_device(dfs.device))) == 1:
        # (a set of one particle is its own batch for the reference's `if np.any(xi)` at every evaluation: a rule of the whole set
        #  that the engine of a shard does not apply)
        raise NotImplementedError("a particle set of ONE particle on a curvilinear grid runs on one GPU, not on column slabs")
    if _carries_resume(plan) or dfs.fs.interp_method != "linear" or dfs.columns:  # (rectilinear fixed-step XLinear_Velocity: 0)
        plan.hint_all_zero, plan.batch_levels = _global_batch_facts(dfs, pdata, dt, endtime, dist, _engine_memory_device(dfs.device))
    if dfs.fs.time_window is not None:
        # first window: where the earliest (latest, backward in time) particle of ANY rank starts -- the same on every rank
        import torch

        sign = 1 if dt > 0 else -1
        todo = evaluated_mask(pdata, dt, endtime)
        t0 = float((sign * pdata["t"][todo]).min()) if todo.any() else np.inf
        device = _engine_memory_device(dfs.device)
        v = torch.tensor([t0], dtype=torch.float64, device=device if dist.get_backend() == "nccl" else "cpu")
        dist.all_reduce(v, op=dist.ReduceOp.MIN)
        if np.isfinite(float(v.item())):
            dfs.fs.slide_window(dfs.device, sign * float(v.item()), sign)
    stats = run_decomposed_resident(dfs, plan, dt, endtime, dist, max_rounds=max_rounds, seed=seed, rng_call=rng_call)
    return download_decomposed(dfs, dt, ngrids=pdata["ei"].shape[1], plan=plan), stats
