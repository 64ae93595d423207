"""Thin Python wrapper of one ``pb_engine`` (one per GPU).  Plumbing only: every call below is
a ctypes call into ``libparcels_b200.so``; all compute happens in the CUDA kernels."""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import AdvectArgs, Report, check, ptr


def _report_dict(r: Report) -> dict:
    return {name: getattr(r, name) for name, _ in Report._fields_ if not name.startswith("reserved")}


# the resident particle columns in the order of the C-ABI's particle arguments (pb_particles_upload, pb_particle_arrays);
# "ei" is the engine's one column: the last grid's
PARTICLE_COLUMNS = ("x", "y", "z", "dx", "dy", "dz", "t", "state", "ei", "particle_id")
_PARTICLE_DTYPES = {"x": np.float32, "y": np.float32, "z": np.float32, "t": np.float64, "state": np.int32}


def _check_particle_dtypes(d: dict):
    for k, dt in _PARTICLE_DTYPES.items():
        if d[k].dtype != dt:
            raise TypeError(f"particle variable {k!r} must be {np.dtype(dt).name} (default Particle), got {d[k].dtype}")


def _column_ptrs(d: dict, ei_last: np.ndarray, names=PARTICLE_COLUMNS) -> list:
    return [ptr(ei_last if k == "ei" else d[k]) for k in names]


class Engine:
    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = C.c_void_p()
        check(self._lib.pb_engine_create(int(device), C.byref(h)))
        self._h = h
        self.device = int(device)
        self._keep = []  # device tensors attached by pointer must outlive the engine's use
        self._owner = None  # weakref to the ParticleSet whose particles are resident in this engine's SoA

    def claim(self, pset):
        """The engine holds ONE resident particle SoA.  Before another ParticleSet uploads into it, the set that was
        resident brings its host arrays up to date (its only copy may live here after a lazy execute()) and forgets
        that the device mirrors it -- every ParticleSet on a FieldSet keeps independent data, as in the reference."""
        import weakref

        prev = self._owner() if self._owner is not None else None
        if prev is not None and prev is not pset:
            prev._release_device()
        if prev is not pset:
            self._owner = weakref.ref(pset)

    def owned_by(self, pset) -> bool:
        return self._owner is not None and self._owner() is pset

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pb_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- grid / fields -------------------------------------------------------------------------
    def upload_rectilinear_grid(self, lon, lat, depth, time_s, spherical, deg2m, xdim, ydim, zdim):
        lon = np.ascontiguousarray(lon)
        cdt = lon.dtype
        if cdt not in (np.float32, np.float64):
            raise TypeError(f"grid coordinates must be float32 or float64, got {cdt}")
        lat = np.ascontiguousarray(lat)
        if lat.dtype != cdt or (depth is not None and np.asarray(depth).dtype != cdt):
            raise TypeError("lon, lat and depth must share one dtype (the reference's arithmetic promotes on it)")
        depth = None if depth is None else np.ascontiguousarray(depth)
        time_s = None if time_s is None else np.ascontiguousarray(time_s, dtype=np.float64)
        check(
            self._lib.pb_grid_upload_rectilinear(
                self._h, ptr(lon), lon.size, ptr(lat), lat.size, ptr(depth), 0 if depth is None else depth.size,
                int(cdt == np.float64), ptr(time_s), 0 if time_s is None else time_s.size, int(bool(spherical)),
                float(deg2m), int(xdim), int(ydim), int(zdim or 0),
            )
        )  # fmt: skip

    def upload_curvilinear_grid(self, lon2d, lat2d, depth, time_s, spherical, deg2m, xdim, ydim, zdim, h: dict):
        lon2d = np.ascontiguousarray(lon2d)
        cdt = lon2d.dtype
        if cdt not in (np.float32, np.float64):
            raise TypeError(f"grid coordinates must be float32 or float64, got {cdt}")
        lat2d = np.ascontiguousarray(lat2d)
        if lat2d.dtype != cdt or (depth is not None and np.asarray(depth).dtype != cdt):
            raise TypeError("lon, lat and depth must share one dtype (the reference's arithmetic promotes on it)")
        depth = None if depth is None else np.ascontiguousarray(depth)
        time_s = None if time_s is None else np.ascontiguousarray(time_s, dtype=np.float64)
        ny, nx = lon2d.shape
        if "keys" in h:  # host-built table (parcels_b200/spatialhash.py, table=True)
            keys = np.ascontiguousarray(h["keys"], dtype=np.uint32)
            starts = np.ascontiguousarray(h["starts"], dtype=np.int64)
            counts = np.ascontiguousarray(h["counts"], dtype=np.int64)
            faces = np.ascontiguousarray(h["faces"], dtype=np.uint32)
            nk, ne = keys.size, faces.size
        else:  # only the quantised boxes: the table is built on the device (csrc/hashbuild.cu)
            keys = starts = counts = faces = None
            nk = ne = 0
        box = np.ascontiguousarray(h["box"], dtype=np.float64)
        qbox = np.ascontiguousarray(h["qbox"], dtype=np.uint64)
        assert qbox.size == (ny - 1) * (nx - 1)
        check(
            self._lib.pb_grid_upload_curvilinear(
                self._h, ptr(lon2d), ptr(lat2d), ny, nx, ptr(depth), 0 if depth is None else depth.size,
                int(cdt == np.float64), ptr(time_s), 0 if time_s is None else time_s.size, int(bool(spherical)),
                float(deg2m), int(xdim), int(ydim), int(zdim or 0), ptr(keys), ptr(starts), ptr(counts), nk,
                ptr(faces), ne, ptr(box), int(h["bitwidth"]), ptr(qbox),
            )
        )  # fmt: skip

    def hash_table(self) -> dict:
        """The spatial-hash table resident on the device (keys, starts, counts, faces), read back."""
        nk, ne = C.c_int64(), C.c_int64()
        check(self._lib.pb_hash_table_size(self._h, C.byref(nk), C.byref(ne)))
        keys, faces = np.empty(nk.value, dtype=np.uint32), np.empty(ne.value, dtype=np.uint32)
        starts, counts = np.empty(nk.value, dtype=np.int64), np.empty(nk.value, dtype=np.int64)
        check(self._lib.pb_hash_table_download(self._h, ptr(keys), ptr(starts), ptr(counts), ptr(faces)))
        return dict(keys=keys, starts=starts, counts=counts, faces=faces)

    def set_interpolation(self, method: int, off_x: int, off_y: int, off_z: int):
        check(self._lib.pb_set_interpolation(self._h, int(method), int(off_x), int(off_y), int(off_z)))

    def upload_field(self, slot: int, data):
        data = np.asarray(data)
        if data.ndim != 4:
            raise ValueError("field data must be laid out (T, Z, Y, X)")
        if data.dtype not in (np.float32, np.float64):
            raise TypeError(f"field data must be float32 or float64, got {data.dtype}")
        data = np.ascontiguousarray(data)
        T, Z, Y, X = data.shape
        check(self._lib.pb_field_upload(self._h, slot, ptr(data), int(data.dtype == np.float64), T, Z, Y, X))

    def window_create(self, slot: int, dtype, shape, window_levels: int):
        T, Z, Y, X = shape
        check(self._lib.pb_field_window_create(self._h, slot, int(np.dtype(dtype) == np.float64), T, Z, Y, X, int(window_levels)))

    def window_load(self, slot: int, level: int, level_data: np.ndarray):
        level_data = np.ascontiguousarray(level_data)
        # the copy is asynchronous for pinned memory: keep the last few host buffers alive until it has run
        self._level_keepalive = (getattr(self, "_level_keepalive", []) + [level_data])[-16:]
        check(self._lib.pb_field_window_load(self._h, slot, int(level), ptr(level_data)))

    def window_set(self, first_level: int, n_levels: int):
        check(self._lib.pb_field_window_set(self._h, int(first_level), int(n_levels)))

    def attach_field_device(self, slot: int, dev_ptr: int, is_f64: bool, shape, keepalive=None):
        T, Z, Y, X = shape
        check(self._lib.pb_field_attach_device(self._h, slot, C.c_void_p(dev_ptr), int(is_f64), T, Z, Y, X))
        self._keep.append(keepalive)

    def clear_field(self, slot: int):
        check(self._lib.pb_field_clear(self._h, slot))

    # -- particles -----------------------------------------------------------------------------
    def upload_particles(self, d: dict, ei_last: np.ndarray):
        n = d["x"].shape[0]
        _check_particle_dtypes(d)
        check(self._lib.pb_particles_upload(self._h, n, *_column_ptrs(d, ei_last)))

    def download_particles(self, d: dict, ei_last: np.ndarray):
        n = d["x"].shape[0]
        check(self._lib.pb_particles_download(self._h, n, *_column_ptrs(d, ei_last, PARTICLE_COLUMNS[:-1])))  # (ids: download_ids)

    def download_ids(self, particle_id: np.ndarray):
        check(self._lib.pb_particles_download_ids(self._h, particle_id.shape[0], ptr(particle_id)))

    # -- output path (device-side ParticleFile.write selection, ordered compaction) -----------------
    OUTPUT_COLUMNS = {"x": np.float32, "y": np.float32, "z": np.float32, "t": np.float64, "particle_id": np.int64}

    def output_select(self, t_out: float, dt: float) -> int:
        m = C.c_int64()
        check(self._lib.pb_output_select(self._h, float(t_out), float(dt), C.byref(m)))
        return int(m.value)

    def output_gather(self, n_selected: int, columns=("x", "y", "z", "t", "particle_id"), with_index=False) -> dict:
        out = {k: np.empty(n_selected, dtype=self.OUTPUT_COLUMNS[k]) for k in columns}
        idx = np.empty(n_selected, dtype=np.int64) if with_index else None
        p = lambda k: ptr(out[k]) if k in out else None  # noqa: E731
        check(self._lib.pb_output_gather(self._h, n_selected, None if idx is None else ptr(idx), p("x"), p("y"), p("z"), p("t"),
                                         p("particle_id")))  # fmt: skip
        if with_index:
            out["index"] = idx
        return out

    def remove_deleted(self) -> int:
        m = C.c_int64()
        check(self._lib.pb_particles_remove_deleted(self._h, C.byref(m)))
        return int(m.value)

    def snapshot(self):
        check(self._lib.pb_particles_snapshot(self._h))

    def restore(self):
        check(self._lib.pb_particles_restore(self._h))

    def synchronize(self):
        check(self._lib.pb_engine_synchronize(self._h))

    def timer_begin(self):
        check(self._lib.pb_timer_begin(self._h))

    def timer_end_ms(self) -> float:
        ms = C.c_float()
        check(self._lib.pb_timer_end_ms(self._h, C.byref(ms)))
        return float(ms.value)

    # -- hot path --------------------------------------------------------------------------------
    @staticmethod
    def make_args(scheme, dt, endtime, *, diffusion=False, delete_on_error=False, kh=(0.0, 0.0), kh_spherical=False,
                  kh_deg2m=1.0, seed=0, rng_call=0, max_iters=-1, hint_all_zero=False, resume=False, kernels_only=False,
                  batch_levels=0) -> AdvectArgs:  # fmt: skip
        return AdvectArgs(int(scheme), int(diffusion), int(delete_on_error), int(kh_spherical), float(dt), float(endtime),
                          float(kh[0]), float(kh[1]), float(kh_deg2m), int(seed), int(rng_call), int(max_iters),
                          int(bool(hint_all_zero)), int(bool(resume)), int(bool(kernels_only)), int(batch_levels))  # fmt: skip

    def advect(self, args) -> dict:
        """``Kernel.execute`` on the device: ``args`` from :meth:`make_args` (pb_advect), :meth:`make_advdiff_args`
        (pb_advect_diffusion: AdvectionDiffusionM1 / EM) or :meth:`make_rk45_args` (pb_advect_rk45_resident_async: AdvectionRK45 on
        the resident dt / next_dt / iteration columns)."""
        from ._lib import AdvDiffArgs, Rk45Args

        rep = Report()
        if isinstance(args, AdvDiffArgs):
            check(self._lib.pb_advect_diffusion(self._h, C.byref(args), C.byref(rep)))
        elif isinstance(args, Rk45Args):
            check(self._lib.pb_advect_rk45_resident_async(self._h, C.byref(args)))
            check(self._lib.pb_last_report(self._h, C.byref(rep)))
        else:
            check(self._lib.pb_advect(self._h, C.byref(args), C.byref(rep)))
        return _report_dict(rep)

    @staticmethod
    def make_rk45_args(dt, endtime, tol, min_dt, max_dt, *, next_dt_is_f32=True, delete_on_error=False, max_iters=-1, kernels_only=False,
                       resume=False, hint_all_zero=False, batch_levels=0):  # fmt: skip
        from ._lib import Rk45Args

        return Rk45Args(float(dt), float(endtime), float(tol), float(min_dt), float(max_dt), int(max_iters), int(next_dt_is_f32),
                        int(delete_on_error), int(bool(kernels_only)), int(bool(resume)), int(bool(hint_all_zero)),
                        int(batch_levels))  # fmt: skip

    def rk45_finalize(self, dt, endtime, total_iters):
        """The batch-level dt clamp of the particles that left the RK45 loop before the call's ``total_iters`` iterations
        (pb_rk45_finalize_resident), once after the last launch of a call on the resident columns."""
        check(self._lib.pb_rk45_finalize_resident(self._h, float(dt), float(endtime), int(total_iters)))

    def upload_resume(self, n, dt=None, next_dt=None, iters=None):
        """Make each particle's resumable state -- dt, next_dt (float64), iteration count (int32) -- resident columns (None: zeros)."""
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=dt_) for a, dt_ in ((dt, np.float64), (next_dt, np.float64),
                                                                                        (iters, np.int32))]  # fmt: skip
        check(self._lib.pb_particles_upload_resume(self._h, int(n), *(ptr(a) for a in arrs)))

    def download_resume(self, n) -> tuple:
        dt, ndt, it = np.empty(n, dtype=np.float64), np.empty(n, dtype=np.float64), np.empty(n, dtype=np.int32)
        check(self._lib.pb_particles_download_resume(self._h, int(n), ptr(dt), ptr(ndt), ptr(it)))
        return dt, ndt, it

    @staticmethod
    def make_advdiff_args(scheme, dt, endtime, *, kh_slots, dres, deg2m_sq, delete_on_error=False, seed=0, rng_call=0, max_iters=-1,
                          kernels_only=False, resume=False, batch_levels=0):
        from ._lib import AdvDiffArgs

        return AdvDiffArgs(int(scheme), int(delete_on_error), int(kh_slots[0]), int(kh_slots[1]), float(dt), float(endtime),
                           float(dres), float(deg2m_sq), int(seed), int(rng_call), int(max_iters), int(bool(kernels_only)),
                           int(bool(resume)), int(batch_levels), 0)  # fmt: skip

    def advect_rk45(self, args, dt_arr, next_dt_arr) -> dict:
        """AdvectionRK45 + Repeat / next_dt state machine (``args`` from :meth:`make_rk45_args`); ``dt_arr`` / ``next_dt_arr``
        (float64, C-contiguous) are updated in place to what the reference leaves in particles.dt / particles.next_dt."""
        rep = Report()
        check(self._lib.pb_advect_rk45(self._h, C.byref(args), ptr(dt_arr), ptr(next_dt_arr), C.byref(rep)))
        return _report_dict(rep)

    def advect_host(self, args: AdvectArgs, d: dict, ei_last: np.ndarray, *, download: bool, n_chunks: int) -> dict:
        """pb_advect_host: upload + start-of-interval snapshot + Kernel.execute (+ download into the same arrays), pipelined
        chunk by chunk so that the copies run under the kernels."""
        from ._lib import ParticleArrays

        n = d["x"].shape[0]
        _check_particle_dtypes(d)
        h = ParticleArrays(*(C.cast(p, C.c_void_p) for p in _column_ptrs(d, ei_last)))
        rep = Report()
        check(self._lib.pb_advect_host(self._h, C.byref(args), n, C.byref(h), int(bool(download)), int(n_chunks), C.byref(rep)))
        return _report_dict(rep)

    def advect_async(self, args):
        """:meth:`advect` without waiting for the kernel; :meth:`last_report` waits and returns the report."""
        from ._lib import AdvDiffArgs, Rk45Args

        if isinstance(args, AdvDiffArgs):
            check(self._lib.pb_advect_diffusion_async(self._h, C.byref(args)))
        elif isinstance(args, Rk45Args):
            check(self._lib.pb_advect_rk45_resident_async(self._h, C.byref(args)))
        else:
            check(self._lib.pb_advect_async(self._h, C.byref(args)))

    def last_report(self) -> dict:
        rep = Report()
        check(self._lib.pb_last_report(self._h, C.byref(rep)))
        return _report_dict(rep)

    def sample_velocity(self, t, z, y, x, *, three_d, positions_are_f32=False, ei_hint=None, no_hint=False):
        t, z, y, x = (np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), np.shape(x)).ravel()) for a in (t, z, y, x))
        n = x.size
        u, v, w = (np.empty(n, dtype=np.float64) for _ in range(3))
        ei = np.empty(n, dtype=np.int32)
        st = np.empty(n, dtype=np.int32)
        hint = None if ei_hint is None else np.ascontiguousarray(ei_hint, dtype=np.int32)
        check(self._lib.pb_sample_velocity(self._h, n, ptr(t), ptr(z), ptr(y), ptr(x), int(positions_are_f32), int(three_d),
                                           ptr(hint), int(no_hint), ptr(u), ptr(v), ptr(w), ptr(ei), ptr(st)))  # fmt: skip
        return u, v, w, ei, st

    SCALAR_METHODS = {"linear": 0, "nearest": 1, "cgrid_tracer": 2, "linear_invdist_land": 3}  # enum pb_scalar_interp

    def sample_scalar(self, slot, method, t, z, y, x, *, positions_are_f32=False, ei_hint=None):
        """One ``Field.eval`` per sample on the device -> (value, ei, state); ``value`` has the dtype NumPy's
        promotion gives the reference's result (float32 only if every sample's arithmetic is float32)."""
        t, z, y, x = (np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), np.shape(x)).ravel()) for a in (t, z, y, x))
        n = x.size
        val = np.empty(n, dtype=np.float64)
        f32 = np.empty(n, dtype=np.int32)
        ei = np.empty(n, dtype=np.int32)
        st = np.empty(n, dtype=np.int32)
        hint = None if ei_hint is None else np.ascontiguousarray(ei_hint, dtype=np.int32)
        check(self._lib.pb_sample_scalar(self._h, int(slot), self.SCALAR_METHODS[method], n, ptr(t), ptr(z), ptr(y), ptr(x),
                                         int(positions_are_f32), ptr(hint), ptr(val), ptr(f32), ptr(ei), ptr(st)))  # fmt: skip
        if n and f32.all():
            val = val.astype(np.float32)
        return val, ei, st

    # -- mode D: domain decomposition + migration ------------------------------------------------------
    def decomp_set(self, nranks, rank, bounds, xi_offset, left_is_global, right_is_global):
        b = np.ascontiguousarray(bounds, dtype=np.float64)
        assert b.size == nranks + 1
        self._nranks = int(nranks)
        check(self._lib.pb_decomp_set(self._h, int(nranks), int(rank), ptr(b), int(xi_offset), int(left_is_global),
                                      int(right_is_global)))  # fmt: skip

    def decomp_set_columns(self, nranks, rank, col_edges, xi_offset, left_is_global, right_is_global):
        """Column slabs of a curvilinear grid (pb_decomp_set_columns): ``col_edges`` are the nranks + 1 cell-column edges."""
        c = np.ascontiguousarray(col_edges, dtype=np.int64)
        assert c.size == nranks + 1
        self._nranks = int(nranks)
        check(self._lib.pb_decomp_set_columns(self._h, int(nranks), int(rank), ptr(c), int(xi_offset), int(left_is_global),
                                              int(right_is_global)))  # fmt: skip

    def migrate_count(self) -> np.ndarray:
        counts = np.zeros(self._nranks, dtype=np.int64)
        check(self._lib.pb_migrate_count(self._h, ptr(counts)))
        return counts

    def migrate_classify_columns(self, no_hint: bool) -> np.ndarray:
        """``migrate_count`` of column slabs: leavers per rank by the column of the cell each particle's next search finds."""
        counts = np.zeros(self._nranks, dtype=np.int64)
        check(self._lib.pb_migrate_classify_columns(self._h, int(bool(no_hint)), ptr(counts)))
        return counts

    def memory_bytes(self) -> tuple[int, int]:
        """(grid bytes, field bytes) the engine holds on its device."""
        g, f = np.zeros(1, dtype=np.int64), np.zeros(1, dtype=np.int64)
        check(self._lib.pb_memory_bytes(self._h, ptr(g), ptr(f)))
        return int(g[0]), int(f[0])

    def migrate_pack(self, sendbuf_ptr: int, capacity_records: int):
        check(self._lib.pb_migrate_pack(self._h, C.c_void_p(sendbuf_ptr), int(capacity_records)))

    def migrate_unpack(self, recvbuf_ptr: int, n_in: int):
        check(self._lib.pb_migrate_unpack(self._h, C.c_void_p(recvbuf_ptr), int(n_in)))

    # the same with the resumable state resident: a second buffer of 24-byte records at the same indices
    def migrate_pack_resume(self, sendbuf_ptr: int, resume_ptr: int, capacity_records: int):
        check(self._lib.pb_migrate_pack_resume(self._h, C.c_void_p(sendbuf_ptr), C.c_void_p(resume_ptr), int(capacity_records)))

    def migrate_unpack_resume(self, recvbuf_ptr: int, resume_ptr: int, n_in: int):
        check(self._lib.pb_migrate_unpack_resume(self._h, C.c_void_p(recvbuf_ptr), C.c_void_p(resume_ptr), int(n_in)))

    # in-kernel migration over peer memory (pb_migrate_p2p_*, include/parcels_b200.h)
    def migrate_p2p_init(self, capacity_records: int):
        """Allocate this engine's inbox.  Returns (64-byte CUDA-IPC handle, device address of the inbox)."""
        handle = np.zeros(64, dtype=np.uint8)
        base = np.zeros(1, dtype=np.uint64)
        check(self._lib.pb_migrate_p2p_init(self._h, int(capacity_records), ptr(handle), ptr(base)))
        return handle.tobytes(), int(base[0])

    def migrate_p2p_connect(self, handles=None, local_bases=None):
        """handles: one 64-byte IPC handle per rank (peers in other processes); local_bases: inbox addresses of peers that live
        in this process (0 = not local)."""
        h = None if handles is None else np.frombuffer(b"".join(handles), dtype=np.uint8).copy()
        b = None if local_bases is None else np.ascontiguousarray(local_bases, dtype=np.uint64)
        assert (h is None or h.size == 64 * self._nranks) and (b is None or b.size == self._nranks)
        check(self._lib.pb_migrate_p2p_connect(self._h, ptr(h), ptr(b)))
        self.p2p = True

    def p2p_disable(self):
        """Leave the peer-memory transport (some rank could not connect): the kernels stop delivering by themselves."""
        check(self._lib.pb_migrate_p2p_disable(self._h))
        self.p2p = False

    def migrate_p2p_finish(self):
        """After the barrier of a round: drop what left, append what arrived.  Returns (arrivals, resident count)."""
        out = np.zeros(2, dtype=np.int64)
        check(self._lib.pb_migrate_p2p_finish(self._h, ptr(out[0:1]), ptr(out[1:2])))
        return int(out[0]), int(out[1])

    def particle_count(self) -> int:
        return int(self._lib.pb_particles_count(self._h))

    def download_all(self, ngrids=1) -> dict:
        """Download the resident particle set (its size may have changed through migration)."""
        from .particle import _CORE, create_particle_data

        n = self.particle_count()
        if n < (1 << 16):
            d = create_particle_data(nparticles=n, ngrids=ngrids, initial={})
        else:  # every column below is overwritten by the download: no initial-value fills (11 passes over a large set)
            d = {name: np.empty(n, dtype=dt) for name, dt in _CORE}
            d["dt"][:] = 1.0  # (the caller sets the nominal dt)
            d["ei"] = np.zeros((n, ngrids), dtype=np.int32) if ngrids > 1 else np.empty((n, 1), dtype=np.int32)
        if ngrids == 1:
            ei_last = d["ei"][:, 0]  # contiguous: the download writes the column in place
            self.download_particles(d, ei_last)
        else:
            ei_last = np.zeros(n, dtype=np.int32)
            self.download_particles(d, ei_last)
            d["ei"][:, -1] = ei_last
        check(self._lib.pb_particles_download_ids(self._h, n, ptr(d["particle_id"])))
        return d

    def flag_view_outside_time(self, dt, endtime):
        check(self._lib.pb_flag_view_outside_time(self._h, float(dt), float(endtime)))

    def delete_view_outside_time(self, dt, endtime):
        check(self._lib.pb_delete_view_outside_time(self._h, float(dt), float(endtime)))

    def debug_normals(self, seed, rng_call, it, particle_id):
        pid = np.ascontiguousarray(particle_id, dtype=np.int64)
        out = np.empty((pid.size, 2), dtype=np.float64)
        check(self._lib.pb_debug_normals(self._h, int(seed), int(rng_call), int(it), pid.size, ptr(pid), ptr(out)))
        return out

    # pb_math_op (include/parcels_b200.h)
    MATH_OPS = {"cos_np": 0, "sin_lat": 1, "sincos_lon": 2, "div_by_cached": 3, "div_by_cached_guarded": 4, "box_muller_f32": 5,
                "cosf": 6, "sinf": 7, "cos": 8, "sin": 9}

    def debug_math(self, op, a, b=None):
        """The kernels' math primitive `op` evaluated on the device: (n, 2) float64 (see pb_debug_math)."""
        a = np.ascontiguousarray(a, dtype=np.float64).ravel()
        if b is not None:
            b = np.ascontiguousarray(np.broadcast_to(np.asarray(b, dtype=np.float64), a.shape))
        out = np.empty((a.size, 2), dtype=np.float64)
        check(self._lib.pb_debug_math(self._h, self.MATH_OPS[op], a.size, ptr(a), ptr(b), ptr(out)))
        return out

    AXES = {"lon": 0, "lat": 1, "depth": 2, "time": 3}

    def debug_axis_cells(self, axis, nodes):
        """The device cell table of a float64 rectilinear axis of `nodes` nodes: (nodes - 1, 4) float64 {lo, hi, 1 / (hi - lo), 0}
        (see pb_debug_axis_cells)."""
        out = np.empty((nodes - 1, 4), dtype=np.float64)
        check(self._lib.pb_debug_axis_cells(self._h, self.AXES[axis], nodes - 1, ptr(out)))
        return out

    LAUNCH_FAMILIES = {"agrid_fast": 0, "agrid": 1, "cgrid": 2, "curv_agrid": 3, "sample_flags": 4}  # enum pb_launch_family

    def debug_launch_block(self, family):
        """Threads per block of the particle kernels of `family` (see pb_debug_launch_block)."""
        block = self._lib.pb_debug_launch_block(self.LAUNCH_FAMILIES[family])
        if block <= 0:
            check(block)
        return block
