"""``ParticleSet`` with the reference's constructor / ``execute`` API (``_core/particleset.py``)
whose inner loop -- ``Kernel.execute`` (``_core/kernel.py:174-247``) -- runs on the GPU.

Host code here is control only: argument normalisation, the outer loop over output
intervals, error mapping and compaction of deleted particles.  It never computes a
trajectory; if the CUDA library or a GPU is missing, ``execute`` raises.
"""

from __future__ import annotations

import datetime
import os

import numpy as np

from .particle import _CORE, Particle, ParticleClass, create_particle_data
from .plan import KernelPlan, _min_or_max, batch_facts, evaluated_mask
from .statuscodes import ERRORS_TO_THROW, StatusCode, raise_for_state

__all__ = ["Kernel", "ParticleSet"]


def _to_float_seconds(v):
    """reference _core/utils/time.py:192-207."""
    if isinstance(v, datetime.timedelta):
        return v.total_seconds()
    if isinstance(v, np.timedelta64):
        return float(v / np.timedelta64(1, "s"))
    if isinstance(v, (np.datetime64, datetime.datetime)):
        raise TypeError(f"a point in time is not a duration: {v!r}")
    return float(v)


def _fill(a, value):
    """``a[:] = value``; whole float64 / int32 columns of a large set go through the library's multi-threaded pass
    (pb_host_fill_*): at 1e7 particles one NumPy thread needs longer for `dt[:] = dt` than the device for the copies."""
    if a.size >= (1 << 20) and a.flags.c_contiguous and a.dtype in (np.float64, np.int32):
        from . import _lib

        lib = _lib.load()
        if a.dtype == np.float64:
            _lib.check(lib.pb_host_fill_f64(_lib.ptr(a), a.size, float(value)))
        else:
            _lib.check(lib.pb_host_fill_i32(_lib.ptr(a), a.size, int(value)))
    else:
        a[:] = value


def _fill_dt(pset, d, dt):
    """``particles.dt = dt`` at the end of Kernel.execute (kernel.py:225-226).  The fused device kernels never touch the host ``dt``
    column: when execute() has just filled THIS array with THIS value (`_dt_filled`), the second 80 MB pass per 1e7 particles is
    skipped; downloads that made new arrays, compacted views, user kernels and RK45 all take the fill."""
    mark = pset.__dict__.get("_dt_filled")
    a = d["dt"]
    if mark is not None and mark[0] is a and mark[1] == dt:
        return
    _fill(a, dt)


_CORE_NAMES = {name for name, _ in _CORE} | {"ei"}


def _remove_deleted_host(d: dict) -> int:
    """Kernel.remove_deleted on host arrays (reference _core/kernel.py:98-106 -> np.delete on every column,
    _core/particleset.py:247-250): drops the rows with state == Delete from EVERY column of ``d`` (the dict object is kept,
    its arrays are replaced, as np.delete does).  Large sets go through the library's multi-threaded compaction."""
    state = d["state"]
    n = len(state)
    if n >= (1 << 20) and all(v.flags.c_contiguous and len(v) == n for v in d.values()) and state.dtype == np.int32:
        import ctypes as C

        from . import _lib

        lib = _lib.load()
        keep = int(lib.pb_host_count_keep(_lib.ptr(state), n, int(StatusCode.Delete)))
        if keep == n:
            return 0
        names = list(d)
        new = {k: np.empty((keep, *d[k].shape[1:]), dtype=d[k].dtype) for k in names}
        src = (C.c_void_p * len(names))(*(d[k].ctypes.data for k in names))
        dst = (C.c_void_p * len(names))(*(new[k].ctypes.data for k in names))
        rb = (C.c_int64 * len(names))(*(d[k].strides[0] if d[k].ndim > 1 else d[k].itemsize for k in names))
        _lib.check(lib.pb_host_compact(_lib.ptr(state), n, int(StatusCode.Delete), len(names), src, dst, rb))
        d.update(new)
        return n - keep
    dele = np.where(state == StatusCode.Delete)[0]
    if len(dele):
        for k in d:
            d[k] = np.delete(d[k], dele, axis=0)
    return len(dele)


def _ei_last(d, owner=None):
    """The last ``ei`` column as a contiguous int32 array (what the device transfers use): the column itself with one grid, a
    copy with several (constant fields, further grids) -- a threaded strided gather into a staging column kept on ``owner``
    for large sets (NumPy into fresh memory: ~18 ms per 1e7)."""
    ei = d["ei"]
    col = ei[:, -1]
    if col.flags.c_contiguous:
        return col
    n = len(col)
    if n >= (1 << 20) and ei.dtype == np.int32 and ei.flags.c_contiguous:
        from . import _lib

        out = None if owner is None else owner.__dict__.get("_ei_stage")
        if out is None or len(out) != n:
            out = np.empty(n, dtype=np.int32)
            if owner is not None:
                owner.__dict__["_ei_stage"] = out
        _lib.check(_lib.load().pb_host_copy_strided_i32(_lib.ptr(out), 1, col.ctypes.data_as(_lib.C.c_void_p), ei.shape[1], n))
        return out
    return np.ascontiguousarray(col)


def _store_ei(d, ei_last):
    """``d["ei"][:, -1] = ei_last`` -- unless ``ei_last`` IS that column (one grid: the contiguous view the download wrote into)."""
    ei = d["ei"]
    col = ei[:, -1]
    if col.flags.c_contiguous and col.ctypes.data == ei_last.ctypes.data:
        return
    n = len(col)
    if n >= (1 << 20) and ei.dtype == np.int32 and ei.flags.c_contiguous and ei_last.dtype == np.int32 and ei_last.flags.c_contiguous:
        from . import _lib

        _lib.check(_lib.load().pb_host_copy_strided_i32(col.ctypes.data_as(_lib.C.c_void_p), ei.shape[1], _lib.ptr(ei_last), 1, n))
        return
    col[:] = ei_last


def _has_nan(a) -> bool:
    """np.isnan(a).any() without the temporary: one NaN-propagating reduction (an inf - inf false positive is re-checked)."""
    s = a.sum() if len(a) else 0.0
    return bool(s != s) and bool(np.isnan(a).any())


def _replay_first_error(plan, eng, rep, rewind, advance, dt, endtime):
    """The reference stops the whole set at the END of the first loop iteration in which any particle is in an error state
    (kernel.py:239-245): after a launch whose report ``rep`` saw one, ``rewind()`` to the start-of-interval copy and ``advance(k)``
    (up to k loop iterations) again so that every particle is left exactly where the reference leaves it.  Returns the report
    of the replay, or None when there is nothing to replay."""
    k = rep["first_error_iter"]
    if rep["n_error"] > 0:
        rewind()
        out = advance(k + 1)  # up to and including that iteration
        if out["n_out_of_time"] > 0:
            # an out-of-interval sample flags the WHOLE evaluated view (index_search.py:85-86, field.py:31-44)
            rewind()
            advance(k)
            eng.flag_view_outside_time(dt, endtime)
        return out
    if plan.delete_on_error and rep["n_out_of_time"] > 0:
        # Same whole-view rule under the DeleteParticle handler: every particle evaluated in the first iteration in which ANY
        # particle sampled outside the time interval is flagged, hence deleted (field.py:31-44 then the handler) -- replay up
        # to that iteration, then delete the view.  (The lanes deleted their own out-of-interval particle; the others ran on.)
        rewind()
        out = advance(k)
        eng.delete_view_outside_time(dt, endtime)
        out["n_deleted"] += 1
        out["max_state"] = max(out["max_state"], int(StatusCode.Delete))
        out["n_out_of_time"] = rep["n_out_of_time"]
        return out
    return None


class Kernel:
    """``Kernel(kernels=[...], pset=pset)`` as in the reference (_core/kernel.py:40-96): validates the list (functions with the
    ``(particles, fieldset)`` signature, RK45 prerequisites) and names it; ``pset.execute`` lowers the same list to device launches."""

    def __init__(self, kernels, pset):
        if not isinstance(kernels, list):  # (KernelPlan also takes a bare function)
            raise ValueError(f"kernels must be a list. Got {kernels=!r}")
        self._fieldset = pset.fieldset
        self._pclass = pset._pclass
        self._plan = KernelPlan(kernels, pset.fieldset, pset._pclass)
        self._kernels = kernels

    funcname = property(lambda self: "".join(f.__name__ for f in self._kernels))
    pclass = property(lambda self: self._pclass)
    fieldset = property(lambda self: self._fieldset)


class ParticleSet:
    """Same construction arguments as the reference (``_core/particleset.py:59-137``):
    ``ParticleSet(fieldset, pclass=Particle, t=, z=, y=, x=, particle_ids=)``; ``t`` may be
    float seconds, timedelta64 or (with a datetime time axis) datetime64."""

    PIPELINE_MIN_PARTICLES = 262_144  # below this one chunk's kernel does not cover the copies of the next (pipeline_chunks)

    def __init__(self, fieldset, pclass=Particle, *, t=None, z=None, y=None, x=None, particle_ids=None, device=0,
                 seed=0, **kwargs):  # fmt: skip
        if not isinstance(pclass, ParticleClass):
            raise NotImplementedError("pclass must be parcels_b200.Particle or Particle.add_variable(...) (float32 positions)")
        self.fieldset = fieldset
        self._pclass = pclass
        self.device = device
        self.seed = int(seed)  # Philox key of the Wiener increments (DiffusionUniformKh)
        self._rng_call = 0
        self._device_synced = False
        # Device-resident intervals (SURVEY.md 8f-2): between the output intervals of one execute() call the particle
        # SoA lives in HBM only; the host arrays are refreshed on first access (the `_data` property).
        self._host = None
        self._host_stale = False
        self.eager_host = False  # True: refresh the host arrays at the end of every execute() (shared-array adapters)
        # > 1: Kernel.execute on host arrays runs as that many pipelined chunks (copies under kernels, pb_advect_host)
        # (default 8: copies of one chunk run under the kernels of the others)
        self.pipeline_chunks = int(os.environ.get("PB_PIPELINE_CHUNKS", "8"))
        self._n_device = 0
        self._stale_dt = 1.0
        self.last_report = None
        y = np.empty(0) if y is None else np.array(y).flatten()
        x = np.empty(0) if x is None else np.array(x).flatten()
        if particle_ids is None:
            particle_ids = np.arange(x.size)
        if z is None:
            depth = fieldset.grid.depth
            if depth is not None and depth.size:
                z = np.ones(x.size) * depth[np.argmin(np.abs(depth))]
            else:
                z = np.zeros(x.size)
        else:
            z = np.array(z).flatten()
        assert x.size == y.size and x.size == z.size, "x, y, z don't all have the same lengths"
        if t is None or np.size(t) == 0:
            t = np.array(np.nan)
        else:
            t = np.array(t).flatten()
            if np.issubdtype(t.dtype, np.datetime64):
                t = ((t - fieldset._time_origin) / np.timedelta64(1, "s")).astype(np.float64)
            elif np.issubdtype(t.dtype, np.timedelta64):
                t = (t / np.timedelta64(1, "s")).astype(np.float64)
            else:
                t = t.astype(np.float64)
        t = np.repeat(t, x.size) if t.size == 1 else t
        assert x.size == t.size, "t and positions (x, y, z) do not have the same lengths."
        ti = fieldset.time_interval
        if ti is not None and t.size and not np.isnan(t).all() and (np.any(t < 0) or np.any(t > ti[1] - ti[0])):
            import warnings  # reference _core/particleset.py:485-494

            from .statuscodes import ParticleSetWarning

            warnings.warn("Some particles are set to be released outside the FieldSet's executable time domain.", ParticleSetWarning,
                          stacklevel=2)  # fmt: skip
        self._data = create_particle_data(
            nparticles=x.size,
            ngrids=len(fieldset.gridset),
            initial=dict(t=t, z=z, y=y, x=x, particle_id=np.asarray(particle_ids)),
            pclass=pclass,
        )
        for k, v in kwargs.items():  # initial values of extra variables (reference particleset.py:129-134)
            if k not in self._data:
                raise RuntimeError(f"Particle class does not have Variable {k}")
            self._data[k][:] = np.array(v).flatten()

    # -- host mirror of the particle SoA --------------------------------------------------------
    @property
    def _data(self):
        if self._host_stale:
            self._sync_host()
        return self._host

    @_data.setter
    def _data(self, value):
        self._host = value
        self._host_stale = False

    def _release_device(self):
        """Another ParticleSet is about to use this engine's resident SoA (Engine.claim): fetch what only lives there."""
        if self._host_stale:
            self._sync_host()
        self._device_synced = False

    def _sync_host(self):
        """Bring the host arrays up to date with the device-resident set (sizes may differ after deletions)."""
        eng = self.fieldset.engine(self.device)
        if not eng.owned_by(self):
            raise RuntimeError("the device-resident particles of this ParticleSet were overwritten by another ParticleSet "
                               "(engine ownership lost before the host arrays were refreshed)")
        d = self._host
        if d is not None and len(d["x"]) == eng.particle_count():
            # nothing was deleted: ids and order are unchanged, refresh the existing (possibly pinned) arrays in place
            ei_last = d["ei"][:, -1]  # the last grid's column: written in place when it is contiguous (one grid)
            if ei_last.flags.c_contiguous:
                eng.download_particles(d, ei_last)
            else:
                ei_last = np.empty(len(d["x"]), dtype=np.int32)
                eng.download_particles(d, ei_last)
                _store_ei(d, ei_last)
        else:
            new = eng.download_all(ngrids=len(self.fieldset.gridset))
            if d is None:
                d = new
            else:  # keep the dict object: it may be shared with the caller (adapter.pset_from_parcels)
                d.update(new)
        _fill_dt(self, d, self._stale_dt)  # kernel.py:225-226
        self._host = d
        self._host_stale = False
        self._device_synced = True

    def _lazy_ok(self, plan) -> bool:
        """Can the set stay device-resident across output intervals?  Built-in kernel lists on rectilinear grids with
        the default Particle variables (extra variables live on the host; the curvilinear hint test needs host `ei`)."""
        fs = self.fieldset
        return plan.kind in ("fixed", "advdiff") and not fs.grid.curvilinear and fs.time_window is None and len(self._pclass.extra) == 0

    def _output_columns(self, t, names, indices=None):
        """Rows due for output at time ``t`` (reference `_to_write_particles`, _core/particlefile.py:198-221) of the
        columns ``names`` -> (dict of compacted arrays, selected_on_device)."""
        from .engine import Engine
        from .particlefile import to_write_particles

        if self._host_stale and indices is None and all(n in Engine.OUTPUT_COLUMNS for n in names):
            eng = self.fieldset.engine(self.device)
            m = eng.output_select(t, self._stale_dt)
            return eng.output_gather(m, columns=tuple(names)), True
        d = self._data
        rows = to_write_particles(d, t) if indices is None else indices
        return {n: d[n][rows] for n in names}, False

    # -- container protocol ----------------------------------------------------------------------
    def __len__(self):
        return self._n_device if self._host_stale else len(self._host["x"])

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        data = self._data if "_host" in self.__dict__ else None
        if data is not None and name in data:
            return data[name]
        raise AttributeError(name)

    def __setattr__(self, name, value):
        """`pset.state = ...` writes the particle variable (reference _core/particleset.py:170-176)."""
        host = self.__dict__.get("_host")
        if not name.startswith("_") and isinstance(host, dict) and name in host:
            self._data[name][:] = value
        else:
            object.__setattr__(self, name, value)

    def __getitem__(self, index):
        """A write-through view on a subset (reference `pset[i]` / `pset[mask]`, _core/particleset.py:166-168)."""
        from .particlesetview import ParticleSetView, SingleParticleView, _global_mask

        if isinstance(index, (int, np.integer)) and not isinstance(index, (bool, np.bool_)):
            if not -len(self) <= index < len(self):
                raise IndexError(f"particle index {index} out of range for a set of {len(self)}")
            return SingleParticleView(self._data, index)
        return ParticleSetView(self._data, _global_mask(np.ones(len(self), dtype=bool), index), self.fieldset)

    @property
    def size(self):
        return len(self)

    def __iter__(self):
        """Single-particle views in storage order (reference _core/particleset.py:144-154)."""
        return (self[i] for i in range(len(self)))

    def add(self, particles):
        """Append another ParticleSet in place; its particle ids are shifted past this set's largest id
        (reference _core/particleset.py:188-224)."""
        assert particles is not None, f"Trying to add another {type(self)} to this one, but the other one is None - invalid operation."
        assert type(particles) is type(self)
        if len(particles) == 0:
            return
        if len(self) == 0:
            self._data = particles._data
            return
        mine, theirs = self._data, particles._data
        theirs["particle_id"] = theirs["particle_id"] + (mine["particle_id"].max() + 1)
        for k in mine:
            mine[k] = np.concatenate((mine[k], theirs[k]))
        self._device_synced = False
        return self

    def __iadd__(self, particles):
        self.add(particles)
        return self

    def remove_indices(self, indices):
        """reference _core/particleset.py:247-250."""
        for k in self._data:
            self._data[k] = np.delete(self._data[k], indices, axis=0)

    @classmethod
    def from_particlefile(cls, fieldset, pclass, filename, restart=True, restarttime=None, **kwargs):
        raise NotImplementedError("ParticleSet.from_particlefile is not yet implemented in v4.")  # reference particleset.py:264-292

    def data_indices(self, variable_name, compare_values, invert=False):
        """Indices of the particles whose ``variable_name`` equals (one of) ``compare_values`` (reference particleset.py:294-319)."""
        compare_values = np.array([compare_values]) if type(compare_values) not in [list, dict, np.ndarray] else compare_values
        return np.where(np.isin(self._data[variable_name], compare_values, invert=invert))[0]

    @property
    def _error_particles(self):
        return self.data_indices("state", [StatusCode.Success, StatusCode.Evaluate], invert=True)

    @property
    def _num_error_particles(self):
        return np.sum(np.isin(self._data["state"], [StatusCode.Success, StatusCode.Evaluate], invert=True))

    def populate_indices(self):
        """Pre-populate the cell guesses ``ei`` (reference _core/particleset.py:252-262): one grid search per grid of the
        gridset -- on the device for the fieldset's grid (`pb_sample_velocity` returns the raveled cell of every sample);
        the one-node grid of the constant fields has the single cell 0 (_core/index_search.py:45-46)."""
        d = self._data
        if len(self) == 0:
            return
        eng = self.fieldset.engine(self.device)
        if self.fieldset.time_window is not None:  # (only the cells are used, but a windowed engine samples resident levels only)
            self.fieldset.cover_window(self.device, np.zeros(1))
        *_, ei, _ = eng.sample_velocity(np.zeros(len(self)), d["z"], d["y"], d["x"], three_d=False, positions_are_f32=True,
                                        ei_hint=None, no_hint=True)  # fmt: skip
        d["ei"][:, 0] = ei
        if d["ei"].shape[1] > 1:
            d["ei"][:, 1:] = 0
        for k, host in enumerate(self.fieldset._extra_grids, start=1):  # further XGrids: the search of one of their fields
            host.engine(self.device)
            if host.time_window is not None:  # (as above)
                host.cover_window(self.device, np.zeros(1))
            if host.vector is not None:
                *_, ei_k, _ = host.engine(self.device).sample_velocity(np.zeros(len(self)), d["z"], d["y"], d["x"], three_d=False,
                                                                        positions_are_f32=True, ei_hint=None, no_hint=True)  # fmt: skip
            else:
                f = host.fields[0]
                _, ei_k, _ = host.engine(self.device).sample_scalar(f._slot, f.interp_method, np.zeros(len(self)), d["z"], d["y"], d["x"],
                                                                     positions_are_f32=True, ei_hint=None)  # fmt: skip
            d["ei"][:, k] = ei_k
        self._device_synced = False

    # -- the hot path ------------------------------------------------------------------------------
    def _kernel_execute(self, plan: KernelPlan, endtime: float, dt: float, *, resident: bool = False, lazy: bool = False):
        """Replaces ``Kernel.execute(pset, endtime, dt)`` (reference _core/kernel.py:174-247).

        ``resident=True`` (set by ``execute`` for the 2nd, 3rd, ... output interval of ONE call): the device
        copy of the particle SoA left by the previous interval is still exact -- nothing on the host can have
        changed it in between -- so the host->device upload is skipped.

        ``lazy=True`` (``_lazy_ok``): the result is NOT downloaded either; deleted particles are compacted on the
        device and the host arrays are refreshed only when somebody reads them (``_data``)."""
        if plan.stepwise:
            from .stepwise import kernel_execute_stepwise

            d = self._data
            if len(self) and np.isnan(d["t"]).any():
                raise ValueError("Time values cannot be NaN.")
            self._device_synced = False
            return kernel_execute_stepwise(self, plan, endtime, dt)
        if plan.kind == "rk45":
            return self._kernel_execute_rk45(plan, endtime, dt)
        eng = self.fieldset.engine(self.device)
        eng.claim(self)  # a ParticleSet that was resident here is synced to its host arrays first
        on_device = lazy and resident and self._host_stale and eng.particle_count() == self._n_device
        if on_device:
            # states are reset to Evaluate by the kernel itself (resume = 0); t cannot have become NaN on the device
            n, d, ei_last = self._n_device, None, None
            if n == 0:
                return
        else:
            d = self._data
            n = len(self)
            # kernel.py:188 `state[:] = Evaluate`: the device kernel resets the states itself (resume = 0) and every path below
            # writes the states it ends with back to the host -- only the windowed path resumes launches from host-visible states
            if self.fieldset.time_window is not None:
                d["state"][:] = StatusCode.Evaluate
            if n == 0:
                return
            if not self.__dict__.pop("_t_nan_free", False) and _has_nan(d["t"]):  # (execute() has just made that pass)
                bad = np.where(np.isnan(d["t"]))[0]
                raise ValueError(f"Time values for particles with indices {bad} cannot be NaN.")  # field.py:396-398
            ei_last = _ei_last(d, self)
        self._rng_call += 1
        if on_device:  # a resident interval: no particle can be back on the first time level; the depth bit of the first interval holds
            hint_all_zero, two_levels = False, self.__dict__.get("_batch_levels_resident", 0) & 2
        else:
            # (curvilinear grids: the reference skips the hint test for the WHOLE batch when every hinted xi is 0, e.g. on the first
            # eval of a fresh set)
            hint_all_zero, two_levels = batch_facts(self.fieldset, d, ei_last, dt, endtime)
            self.__dict__["_batch_levels_resident"] = two_levels

        def args(max_iters=-1, resume=False):
            return plan.launch_args(eng, dt, endtime, seed=self.seed, rng_call=self._rng_call, max_iters=max_iters, resume=resume,
                                    hint_all_zero=hint_all_zero, batch_levels=two_levels)  # fmt: skip

        needs_upload = not on_device and not (resident and self._device_synced and eng.particle_count() == n)
        # host arrays in (and out): cut into chunks whose copies run under the kernels of the other chunks (pb_advect_host)
        pipelined = (needs_upload and self.pipeline_chunks > 1 and n >= self.PIPELINE_MIN_PARTICLES and plan.kind == "fixed"
                     and self.fieldset.time_window is None)  # fmt: skip
        if not on_device and not pipelined and self.__dict__.get("_dt_pending") is not None:
            _fill(d["dt"], self.__dict__.pop("_dt_pending"))  # (not the pipelined path: the deferred fill is done here)
            self.__dict__["_dt_filled"] = (d["dt"], dt)
        downloaded = False
        if needs_upload and not pipelined:
            eng.upload_particles(d, ei_last)
        self._device_synced = False
        # start-of-interval state for the error replay: the host arrays, or (device-resident) a snapshot in HBM
        # (with the delete handler only an out-of-interval sample needs a replay: fields with a time axis)
        can_raise = not plan.delete_on_error
        if lazy and not pipelined and (can_raise or self.fieldset.time_interval is not None):
            eng.snapshot()
        rewind = eng.restore if (lazy or pipelined) else (lambda: eng.upload_particles(d, ei_last))
        windowed = self.fieldset.time_window is not None

        def advance(max_iters=-1):
            """One Kernel.execute on the device particles (up to ``max_iters`` loop iterations)."""
            if not windowed:
                return eng.advect(args(max_iters=max_iters))

            def launch(resume):
                if resume and plan.diffusion:
                    # the Wiener increments of DiffusionUniformKh are keyed by (particle, iteration OF THE LAUNCH, call): a resumed
                    # advect_kernel restarts its iteration count, so it gets its own call index -- otherwise the same increments
                    # would be drawn again.  (pb_advect_diffusion continues each particle's count: its stream needs no new index.)
                    self._rng_call += 1
                eng.advect_async(args(max_iters=max_iters, resume=resume))

            return self._advect_windowed(eng, d, dt, endtime, launch)

        # pb_advect_diffusion counts the iterations of a windowed call across its launches: its replay is exact as well
        replayable = not windowed or plan.kind == "advdiff"
        if windowed:
            rep = advance()
        elif pipelined:
            # the result comes back with the same call when somebody is going to read it on the host anyway
            downloaded = not lazy or self.eager_host
            filler = None
            if self.__dict__.pop("_dt_pending", None) is not None:  # the deferred `particles.dt = dt` under the GPU work
                import threading

                filler = threading.Thread(target=_fill, args=(d["dt"], dt))
                filler.start()
                self.__dict__["_dt_filled"] = (d["dt"], dt)
            try:
                rep = eng.advect_host(args(), d, ei_last, download=downloaded, n_chunks=self.pipeline_chunks)
            finally:
                if filler is not None:
                    filler.join()
        else:
            rep = advance()
        replayed = _replay_first_error(plan, eng, rep, rewind, advance, dt, endtime) if replayable else None
        if replayed is not None:
            rep, downloaded = replayed, False
        self.last_report = rep
        self._stale_dt = dt
        if lazy and rep["max_state"] < StatusCode.Error:
            # nothing to raise: stay in HBM.  Deleted particles are dropped there, order preserved
            # (Kernel.remove_deleted -> np.delete, kernel.py:98-106, particleset.py:247-250)
            deletions = rep["n_deleted"] > 0 or rep["max_state"] == StatusCode.Delete
            self._n_device = eng.remove_deleted() if deletions else n
            if downloaded and not deletions:  # the pipelined call has already brought the result back: host == device
                self._host_stale = False
                _store_ei(d, ei_last)
                _fill_dt(self, d, dt)  # kernel.py:225-226
                self._device_synced = True
            else:
                self._host_stale = True
            return
        if lazy:
            self._host_stale = True
            self._n_device = n
            d = self._data  # full download
        elif (rep["n_deleted"] > 0 and rep["max_state"] < StatusCode.Error and len(self._pclass.extra) == 0
              and d["ei"].shape[1] == 1 and self.fieldset.time_window is None and set(d) == _CORE_NAMES
              and all(v.flags.c_contiguous for v in d.values())):  # fmt: skip
            # deletions, nothing to raise: drop the deleted particles in HBM (order preserved, like np.delete) and download the
            # compacted set INTO THE PREFIX of the existing host arrays (views of the same -- possibly pinned -- buffers: no 11
            # fresh columns to fault in, no np.delete pass over every host array, kernel.py:98-106).  Also after a pipelined call
            # that already brought the uncompacted result back: a second, compacted D2H is cheaper than compacting on the host.
            keep = eng.remove_deleted()
            new = {k: v[:keep] for k, v in d.items()}
            eng.download_particles(new, new["ei"][:, -1])
            eng.download_ids(new["particle_id"])
            new["dt"][:] = dt  # kernel.py:225-226
            d.update(new)  # keep the dict object: it may be shared with the caller (adapter.pset_from_parcels)
            self._device_synced = True
            return
        else:
            if not downloaded:
                eng.download_particles(d, ei_last)
            _store_ei(d, ei_last)
            _fill_dt(self, d, dt)  # kernel.py:225-226
        # the device report says whether any particle was deleted / errored: the O(N) host scans of
        # kernel.py:98-106,239-245 only run when there is something to find
        self._device_synced = True  # host arrays == device arrays from here on (until the host compacts them)
        if rep["n_deleted"] > 0 or rep["max_state"] == StatusCode.Delete:
            if _remove_deleted_host(d) > 0:
                self._device_synced = False
        if rep["max_state"] >= StatusCode.Error:
            for code in ERRORS_TO_THROW:
                hit = d["state"] == code
                if np.any(hit):
                    raise_for_state(code, d["z"][hit], d["y"][hit], d["x"][hit], d["t"][hit])

    def _kernel_execute_rk45(self, plan, endtime, dt):
        """``Kernel.execute`` with AdvectionRK45 (reference _core/kernel.py:108-120,190-245): per-particle dt / next_dt,
        Repeat loop and step doubling run inside ONE device kernel (csrc/rk45.cu); dt is not reset to the nominal step."""
        d = self._data
        self._device_synced = False
        d["state"][:] = StatusCode.Evaluate
        if len(self) == 0:
            return
        if np.isnan(d["t"]).any():
            raise ValueError(f"Time values for particles with indices {np.where(np.isnan(d['t']))[0]} cannot be NaN.")
        eng = self.fieldset.engine(self.device)
        eng.claim(self)
        rep = self._advect_rk45(plan, eng, dt, endtime)
        if rep["max_state"] == StatusCode.Delete:
            dele = np.where(d["state"] == StatusCode.Delete)[0]
            if len(dele) > 0:
                self.remove_indices(dele)

    def _advect_rk45(self, plan, eng, dt, endtime, *, stepwise=False):
        """Upload, AdvectionRK45 on the device (pb_advect_rk45) and write-back of positions, states, ``ei``, dt and next_dt (the
        reference leaves every particle's own dt: it is not reset to the nominal step, kernel.py:224-226).  ``stepwise``: ONE
        iteration of a stepwise list (kernels_only) -- every evaluated particle's attempts until its step is accepted, the
        reference's `while state == Repeat` re-runs of the kernel (kernel.py:212-216); the host does the position update.
        Otherwise the whole loop of the call, through the time window's levels on a time-windowed FieldSet."""
        d = self._data
        ei_last = np.ascontiguousarray(d["ei"][:, -1])
        eng.upload_particles(d, ei_last)
        dt_arr = np.ascontiguousarray(d["dt"], dtype=np.float64)
        ndt_arr = np.ascontiguousarray(d["next_dt"], dtype=np.float64)
        hint_all_zero, two_levels = batch_facts(self.fieldset, d, ei_last, dt, endtime, mid_iteration=stepwise)

        def launch(resume):  # (a resumed launch continues every particle's dt, next_dt and iteration count)
            args = plan.launch_args(eng, dt, endtime, hint_all_zero=hint_all_zero, batch_levels=two_levels, resume=resume,
                                    kernels_only=stepwise, next_dt_dtype=d["next_dt"].dtype)  # fmt: skip
            return eng.advect_rk45(args, dt_arr, ndt_arr)

        if stepwise:
            from .stepwise import _no_wait

            rep = launch(True)
            _no_wait(rep)
        elif self.fieldset.time_window is None:
            rep = self.last_report = launch(False)
        else:
            rep = self.last_report = self._advect_windowed(eng, d, dt, endtime, launch, synchronous=True)
        eng.download_particles(d, ei_last)
        _store_ei(d, ei_last)
        d["dt"][:] = dt_arr
        d["next_dt"][:] = ndt_arr
        if rep["n_error"] > 0:
            stuck = np.where(d["state"] == StatusCode.Error)[0]
            if stepwise:
                raise RuntimeError(f"AdvectionRK45: particles {stuck[:10]} have dt == 0 before endtime={endtime}; reset pset.dt before continuing")
            raise RuntimeError(f"AdvectionRK45: particles {stuck[:10]} have dt == 0 before endtime={endtime}; the reference's loop "
                               "never terminates on them (kernel.py:199-203 clamps the dt of particles that finished an earlier "
                               "interval to 0 and RK45 mode never restores it).  Reset pset.dt before continuing.")  # fmt: skip
        return rep

    def _advect_windowed(self, eng, d, dt, endtime, launch, *, synchronous=False):
        """Time-slab streaming: advance until every particle reached ``endtime``, sliding the resident time levels as the
        particles' clock crosses them.  ``launch(resume)`` runs one launch of the call on the device particles -- pb_advect,
        pb_advect_diffusion or pb_advect_rk45 -- with ``resume`` from the second launch on.  An asynchronous launch returns
        None and the next level is copied while its kernel runs.  A ``synchronous`` one (pb_advect_rk45: it brings dt / next_dt
        back) returns its report; the next level is copied before it, under the kernel only when the level data is pinned."""
        fs = self.fieldset
        sign = 1 if dt > 0 else -1
        todo = evaluated_mask(d, dt, endtime)
        t_ref = (d["t"][todo].min() if sign > 0 else d["t"][todo].max()) if todo.any() else float(d["t"][0])
        fs.slide_window(self.device, t_ref, sign)
        total = None
        first = True
        while True:
            if synchronous:
                fs.prefetch_next(self.device, sign)
            rep = launch(not first)
            if not synchronous:
                fs.prefetch_next(self.device, sign)  # H2D of the next level overlaps the kernel
                rep = eng.last_report()
            if total is None:
                total = dict(rep)
            else:
                for k in ("particle_steps", "cache_refills", "kernel_ms", "n_error", "n_deleted", "n_out_of_time"):
                    total[k] += rep[k]
                for k in ("max_state", "max_iters_done"):
                    total[k] = max(total[k], rep[k])
                if rep["first_error_iter"] >= 0 and not 0 <= total["first_error_iter"] <= rep["first_error_iter"]:
                    total["first_error_iter"] = rep["first_error_iter"]
                total["n_wait_window"] = rep["n_wait_window"]
            first = False
            if rep["n_wait_window"] == 0:
                return total
            moved = fs.slide_window(self.device, rep["wait_t_min"] if sign > 0 else rep["wait_t_max"], sign)
            if not moved:
                raise RuntimeError(f"time window of {fs.time_window} levels cannot cover one step of dt={dt}: widen time_window")

    def execute(self, kernels, dt, endtime=None, runtime=None, output_file=None, verbose_progress=False):
        """reference _core/particleset.py:355-470 (outer loop) and :497-585 (argument handling)."""
        if len(self) == 0:
            return
        plan = KernelPlan(kernels, self.fieldset, self._pclass)
        try:
            dt = _to_float_seconds(dt)
            sign_dt = int(np.sign(dt))
            assert sign_dt in (-1, 1)
        except (ValueError, TypeError, AssertionError) as e:
            raise ValueError(f"dt must be a non-zero datetime.timedelta or np.timedelta64 object, got {dt=!r}") from e
        # `particles.dt = dt` (particleset.py:414).  The fused device kernels never read or write this host column, so for them the
        # 80 MB pass per 1e7 particles is taken off the critical path: a large set's column is filled by a helper thread WHILE the first
        # pipelined Kernel.execute runs on the GPU (`_dt_pending` -> `_kernel_execute`); `_fill_dt` need not write it again at the end
        # (`_dt_filled`).  Plans with user kernels or RK45 read / write per-particle steps: filled here, no mark.
        fused = plan.kind in ("fixed", "advdiff")
        if fused and len(self) >= self.PIPELINE_MIN_PARTICLES and not self._host_stale:
            self.__dict__["_dt_pending"] = dt
        else:
            _fill(self._data["dt"], dt)
            self.__dict__["_dt_filled"] = (self._data["dt"], dt) if fused else None
        if runtime is not None:
            try:
                runtime = _to_float_seconds(runtime)
            except (ValueError, TypeError) as e:  # reference _core/particleset.py:510-518
                raise ValueError(f"The runtime must be a datetime.timedelta, np.timedelta64 or float object. Got {type(runtime)}") from e
            if runtime < 0:
                raise ValueError(f"The runtime must be a non-negative timedelta or float. Got {runtime=!r}")
        ti = self.fieldset.time_interval
        if runtime is not None and endtime is not None:
            raise ValueError(f"runtime and endtime are mutually exclusive - provide one or the other. Got {runtime=!r}, {endtime=!r}")
        if runtime is None and ti is None:
            raise ValueError("The runtime must be provided when the time_interval is not defined for a fieldset.")
        if runtime is None and endtime is None:
            raise ValueError("Either runtime or endtime must be provided.")
        t = self._data["t"]
        # `particle_release_times.min()` / `.max()` (reference particleset.py:541-544) PROPAGATE NaN: as soon as one release time
        # is unset the start time is the fieldset's start (`_get_start_time`, :575-585) and EVERY particle's t is set to it (:413-414)
        first = _min_or_max(t, sign_dt == 1)
        any_nan = bool(np.isnan(first))
        if endtime is not None:
            origin = self.fieldset._time_origin
            stamped = isinstance(origin, (np.datetime64, np.timedelta64))
            if stamped and type(endtime) is not type(origin):  # reference _core/particleset.py:545-549
                raise ValueError(f"The endtime must be of the same type as the fieldset.time_interval start time. Got {endtime=!r} "
                                 f"with a time axis starting at {origin!r}")
            if stamped:
                endtime = float((endtime - origin) / np.timedelta64(1, "s"))
            else:  # a time axis given in seconds (this package's from_arrays): seconds
                try:
                    endtime = _to_float_seconds(endtime)
                except TypeError as e:
                    raise ValueError(f"The endtime must be of the same type as the fieldset.time_interval start time. Got {endtime=!r}") from e
            if ti is not None and not (ti[0] <= endtime <= ti[1]):
                raise ValueError(f"Calculated/provided end time of {endtime!r} is not in fieldset time interval {ti!r}.")
        if np.isnan(first):
            start_time = 0.0 if sign_dt == 1 else float(ti[1] if ti is not None else runtime)
        else:
            start_time = float(first)
        end_time = endtime if endtime is not None else start_time + sign_dt * runtime
        if any_nan:
            t[:] = start_time
        outputdt = _to_float_seconds(output_file.outputdt) if output_file is not None else None
        if outputdt and np.isfinite(outputdt) and len(t) <= 1_000_000 and np.any(np.isfinite(t) & ((t - start_time) % outputdt != 0)):
            import warnings  # reference _core/particleset.py:473-482

            from .statuscodes import ParticleSetWarning

            warnings.warn("Some of the particles have a start time difference that is not a multiple of outputdt. This could cause the "
                          "first output of some of the particles that start later in the simulation to be at a different time than "
                          "expected.", ParticleSetWarning, stacklevel=2)  # fmt: skip
        if output_file is not None and hasattr(output_file, "set_metadata"):  # reference particleset.py:400-403
            output_file.set_metadata(self.fieldset.grid.mesh)
            output_file.metadata["parcels_kernels"] = plan.funcname
        next_output = None
        if output_file is not None:
            output_file.write(self, start_time)
            next_output = start_time + outputdt * sign_dt
        time = start_time
        interval = 0
        self._device_synced = False  # between execute() calls the host owns the arrays
        lazy = self._lazy_ok(plan)
        self.__dict__["_t_nan_free"] = True  # no NaN times (left) after the pass above: the first Kernel.execute need not look again
        try:
            while sign_dt * (time - end_time) < 0:
                if next_output is not None:
                    next_time = min(next_output, end_time) if sign_dt > 0 else max(next_output, end_time)
                else:
                    next_time = end_time
                self._kernel_execute(plan, next_time, dt, resident=interval > 0, lazy=lazy)
                interval += 1
                if next_output is not None and np.abs(next_time - next_output) < 0.001:
                    output_file.write(self, next_output)
                    if np.isfinite(outputdt):
                        next_output += outputdt * sign_dt
                time = next_time
        finally:
            self.__dict__.pop("_t_nan_free", None)
            self.__dict__.pop("_dt_filled", None)
            if self.__dict__.pop("_dt_pending", None) is not None and not self._host_stale:  # (no Kernel.execute ran: runtime 0)
                _fill(self._data["dt"], dt)
            if output_file is not None and hasattr(output_file, "close"):  # `with output_file:` (particleset.py:444)
                output_file.close()
        if self.eager_host and self._host_stale:
            self._sync_host()
