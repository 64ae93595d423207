"""``ParticleSet`` with the reference's constructor / ``execute`` API (``_core/particleset.py``)
whose inner loop -- ``Kernel.execute`` (``_core/kernel.py:174-247``) -- runs on the GPU.

Host code here is control only: argument normalisation, the outer loop over output
intervals, error mapping and compaction of deleted particles.  It never computes a
trajectory; if the CUDA library or a GPU is missing, ``execute`` raises.
"""

from __future__ import annotations

import datetime
import os
import types

import numpy as np

from . import kernels as K
from .particle import _CORE, Particle, ParticleClass, create_particle_data
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


def _min_or_max(t, want_min: bool) -> float:
    """``t.min()`` / ``t.max()`` with NumPy's NaN propagation (any NaN -> NaN), as the reference takes them (particleset.py:541-544).
    (NumPy's own SIMD reduction: 3.5 ms for 1e7 values; a threaded scalar loop in the library measured 15 ms.)"""
    return float(t.min() if want_min else t.max())


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


def _first_eval_two_levels(fieldset, t, evaluated) -> bool:
    """float32 grids with a time axis: True when some evaluated particle is NOT exactly on the first time level.  The reference
    decides `lenT = 2 if any(tau > 0)` for the whole batch of an evaluation (_xinterpolators.py:130); tau == 0 only AT the first
    level (`_search_1d_array` is left-sided: any later level gives tau == 1), so only the first evaluation of a call can mix the
    two cases -- and there a two-level batch promotes the value of a first-level particle to float64.  On float64 grids every
    barycentric coordinate is float64 and the promotion changes nothing."""
    if fieldset._time_s is None or fieldset.grid.lon.dtype != np.float32:
        return False
    t0 = float(fieldset._time_s[0])
    if t.size >= (1 << 20) and _min_or_max(t, True) == t0 and _min_or_max(t, False) == t0:
        return False  # every particle sits on the first level (the usual fresh set): no masked copies of a large column
    te = t[evaluated() if callable(evaluated) else evaluated]
    return bool(te.size) and bool(np.any(te != float(fieldset._time_s[0])))


def _batch_levels(fieldset, d, evaluated) -> int:
    """``pb_advect_args.batch_levels``: the reference's per-batch decisions a lane cannot make by itself.
    PB_BATCH_FIRST_EVAL_TWO_T (1): see `_first_eval_two_levels`.  PB_BATCH_TWO_Z (2): `lenZ = 2 if any(zeta > 0)`
    (_xinterpolators.py:401) -- with XFreeslip / XPartialslip the land test then looks at the second depth level for every particle
    of the batch (:426-447); zeta > 0 means below the first depth level (left-sided search), taken as constant over the call."""
    flags = 1 if _first_eval_two_levels(fieldset, d["t"], evaluated) else 0  # (`evaluated`: mask, or a callable making it on demand)
    depth = fieldset.grid.depth
    if fieldset.interp_method in ("freeslip", "partialslip") and depth is not None and len(depth) > 1:
        ze = d["z"][evaluated() if callable(evaluated) else evaluated]
        if ze.size and np.any(ze > depth[0]):
            flags |= 2
    return flags


def _hint_all_zero(ei_last, evaluated, xdim) -> bool:
    """Curvilinear grids: True when the hinted xi (= ei % xdim) of EVERY evaluated particle is 0 -- the reference then skips
    the hint test for the whole batch (`if np.any(xi)`, _core/index_search.py:269).  `evaluated(slice)` gives the mask of a
    slice of the set; a non-zero hint among the first few thousand particles settles the (usual) answer without a full pass."""
    head = slice(0, min(len(ei_last), 4096))
    if np.any((ei_last[head][evaluated(head)].astype(np.int64) % xdim) != 0):
        return False
    if not ei_last.any():  # a fresh set: every hint is 0 (one pass over the int32 column, no masked / widened copies)
        return True
    full = slice(None)
    return not np.any((ei_last[evaluated(full)].astype(np.int64) % xdim) != 0)


def _builtin_name(f):
    """Name of the built-in kernel ``f`` stands for, or None for a user function.  Built-ins are this package's
    tokens (kernels.py, by identity) and the reference package's own kernel functions (by module + name); a user
    function that merely shares a name -- e.g. the ubiquitous user-defined ``DeleteParticle`` -- is NOT one."""
    n = f.__name__
    if n != "_none" and getattr(K, n, None) is f:
        return n
    mod = getattr(f, "__module__", "") or ""
    if mod.startswith("parcels.kernels") and (n in K.SCHEMES or n in K.ADVDIFF or n in ("DiffusionUniformKh", "AdvectionRK45")) and n != "_none":
        return n
    return None


def _delete_on_error(particles, fieldset):
    """DeleteParticle token inside a stepwise list (reference idiom tests/common_kernels.py:12-13)."""
    s = np.asarray(particles.state)
    particles.state = np.where(s >= 50, StatusCode.Delete, s)


def _assert_kernel_signature(f):
    """A kernel function is ``f(particles, fieldset)`` (reference _python.py:33-52 `assert_same_function_signature` against
    AdvectionRK4, called from Kernel.__init__, _core/kernel.py:69)."""
    import inspect

    params = list(inspect.signature(f).parameters.values())
    if len(params) != 2:
        raise ValueError(f"Kernel function must have 2 parameters, got {len(params)}")
    for want, got in zip(("particles", "fieldset"), params, strict=True):
        if got.kind != inspect.Parameter.POSITIONAL_OR_KEYWORD:
            raise ValueError(f"Parameter '{got.name}' has incorrect parameter kind. Expected POSITIONAL_OR_KEYWORD, got {got.kind}")
        if got.name != want:
            raise ValueError(f"Parameter '{got.name}' has incorrect name. Expected '{want}', got '{got.name}'")


class KernelPlan:
    """The kernel list lowered to the fused device kernel's switches (include/parcels_b200.h)."""

    def __init__(self, kernel_list, fieldset, pclass=None):
        if isinstance(kernel_list, types.FunctionType):
            kernel_list = [kernel_list]
        if not isinstance(kernel_list, list):
            raise ValueError(f"kernels must be a list. Got {kernel_list=!r}")
        if len(kernel_list) == 0:
            raise ValueError("List of `kernels` should have at least one function.")
        for f in kernel_list:
            if not isinstance(f, types.FunctionType):
                raise TypeError(f"Argument `kernels` should be a function or list of functions. Got {type(f)}")
            _assert_kernel_signature(f)
        self.funcname = "".join(f.__name__ for f in kernel_list)
        tokens = [_builtin_name(f) for f in kernel_list]  # None for user functions (recognised by identity, not by name)
        names = list(tokens)
        self.delete_on_error = self.diffusion = False
        if names and names[-1] == "DeleteParticle":
            self.delete_on_error = True
            names = names[:-1]
        if names and names[-1] == "DiffusionUniformKh":
            self.diffusion = True
            names = names[:-1]
        if len(names) == 0 and self.diffusion:
            names = ["_none"]
        self.rk45 = None
        self.advdiff = None
        self._kernel_list, self._tokens = kernel_list, tokens
        if "AdvectionRK45" in tokens:
            self._setup_rk45(names, fieldset, pclass)
            return
        if len(names) == 1 and names[0] in K.ADVDIFF and not self.diffusion:
            self._setup_advdiff(names, fieldset)  # [kernel] or [kernel, DeleteParticle]: the whole loop in one launch
            return
        if "DiffusionUniformKh" in tokens and any(n in K.ADVDIFF for n in tokens if n):
            raise NotImplementedError("AdvectionDiffusionM1/EM already diffuse: combining them with DiffusionUniformKh is not supported")
        self.stepwise = not (len(names) == 1 and names[0] in K.SCHEMES)
        if fieldset.time_window is not None and not self.delete_on_error:
            # without the DeleteParticle token an error must stop the whole set at the end of its iteration; the fused kernel
            # could only replay that iteration from the start of the interval, whose time levels the window has left behind
            self.stepwise = True
        if self.stepwise:
            # the list mixes built-ins with user Python kernels: the loop control runs on the host step by step
            # (stepwise.py), every built-in kernel still runs on the device
            self.delete_on_error = self.diffusion = False
            self.items = []
            for f, n in zip(kernel_list, tokens, strict=True):
                if n in K.SCHEMES:
                    if n in K.SCHEMES_3D and fieldset.W is None:
                        raise AttributeError("FieldSet has no UVW VectorField (no W field) for a 3-D advection kernel")
                    self.items.append(["device", K.SCHEMES[n], False, self])
                elif n == "DiffusionUniformKh":
                    if self.items and self.items[-1][0] == "device" and not self.items[-1][2]:
                        self.items[-1][2] = True  # fused with the advection kernel right before it
                    else:
                        self.items.append(["device", K.SCHEMES["_none"], True, self])
                elif n in K.ADVDIFF:  # mixed with user kernels: one device launch per step (kernels_only)
                    self.items.append(["advdiff", _advdiff_params(fieldset, n)])
                elif n == "DeleteParticle":
                    self.items.append(["python", _delete_on_error])
                else:
                    self.items.append(["python", f])
            self.scheme_name, self.scheme = "stepwise", -1
        else:
            self.scheme_name = names[0]
            self.scheme = K.SCHEMES[names[0]]
            if names[0] in K.SCHEMES_3D and fieldset.W is None:
                raise AttributeError("FieldSet has no UVW VectorField (no W field) for a 3-D advection kernel")
        self.kh = (0.0, 0.0)
        self.kh_spherical = False
        self.kh_deg2m = 1.0
        if self.diffusion or (self.stepwise and any(i[0] == "device" and i[2] for i in self.items)):
            try:
                self.kh = (fieldset.constants["Kh_zonal"], fieldset.constants["Kh_meridional"])
            except KeyError as e:
                raise AttributeError("DiffusionUniformKh needs constant fields Kh_zonal and Kh_meridional") from e
            g = fieldset.Kh_zonal.grid
            self.kh_spherical = g.is_spherical()
            self.kh_deg2m = g.deg2m


def _setup_rk45(self, names, fieldset, pclass):
    """AdvectionRK45 (reference _core/kernel.py:134-159 `check_fieldsets_in_kernels`): needs a `next_dt` Variable; missing
    RK45_tol / RK45_min_dt / RK45_max_dt get the reference's defaults with a KernelWarning; on a spherical mesh the
    tolerance is converted to degrees -- like the reference, in place, every time a kernel list is built."""
    import warnings

    from .statuscodes import KernelWarning

    fused = names == ["AdvectionRK45"] and not self.diffusion
    if self.diffusion or any(n in K.SCHEMES or n in K.ADVDIFF or n == "DiffusionUniformKh" for n in names if n):
        raise NotImplementedError("AdvectionRK45 combines with user kernels and the DeleteParticle token, not with other built-in kernels")
    if pclass is None or "next_dt" not in [v.name for v in pclass.variables]:
        raise ValueError('ParticleClass requires a "next_dt" for AdvectionRK45 Kernel.')
    if not ((fieldset.interp_method in ("linear", "freeslip", "partialslip") and not fieldset.grid.curvilinear)
            or fieldset.interp_method == "cgrid_velocity"):  # fmt: skip
        raise NotImplementedError("AdvectionRK45 is implemented for XLinear_Velocity, XFreeslip or XPartialslip "
                                  "(rectilinear A-grids) or CGrid_Velocity (rectilinear and curvilinear C-grids)")
    ctx = fieldset.context
    if "RK45_tol" not in ctx:
        warnings.warn("Setting RK45 tolerance to 10 m. Use fieldset.add_context('RK45_tol', [distance]) to change.", KernelWarning, stacklevel=4)
        fieldset.add_context("RK45_tol", 10)
    if fieldset.grid.is_spherical() and not getattr(fieldset, "_context_is_reference", False):
        # (under parcels_b200.install() the context mirrors the reference FieldSet's, whose own Kernel.__init__ has converted it)
        ctx["RK45_tol"] = ctx["RK45_tol"] / fieldset.grid.deg2m
    if "RK45_min_dt" not in ctx:
        warnings.warn("Setting RK45 minimum timestep to 1 s. Use fieldset.add_context('RK45_min_dt', [timestep]) to change.", KernelWarning, stacklevel=4)
        fieldset.add_context("RK45_min_dt", 1)
    if "RK45_max_dt" not in ctx:
        warnings.warn("Setting RK45 maximum timestep to 1 day. Use fieldset.add_context('RK45_max_dt', [timestep]) to change.", KernelWarning, stacklevel=4)
        fieldset.add_context("RK45_max_dt", 60 * 60 * 24)
    self.rk45 = (float(ctx["RK45_tol"]), float(ctx["RK45_min_dt"]), float(ctx["RK45_max_dt"]))
    self.kh, self.kh_spherical, self.kh_deg2m = (0.0, 0.0), False, 1.0
    if fused:  # [AdvectionRK45] or [AdvectionRK45, DeleteParticle]: the whole loop in one launch
        self.stepwise = False
        self.scheme_name, self.scheme = "AdvectionRK45", K.RK45
        return
    # mixed with user kernels (the reference's own tests/test_advection.py:354-387: [AdvectionRK45, UpdateP]): the host drives the
    # loop, every iteration's RK45 attempts run on the device (pb_advect_rk45 with kernels_only)
    self.stepwise = True
    self.scheme_name, self.scheme = "stepwise", -1
    self.delete_on_error = False
    self.items = []
    for f, n in zip(self._kernel_list, self._tokens, strict=True):
        if n == "AdvectionRK45":
            self.items.append(["rk45", self.rk45])
        elif n == "DeleteParticle":
            self.items.append(["python", _delete_on_error])
        else:
            self.items.append(["python", f])
    self.rk45 = None  # (fused-path marker)


KernelPlan._setup_rk45 = _setup_rk45


def _advdiff_params(fieldset, name):
    """AdvectionDiffusionM1 / AdvectionDiffusionEM (reference kernels/_advectiondiffusion.py:21-117): need the scalar fields
    ``Kh_zonal`` / ``Kh_meridional`` on the fieldset's grid and the context value ``dres`` -> arguments of pb_advect_diffusion."""
    from .fieldset import Field

    kz, km = fieldset.fields.get("Kh_zonal"), fieldset.fields.get("Kh_meridional")
    if not isinstance(kz, Field) or not isinstance(km, Field):
        raise AttributeError(f"{name} needs fields Kh_zonal and Kh_meridional (FieldSet.add_field)")
    if kz._slot is None or km._slot is None or kz.interp_method != "linear" or km.interp_method != "linear":
        raise NotImplementedError(f"{name}: Kh_zonal / Kh_meridional must be XLinear scalar fields on the FieldSet's grid "
                                  "(FieldSet.add_field(name, data)); constant fields have no gradient -- use DiffusionUniformKh")  # fmt: skip
    if fieldset.grid.curvilinear or fieldset.interp_method not in ("linear", "cgrid_velocity"):
        raise NotImplementedError(f"{name} is implemented for rectilinear fields (XLinear_Velocity or CGrid_Velocity)")
    if kz.data.dtype != km.data.dtype or (kz.data.shape[0] > 1) != (km.data.shape[0] > 1):
        raise NotImplementedError("Kh_zonal and Kh_meridional must share dtype and time dimension")
    if "dres" not in fieldset.context:
        raise AttributeError(f"{name} needs fieldset.add_context('dres', <resolution of the Kh gradient>)")
    dres = fieldset.context["dres"]
    if isinstance(dres, np.generic) or not isinstance(dres, (int, float)):
        # a NumPy float64 scalar is a STRONG type: `particles.x + dres` would be a float64 array in the reference and the
        # whole kernel would run in other dtypes; the reference's own usage passes a Python float (tests/test_diffusion.py:65)
        raise NotImplementedError("fieldset.dres must be a Python float (fieldset.add_context('dres', float(...)))")
    return dict(scheme=K.ADVDIFF[name], kh_slots=(kz._slot, km._slot), dres=float(dres), deg2m_sq=pow(fieldset.grid.deg2m, 2))


def _setup_advdiff(self, names, fieldset):
    self.advdiff = _advdiff_params(fieldset, names[0])
    self.stepwise = False
    self.scheme_name, self.scheme = names[0], -2
    self.kh, self.kh_spherical, self.kh_deg2m = (0.0, 0.0), False, 1.0


KernelPlan._setup_advdiff = _setup_advdiff


class Kernel:
    """``Kernel(kernels=[...], pset=pset)`` as in the reference (_core/kernel.py:40-96): validates the list (functions with the
    ``(particles, fieldset)`` signature, RK45 prerequisites) and names it; ``pset.execute`` lowers the same list to device launches."""

    def __init__(self, kernels, pset):
        if not isinstance(kernels, list):
            raise ValueError(f"kernels must be a list. Got {kernels=!r}")
        for f in kernels:
            if not isinstance(f, types.FunctionType):
                raise TypeError(f"Argument `kernels` should be a function or list of functions. Got {type(f)}")
            _assert_kernel_signature(f)
        if len(kernels) == 0:
            raise ValueError("List of `kernels` should have at least one function.")
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
        return not plan.stepwise and plan.rk45 is None and not fs.grid.curvilinear and fs.time_window is None and len(self._pclass.extra) == 0

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
        if plan.rk45 is not None:
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
        hint_all_zero = False
        g = self.fieldset.grid
        if g.curvilinear:
            # the reference skips the hint test for the WHOLE batch when every hinted xi is 0
            # (`if np.any(xi)`, _core/index_search.py:269), e.g. on the first eval of a fresh set
            sign = 1 if dt > 0 else -1
            hint_all_zero = _hint_all_zero(ei_last, lambda s_: sign * (endtime - d["t"][s_]) >= 0, g.xdim)

        if on_device:  # a resident interval: no particle can be back on the first time level; the depth bit of the first interval holds
            two_levels = self.__dict__.get("_batch_levels_resident", 0) & 2
        else:
            two_levels = _batch_levels(self.fieldset, d, lambda: (1 if dt > 0 else -1) * (endtime - d["t"]) >= 0)
            self.__dict__["_batch_levels_resident"] = two_levels

        def args(max_iters=-1):
            if plan.advdiff is not None:
                return eng.make_advdiff_args(dt=dt, endtime=endtime, delete_on_error=plan.delete_on_error, seed=self.seed,
                                             rng_call=self._rng_call, max_iters=max_iters, batch_levels=two_levels,
                                             **plan.advdiff)  # fmt: skip
            return eng.make_args(plan.scheme, dt, endtime, diffusion=plan.diffusion, delete_on_error=plan.delete_on_error,
                                 kh=plan.kh, kh_spherical=plan.kh_spherical, kh_deg2m=plan.kh_deg2m, seed=self.seed,
                                 rng_call=self._rng_call, max_iters=max_iters, hint_all_zero=hint_all_zero,
                                 batch_levels=two_levels)  # fmt: skip

        needs_upload = not on_device and not (resident and self._device_synced and eng.particle_count() == n)
        if not on_device and self.__dict__.get("_dt_pending") is not None and not (
                needs_upload and self.pipeline_chunks > 1 and n >= self.PIPELINE_MIN_PARTICLES and plan.advdiff is None
                and self.fieldset.time_window is None):  # fmt: skip
            _fill(d["dt"], self.__dict__.pop("_dt_pending"))  # (not the pipelined path: the deferred fill is done here)
            self.__dict__["_dt_filled"] = (d["dt"], dt)
        # host arrays in (and out): cut into chunks whose copies run under the kernels of the other chunks (pb_advect_host)
        pipelined = (needs_upload and self.pipeline_chunks > 1 and n >= self.PIPELINE_MIN_PARTICLES and plan.advdiff is None
                     and self.fieldset.time_window is None)  # fmt: skip
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
                a = args(max_iters=max_iters)
                a.resume = int(resume)
                eng.advect_async(a)

            return self._advect_windowed(eng, d, dt, endtime, launch)

        # pb_advect_diffusion counts the iterations of a windowed call across its launches: its replay is exact as well
        replayable = not windowed or plan.advdiff is not None
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
        if rep["n_error"] > 0 and replayable:
            # The reference stops the whole set at the END of the first loop iteration in which any
            # particle is in an error state (kernel.py:239-245).  Replay from the start-of-interval copy up to
            # and including that iteration so every particle is left exactly where the reference leaves it.
            k = rep["first_error_iter"]
            rewind()
            downloaded = False
            rep = advance(k + 1)
            if rep["n_out_of_time"] > 0:
                # an out-of-interval sample flags the WHOLE evaluated view (index_search.py:85-86, field.py:31-44)
                rewind()
                advance(k)
                eng.flag_view_outside_time(dt, endtime)
        elif plan.delete_on_error and rep["n_out_of_time"] > 0 and replayable:
            # Same whole-view rule under the DeleteParticle handler: every particle evaluated in the first iteration in which ANY
            # particle sampled outside the time interval is flagged, hence deleted (field.py:31-44 then the handler) -- replay up
            # to that iteration, then delete the view.  (The lanes deleted their own out-of-interval particle; the others ran on.)
            k = rep["first_error_iter"]
            rewind()
            downloaded = False
            first = rep
            rep = advance(k)
            eng.delete_view_outside_time(dt, endtime)
            rep["n_deleted"] += 1
            rep["max_state"] = max(rep["max_state"], int(StatusCode.Delete))
            rep["n_out_of_time"] = first["n_out_of_time"]
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
        n = len(self)
        self._device_synced = False
        d["state"][:] = StatusCode.Evaluate
        if n == 0:
            return
        if np.isnan(d["t"]).any():
            raise ValueError(f"Time values for particles with indices {np.where(np.isnan(d['t']))[0]} cannot be NaN.")
        eng = self.fieldset.engine(self.device)
        eng.claim(self)
        ei_last = np.ascontiguousarray(d["ei"][:, -1])
        eng.upload_particles(d, ei_last)
        dt_arr = np.ascontiguousarray(d["dt"], dtype=np.float64)
        ndt_arr = np.ascontiguousarray(d["next_dt"], dtype=np.float64)
        tol, min_dt, max_dt = plan.rk45
        hint_all_zero = False
        if self.fieldset.grid.curvilinear:  # batch-level `if np.any(xi)` of the first evaluation (index_search.py:269)
            sign = 1 if dt > 0 else -1
            hint_all_zero = _hint_all_zero(ei_last, lambda s_: sign * (endtime - d["t"][s_]) >= 0, self.fieldset.grid.xdim)
        two_levels = _batch_levels(self.fieldset, d, lambda: (1 if dt > 0 else -1) * (endtime - d["t"]) >= 0)

        def launch(resume):  # (a resumed launch continues every particle's dt, next_dt and iteration count)
            return eng.advect_rk45(dt, endtime, tol, min_dt, max_dt, dt_arr, ndt_arr, next_dt_is_f32=d["next_dt"].dtype == np.float32,
                                   delete_on_error=plan.delete_on_error, hint_all_zero=hint_all_zero, batch_levels=two_levels,
                                   resume=resume)  # fmt: skip

        if self.fieldset.time_window is not None:
            rep = self._advect_windowed(eng, d, dt, endtime, launch, synchronous=True)
        else:
            rep = launch(False)
        self.last_report = rep
        eng.download_particles(d, ei_last)
        _store_ei(d, ei_last)
        d["dt"][:] = dt_arr  # RK45 mode: dt is NOT reset to the nominal step (kernel.py:224-226)
        d["next_dt"][:] = ndt_arr
        if rep["n_error"] > 0:
            stuck = np.where(d["state"] == StatusCode.Error)[0]
            raise RuntimeError(f"AdvectionRK45: particles {stuck[:10]} have dt == 0 before endtime={endtime}; the reference's loop "
                               "never terminates on them (kernel.py:199-203 clamps the dt of particles that finished an earlier "
                               "interval to 0 and RK45 mode never restores it).  Reset pset.dt before continuing.")  # fmt: skip
        if rep["max_state"] == StatusCode.Delete:
            dele = np.where(d["state"] == StatusCode.Delete)[0]
            if len(dele) > 0:
                self.remove_indices(dele)

    def _advect_windowed(self, eng, d, dt, endtime, launch, *, synchronous=False):
        """Time-slab streaming: advance until every particle reached ``endtime``, sliding the resident time levels as the
        particles' clock crosses them.  ``launch(resume)`` runs one launch of the call on the device particles -- pb_advect,
        pb_advect_diffusion or pb_advect_rk45 -- with ``resume`` from the second launch on.  An asynchronous launch returns
        None and the next level is copied while its kernel runs.  A ``synchronous`` one (pb_advect_rk45: it brings dt / next_dt
        back) returns its report; the next level is copied before it, under the kernel only when the level data is pinned."""
        fs = self.fieldset
        sign = 1 if dt > 0 else -1
        todo = sign * (endtime - d["t"]) >= 0
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
        fused = not plan.stepwise and plan.rk45 is None
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
