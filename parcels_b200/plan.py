"""A kernel list lowered once into a typed plan, the argument struct of every device launch built from it, and the batch-level
facts of a launch (the reference's per-batch decisions a lane cannot make by itself)."""

from __future__ import annotations

import types
from typing import NamedTuple

import numpy as np

from . import kernels as K
from .statuscodes import StatusCode


def _min_or_max(t, want_min: bool) -> float:
    """``t.min()`` / ``t.max()`` with NumPy's NaN propagation (any NaN -> NaN), as the reference takes them (particleset.py:541-544).
    (NumPy's own SIMD reduction: 3.5 ms for 1e7 values; a threaded scalar loop in the library measured 15 ms.)"""
    return float(t.min() if want_min else t.max())


def evaluated_mask(d, dt, endtime, rows=slice(None), mid_iteration=False):
    """The particles (of ``rows``) a launch evaluates: time left to ``endtime`` in the direction of ``dt`` (kernel.py:190-197);
    ``mid_iteration`` (one iteration of a stepwise list) also requires a state in {Success, Evaluate}."""
    sign = 1 if dt > 0 else -1
    mask = sign * (endtime - d["t"][rows]) >= 0
    if mid_iteration:
        mask &= np.isin(d["state"][rows], [StatusCode.Success, StatusCode.Evaluate])
    return mask


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
    te = t[evaluated()]
    return bool(te.size) and bool(np.any(te != float(fieldset._time_s[0])))


def _batch_levels(fieldset, d, evaluated) -> int:
    """``pb_advect_args.batch_levels``.  PB_BATCH_FIRST_EVAL_TWO_T (1): see `_first_eval_two_levels`.  PB_BATCH_TWO_Z (2):
    `lenZ = 2 if any(zeta > 0)` (_xinterpolators.py:401) -- with XFreeslip / XPartialslip the land test then looks at the second
    depth level for every particle of the batch (:426-447); zeta > 0 means below the first depth level (left-sided search), taken
    as constant over the call.  ``evaluated()`` makes the mask of the evaluated particles on demand."""
    flags = 1 if _first_eval_two_levels(fieldset, d["t"], evaluated) else 0
    depth = fieldset.grid.depth
    if fieldset.interp_method in ("freeslip", "partialslip") and depth is not None and len(depth) > 1:
        ze = d["z"][evaluated()]
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


def batch_facts(fieldset, d, ei_last, dt, endtime, *, mid_iteration=False) -> tuple[bool, int]:
    """``(hint_all_zero, batch_levels)`` of a launch over the particles ``d`` (``ei_last``: their last grid's cells): the reference's
    batch-level decisions of the launch's first evaluation.  The evaluated mask is only made when a decision needs it."""
    mask = lambda rows=slice(None): evaluated_mask(d, dt, endtime, rows, mid_iteration)  # noqa: E731
    g = fieldset.grid
    return bool(g.curvilinear and _hint_all_zero(ei_last, mask, g.xdim)), _batch_levels(fieldset, d, mask)


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


# the items of a stepwise plan, in list order: one iteration of each runs on the device, PythonStep on the host
class FixedStep(NamedTuple):
    """A fixed-step advection scheme (``K.SCHEMES``; "_none": DiffusionUniformKh alone), fused with DiffusionUniformKh."""

    scheme: int
    diffusion: bool


class AdvDiffStep(NamedTuple):
    """AdvectionDiffusionM1 / EM: the arguments of pb_advect_diffusion (`_advdiff_params`)."""

    params: dict


class Rk45Step(NamedTuple):
    """AdvectionRK45, with the plan's ``rk45`` tolerances."""


class PythonStep(NamedTuple):
    """A user kernel (or the DeleteParticle token), called on the host with a ParticleSetView."""

    func: types.FunctionType


class KernelPlan:
    """The kernel list lowered to the device kernels' switches (include/parcels_b200.h).  ``kind`` is the route of a Kernel.execute:

    * "fixed": one fixed-step scheme (``scheme``), optionally with DiffusionUniformKh (``diffusion``), the whole loop in one launch;
    * "rk45": [AdvectionRK45], the whole loop in one launch (pb_advect_rk45);
    * "advdiff": [AdvectionDiffusionM1 | EM], the whole loop in one launch (pb_advect_diffusion, ``advdiff``);
    * "stepwise": the host drives the loop (stepwise.py) over ``items``.

    Every kind may end with the DeleteParticle token (``delete_on_error``, never set on "stepwise": there it is a PythonStep)."""

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
        self.scheme = self.rk45 = self.advdiff = None
        self.items = ()
        self.kh, self.kh_spherical, self.kh_deg2m = (0.0, 0.0), False, 1.0
        self.next_dt_dtype = None  # (AdvectionRK45: the dtype of the next_dt Variable)
        self.batch_levels = 0  # the call's batch-level bits where all launches of a call share them (mode D, distributed.py)
        self.hint_all_zero = False  # mode D on column slabs: the whole set's hint_all_zero of the call's first evaluation
        if "AdvectionRK45" in tokens:
            self._setup_rk45(names, fieldset, pclass)
            # [AdvectionRK45] or [AdvectionRK45, DeleteParticle]: the whole loop in one launch.  Mixed with user kernels (the
            # reference's own tests/test_advection.py:354-387: [AdvectionRK45, UpdateP]) the host drives the loop, every
            # iteration's RK45 attempts run on the device (pb_advect_rk45 with kernels_only)
            self.kind = "rk45" if names == ["AdvectionRK45"] else "stepwise"
        elif len(names) == 1 and names[0] in K.ADVDIFF and not self.diffusion:
            self.advdiff = _advdiff_params(fieldset, names[0])  # [kernel] or [kernel, DeleteParticle]: the whole loop in one launch
            self.kind = "advdiff"
        else:
            if "DiffusionUniformKh" in tokens and any(n in K.ADVDIFF for n in tokens if n):
                raise NotImplementedError("AdvectionDiffusionM1/EM already diffuse: combining them with DiffusionUniformKh is not supported")
            # without the DeleteParticle token on a time-windowed FieldSet an error must stop the whole set at the end of its
            # iteration; the fused kernel could only replay that iteration from the start of the interval, whose time levels the
            # window has left behind
            fused = len(names) == 1 and names[0] in K.SCHEMES and (fieldset.time_window is None or self.delete_on_error)
            self.kind = "fixed" if fused else "stepwise"
            if fused:
                self.scheme = K.SCHEMES[names[0]]
                if names[0] in K.SCHEMES_3D and fieldset.W is None:
                    raise AttributeError("FieldSet has no UVW VectorField (no W field) for a 3-D advection kernel")
        if self.kind == "stepwise":
            # the list mixes built-ins with user Python kernels: the loop control runs on the host step by step
            # (stepwise.py), every built-in kernel still runs on the device
            self.delete_on_error = self.diffusion = False
            self.items = self._steps(kernel_list, tokens, fieldset)
        if self.diffusion or any(isinstance(s, FixedStep) and s.diffusion for s in self.items):
            try:
                self.kh = (fieldset.constants["Kh_zonal"], fieldset.constants["Kh_meridional"])
            except KeyError as e:
                raise AttributeError("DiffusionUniformKh needs constant fields Kh_zonal and Kh_meridional") from e
            g = fieldset.Kh_zonal.grid
            self.kh_spherical = g.is_spherical()
            self.kh_deg2m = g.deg2m

    @property
    def stepwise(self) -> bool:
        return self.kind == "stepwise"

    @staticmethod
    def _steps(kernel_list, tokens, fieldset) -> tuple:
        steps = []
        for f, n in zip(kernel_list, tokens, strict=True):
            if n == "AdvectionRK45":
                steps.append(Rk45Step())
            elif n in K.SCHEMES:
                if n in K.SCHEMES_3D and fieldset.W is None:
                    raise AttributeError("FieldSet has no UVW VectorField (no W field) for a 3-D advection kernel")
                steps.append(FixedStep(K.SCHEMES[n], False))
            elif n == "DiffusionUniformKh":
                if steps and isinstance(steps[-1], FixedStep) and not steps[-1].diffusion:
                    steps[-1] = steps[-1]._replace(diffusion=True)  # fused with the advection kernel right before it
                else:
                    steps.append(FixedStep(K.SCHEMES["_none"], True))
            elif n in K.ADVDIFF:  # mixed with user kernels: one device launch per step (kernels_only)
                steps.append(AdvDiffStep(_advdiff_params(fieldset, n)))
            else:
                steps.append(PythonStep(_delete_on_error if n == "DeleteParticle" else f))
        return tuple(steps)

    def _setup_rk45(self, names, fieldset, pclass):
        """AdvectionRK45 (reference _core/kernel.py:134-159 `check_fieldsets_in_kernels`): needs a `next_dt` Variable; missing
        RK45_tol / RK45_min_dt / RK45_max_dt get the reference's defaults with a KernelWarning; on a spherical mesh the
        tolerance is converted to degrees -- like the reference, in place, every time a kernel list is built."""
        import warnings

        from .statuscodes import KernelWarning

        if self.diffusion or any(n in K.SCHEMES or n in K.ADVDIFF or n == "DiffusionUniformKh" for n in names if n):
            raise NotImplementedError("AdvectionRK45 combines with user kernels and the DeleteParticle token, not with other built-in kernels")
        next_dt = [v for v in (pclass.variables if pclass is not None else ()) if v.name == "next_dt"]
        if not next_dt:
            raise ValueError('ParticleClass requires a "next_dt" for AdvectionRK45 Kernel.')
        self.next_dt_dtype = np.dtype(next_dt[0].dtype)
        if not ((fieldset.interp_method in ("linear", "freeslip", "partialslip") and not fieldset.grid.curvilinear)
                or fieldset.interp_method == "cgrid_velocity"):  # fmt: skip
            raise NotImplementedError("AdvectionRK45 is implemented for XLinear_Velocity, XFreeslip or XPartialslip "
                                      "(rectilinear A-grids) or CGrid_Velocity (rectilinear and curvilinear C-grids)")
        ctx = fieldset.context
        if "RK45_tol" not in ctx:
            warnings.warn("Setting RK45 tolerance to 10 m. Use fieldset.add_context('RK45_tol', [distance]) to change.",
                          KernelWarning, stacklevel=4)  # fmt: skip
            fieldset.add_context("RK45_tol", 10)
        if fieldset.grid.is_spherical() and not getattr(fieldset, "_context_is_reference", False):
            # (under parcels_b200.install() the context mirrors the reference FieldSet's, whose own Kernel.__init__ has converted it)
            ctx["RK45_tol"] = ctx["RK45_tol"] / fieldset.grid.deg2m
        if "RK45_min_dt" not in ctx:
            warnings.warn("Setting RK45 minimum timestep to 1 s. Use fieldset.add_context('RK45_min_dt', [timestep]) to change.",
                          KernelWarning, stacklevel=4)  # fmt: skip
            fieldset.add_context("RK45_min_dt", 1)
        if "RK45_max_dt" not in ctx:
            warnings.warn("Setting RK45 maximum timestep to 1 day. Use fieldset.add_context('RK45_max_dt', [timestep]) to change.",
                          KernelWarning, stacklevel=4)  # fmt: skip
            fieldset.add_context("RK45_max_dt", 60 * 60 * 24)
        self.rk45 = (float(ctx["RK45_tol"]), float(ctx["RK45_min_dt"]), float(ctx["RK45_max_dt"]))

    def launch_args(self, eng, dt, endtime, *, step=None, seed=0, rng_call=0, batch_levels=0, hint_all_zero=False, max_iters=-1,
                    resume=False, kernels_only=False, next_dt_dtype=None):  # fmt: skip
        """The argument struct of one device launch of this plan -- of its stepwise item ``step`` when given: ``AdvectArgs``,
        ``AdvDiffArgs`` or ``Rk45Args`` (``next_dt_dtype``: that of the particles' next_dt column)."""
        if self.rk45 is not None:  # (AdvectionRK45 is the only device kernel of its list)
            return eng.make_rk45_args(dt, endtime, *self.rk45, next_dt_is_f32=next_dt_dtype == np.float32,
                                      delete_on_error=self.delete_on_error, max_iters=max_iters, kernels_only=kernels_only,
                                      resume=resume, hint_all_zero=hint_all_zero, batch_levels=batch_levels)  # fmt: skip
        if self.kind == "advdiff" or isinstance(step, AdvDiffStep):
            return eng.make_advdiff_args(dt=dt, endtime=endtime, delete_on_error=self.delete_on_error, seed=seed, rng_call=rng_call,
                                         max_iters=max_iters, kernels_only=kernels_only, resume=resume, batch_levels=batch_levels,
                                         **(self.advdiff if step is None else step.params))  # fmt: skip
        scheme, diffusion = (self.scheme, self.diffusion) if step is None else step
        return eng.make_args(scheme, dt, endtime, diffusion=diffusion, delete_on_error=self.delete_on_error, kh=self.kh,
                             kh_spherical=self.kh_spherical, kh_deg2m=self.kh_deg2m, seed=seed, rng_call=rng_call, max_iters=max_iters,
                             hint_all_zero=hint_all_zero, resume=resume, kernels_only=kernels_only, batch_levels=batch_levels)  # fmt: skip
