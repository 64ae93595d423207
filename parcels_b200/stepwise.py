"""``Kernel.execute`` for kernel lists that mix built-in kernels with USER Python kernels
(the common idiom of the reference's own tests, e.g. ``[AdvectionRK4_3D, DeleteParticle]`` with a user-defined
handler, periodic-boundary or ageing kernels; reference ``_core/kernel.py:174-247``).

The loop control of one ``Kernel.execute`` call runs here, step by step, exactly as in the reference; every
BUILT-IN kernel of the list is still executed on the device (``pb_advect(kernels_only=1)``: one iteration's kernel
functions on the evaluated particles), user functions are called on the host with a ``ParticleSetView``.  The
price is one host<->device round trip of the particle SoA per time step; lists made of built-ins only come here only
on a time-windowed FieldSet without the DeleteParticle token (elsewhere they run the whole loop in one kernel launch).

On a time-windowed FieldSet every device launch of an iteration first makes the levels of the evaluated particles'
steps [t, t + dt] resident (``FieldSet.cover_window``); user kernels' ``fieldset.UV[...]`` do the same for their own
sample times.  An iteration whose particles are spread over more time levels than the window holds raises.
"""

from __future__ import annotations

import numpy as np

from .particlesetview import ParticleSetView
from .plan import PythonStep, Rk45Step, batch_facts
from .statuscodes import ERRORS_TO_THROW, StatusCode, raise_for_state


def kernel_execute_stepwise(pset, plan, endtime: float, dt: float):
    d = pset._data
    fs = pset.fieldset
    eng = fs.engine(pset.device)
    eng.claim(pset)
    sign = 1 if dt > 0 else -1
    d["state"][:] = StatusCode.Evaluate
    steps = 0
    # RK45 mode (reference kernel.py:118-120,224-226: `hasattr(fieldset, "RK45_tol")`): dt <- next_dt after the position update,
    # and dt is NOT reset to the nominal step at the end of the iteration
    rk45_mode = "RK45_tol" in fs.context
    while len(d["x"]) > 0 and np.any(np.isin(d["state"], [StatusCode.Evaluate, StatusCode.Repeat])):
        tte = sign * (endtime - d["t"])
        evaluate = np.isin(d["state"], [StatusCode.Success, StatusCode.Evaluate]) & (tte >= 0)
        if not np.any(evaluate):
            break
        # adapt dt to end exactly on endtime (kernel.py:199-203)
        d["dt"][:] = np.maximum(np.minimum(d["dt"], tte), 0) if sign == 1 else np.minimum(np.maximum(d["dt"], -tte), 0)
        steps += int(np.count_nonzero(evaluate))
        for step in plan.items:
            if not isinstance(step, PythonStep) and fs.time_window is not None:
                _cover_steps(pset, evaluate, sign)
            if isinstance(step, Rk45Step):
                pset._advect_rk45(plan, eng, dt, endtime, stepwise=True)
            elif not isinstance(step, PythonStep):
                _device_kernels(pset, eng, plan, step, dt, endtime)
            else:
                f = step.func
                f(ParticleSetView(d, evaluate, fs), fs)
                repeat = d["state"] == StatusCode.Repeat
                while np.any(repeat):  # kernel.py:213-216
                    f(ParticleSetView(d, repeat, fs), fs)
                    repeat = d["state"] == StatusCode.Repeat
        # position update only for particles still in a normal state (kernel.py:108-116,220-222)
        upd = evaluate & np.isin(d["state"], [StatusCode.Evaluate, StatusCode.Success])
        if np.any(upd):
            d["x"][upd] += d["dx"][upd]
            d["y"][upd] += d["dy"][upd]
            d["z"][upd] += d["dz"][upd]
            d["t"][upd] += d["dt"][upd]
            d["dx"][upd] = 0
            d["dy"][upd] = 0
            d["dz"][upd] = 0
            if rk45_mode:
                d["dt"][upd] = d["next_dt"][upd]
        if not rk45_mode:
            d["dt"][:] = dt
        d["state"][(d["state"] == StatusCode.Evaluate) & (d["t"] == endtime)] = StatusCode.EndofLoop
        dele = np.where(d["state"] == StatusCode.Delete)[0]
        if len(dele) > 0:
            pset.remove_indices(dele)
            d = pset._data
        if np.any(d["state"] == StatusCode.StopAllExecution):
            break
        for code in ERRORS_TO_THROW:
            hit = d["state"] == code
            if np.any(hit):
                raise_for_state(code, d["z"][hit], d["y"][hit], d["x"][hit], d["t"][hit])
    pset.last_report = dict(particle_steps=steps, mode="stepwise")


def _cover_steps(pset, evaluate, sign):
    """Time-windowed U, V, W: make the levels of this iteration's steps [t, t + dt] (dt after the endtime clamp) of the
    evaluated particles resident -- the part of them inside the time axis (outside it is OutsideTimeInterval)."""
    fs = pset.fieldset
    d = pset._data
    ta = d["t"][evaluate]
    tb = ta + d["dt"][evaluate]
    lo, hi = np.minimum(ta, tb), np.maximum(ta, tb)
    t0, t1 = float(fs._time_s[0]), float(fs._time_s[-1])
    meets = (hi >= t0) & (lo <= t1)
    if np.any(meets):
        fs.cover_window(pset.device, np.clip([lo[meets].min(), hi[meets].max()], t0, t1), sign)


def _no_wait(rep):
    if rep["n_wait_window"] > 0:  # (the iteration's levels were made resident before the launch)
        raise RuntimeError(f"{rep['n_wait_window']} particles found their time levels not resident: widen time_window")


def _device_kernels(pset, eng, plan, step, dt, endtime):
    """One iteration of the built-in kernels ``step`` (a FixedStep or an AdvDiffStep of ``plan``) on the device: the kernel
    applies the reference's own evaluate mask (state in {Success, Evaluate} and time-to-endtime >= 0) and dt clamp, accumulates
    dx/dy/dz and updates state/ei; nothing else."""
    d = pset._data
    pset._rng_call += 1
    ei_last = np.ascontiguousarray(d["ei"][:, -1])
    hint_all_zero, two_levels = batch_facts(pset.fieldset, d, ei_last, dt, endtime, mid_iteration=True)
    eng.upload_particles(d, ei_last)
    rep = eng.advect(plan.launch_args(eng, dt, endtime, step=step, seed=pset.seed, rng_call=pset._rng_call, hint_all_zero=hint_all_zero,
                                      batch_levels=two_levels, resume=True, kernels_only=True))  # fmt: skip
    _no_wait(rep)
    eng.download_particles(d, ei_last)
    d["ei"][:, -1] = ei_last
    if rep["n_out_of_time"] > 0:  # the reference flags the whole evaluated view (index_search.py:85-86, field.py:31-44)
        sign = 1 if dt > 0 else -1
        view = np.isin(d["state"], [StatusCode.Success, StatusCode.Evaluate, StatusCode.ErrorOutsideTimeInterval]) & (
            sign * (endtime - d["t"]) >= 0
        )
        d["state"][view] = StatusCode.ErrorOutsideTimeInterval
