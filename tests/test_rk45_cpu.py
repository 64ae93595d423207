"""AdvectionRK45 + the Repeat / next_dt state machine: the oracle restatement against what the reference's own
Kernel.execute produces (tests/golden/rk45.npz, oracle/make_golden.py) -- positions, times, the per-particle dt and
next_dt the reference leaves behind, states, cell indices: all bit-exact."""

import os

import numpy as np
import pytest

import parcels_b200 as pb
from oracle import parcels_oracle as po
from oracle.make_golden import RK45_CASES
from oracle_run import load_case, oracle_fieldset


def run_oracle_rk45(name, count=None):
    tol, min_dt, fmax, runtime, dt = RK45_CASES[name]
    c = load_case(name)
    ofs = oracle_fieldset(c)
    if ofs.grid.spherical:
        tol = tol / ofs.grid.deg2m  # kernel.py:144-145
    ofs.context.update(RK45_tol=tol, RK45_min_dt=min_dt, RK45_max_dt=fmax * abs(dt))
    pd = po.create_particle_data(c["x"], c["y"], np.abs(np.asarray(c["z"])), c["t"])
    pd["next_dt"] = np.zeros(len(pd["x"]), dtype=np.float32)

    def Kernel(p, fs):
        if count is not None:
            count[0] += p.n()
        po.AdvectionRK45(p, fs)

    steps = po.pset_execute(pd, ofs, [Kernel], dt, runtime=runtime)
    return c, pd, steps, tol


@pytest.mark.parametrize("name", list(RK45_CASES))
def test_oracle_rk45_matches_reference_outputs(name, golden_dir):
    g = np.load(os.path.join(golden_dir, "rk45.npz"))
    attempts = [0]
    _, pd, steps, tol = run_oracle_rk45(name, attempts)
    assert tol == float(g[f"{name}/tol_used"])
    for k in ("x", "y", "z", "t", "dt", "next_dt", "state", "ei"):
        np.testing.assert_array_equal(pd[k], g[f"{name}/{k}"], err_msg=f"{name}:{k}")
    assert attempts[0] > steps  # the case exercises rejected steps (state Repeat)


def test_rk45_plan_checks():
    from parcels_b200.particleset import KernelPlan

    lon, lat = np.linspace(0, 10, 6), np.linspace(0, 5, 4)
    U = np.ones((1, 1, 4, 6), dtype=np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, U=U, V=U, mesh="spherical")
    with pytest.raises(ValueError, match='ParticleClass requires a "next_dt" for AdvectionRK45 Kernel.'):
        KernelPlan([pb.AdvectionRK45], fs, pb.Particle)  # reference tests/test_kernel.py:107-112
    P = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=1))
    with pytest.warns(pb.KernelWarning):  # reference tests/test_kernel.py:115-124: defaults are set with a warning
        plan = KernelPlan([pb.AdvectionRK45, pb.DeleteParticle], fs, P)
    assert fs.context["RK45_min_dt"] == 1 and fs.context["RK45_max_dt"] == 86400
    assert fs.context["RK45_tol"] == 10 / fs.grid.deg2m and plan.rk45 == (10 / fs.grid.deg2m, 1.0, 86400.0)
    assert plan.kind == "rk45" and plan.delete_on_error and not plan.stepwise
    with pytest.raises(NotImplementedError):
        KernelPlan([pb.AdvectionRK45, pb.DiffusionUniformKh], fs, P)
