"""AdvectionDiffusionM1 / AdvectionDiffusionEM: the oracle restatement against what the reference's own Kernel.execute
produces with the same np.random stream (tests/golden/advdiff.npz, oracle/make_golden.py) -- bit-exact -- and the
host-side plan checks of the product."""

import os

import numpy as np
import pytest

import parcels_b200 as pb
from advdiff_run import run_oracle_advdiff
from oracle.make_golden import ADVDIFF_CASES

ERR_NAME = {60: "FieldOutOfBoundError", 61: "FieldOutOfBoundSurfaceError", 70: "OutsideTimeInterval", 51: "FieldInterpolationError"}


@pytest.mark.parametrize("name", list(ADVDIFF_CASES))
def test_oracle_advdiff_matches_reference_outputs(name, golden_dir):
    g = np.load(os.path.join(golden_dir, "advdiff.npz"))
    pd, err = run_oracle_advdiff(name)
    assert (ERR_NAME[err] if err else "") == str(g[f"{name}/error"])
    for k in ("particle_id", "state", "t", "dt", "ei", "x", "y", "z", "dx", "dy"):
        np.testing.assert_array_equal(pd[k], g[f"{name}/{k}"], err_msg=f"{name}:{k}")


def _fieldset(with_kh=True, dres=0.5):
    lon, lat = np.linspace(0, 10, 6), np.linspace(0, 5, 4)
    U = np.ones((1, 1, 4, 6), dtype=np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, U=U, V=U, mesh="spherical")
    if with_kh:
        fs.add_field("Kh_zonal", 10 * U)
        fs.add_field("Kh_meridional", 10 * U)
    if dres is not None:
        fs.add_context("dres", dres)
    return fs


def test_advdiff_plan_checks():
    from parcels_b200.particleset import KernelPlan

    plan = KernelPlan([pb.AdvectionDiffusionM1, pb.DeleteParticle], _fieldset())
    assert plan.advdiff == dict(scheme=0, kh_slots=(3, 4), dres=0.5, deg2m_sq=pow(_fieldset().grid.deg2m, 2))
    assert plan.kind == "advdiff" and plan.delete_on_error and not plan.stepwise
    assert KernelPlan([pb.AdvectionDiffusionEM], _fieldset()).advdiff["scheme"] == 1
    with pytest.raises(AttributeError, match="Kh_zonal"):
        KernelPlan([pb.AdvectionDiffusionM1], _fieldset(with_kh=False))
    with pytest.raises(AttributeError, match="dres"):
        KernelPlan([pb.AdvectionDiffusionEM], _fieldset(dres=None))
    with pytest.raises(NotImplementedError, match="Python float"):
        KernelPlan([pb.AdvectionDiffusionEM], _fieldset(dres=np.float64(0.5)))
    with pytest.raises(NotImplementedError):
        KernelPlan([pb.AdvectionDiffusionM1, pb.DiffusionUniformKh], _fieldset())
    fs = _fieldset(with_kh=False)
    fs.add_constant_field("Kh_zonal", 10.0)
    fs.add_constant_field("Kh_meridional", 10.0)
    with pytest.raises(NotImplementedError, match="DiffusionUniformKh"):
        KernelPlan([pb.AdvectionDiffusionM1], fs)
