"""GPU parity of scalar Field.eval (pb_sample_scalar): cell indices and states bit-exact, values bit-exact on the
cases below (IEEE +,-,*,/ only, in the reference's order and dtype) -- against the oracle and against the
reference's own outputs (tests/golden/scalar_eval.npz); plus a user sampling kernel in a mixed kernel list."""

import os

import numpy as np
import pytest

import parcels_b200 as pb
from engine_run import make_fieldset
from oracle import parcels_oracle as po
from oracle.make_golden import SCALAR_CASES, land_tracer_inputs, scalar_inputs
from oracle_run import load_case, oracle_fieldset
from device_trig import DeviceTrig
from oracle import trig

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", SCALAR_CASES)
def test_scalar_eval_matches_oracle_and_reference(name, golden_dir):
    g = np.load(os.path.join(golden_dir, "scalar_eval.npz"))
    c = load_case(name)
    ofs = oracle_fieldset(c)
    for T in (c["U"].shape[0], 1):
        P, tq = scalar_inputs(c, T)
        for how in ("linear", "nearest", "cgrid_tracer"):
            fs = make_fieldset(c)
            fs.add_field("P", P, interp_method=how)
            ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
            val = fs.P.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
            pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"])
            oval = po.eval_scalar(ofs, P, how, tq, pd["z"], pd["y"], pd["x"], po.View(pd, np.ones(len(pd["x"]), dtype=bool)))
            key = f"{name}/T{T}/{how}"
            assert val.dtype == oval.dtype == g[f"{key}/value"].dtype, key
            np.testing.assert_array_equal(ps._data["ei"], pd["ei"], err_msg=key)
            np.testing.assert_array_equal(ps._data["state"], pd["state"], err_msg=key)
            np.testing.assert_array_equal(val, oval, err_msg=key)
            np.testing.assert_array_equal(val, g[f"{key}/value"], err_msg=key)
            np.testing.assert_array_equal(ps._data["state"], g[f"{key}/state"], err_msg=key)
            # float64 sample positions (an RK stage position), hinted by the cells just found
            x2 = np.asarray(c["x"], dtype=np.float64) + 1e-3
            v2 = fs.P.eval(tq, np.asarray(c["z"], dtype=np.float64), np.asarray(c["y"], dtype=np.float64), x2, ps)
            pd2 = {k: v.copy() for k, v in pd.items()}
            o2 = po.eval_scalar(ofs, P, how, tq, np.asarray(c["z"], dtype=np.float64), np.asarray(c["y"], dtype=np.float64), x2,
                                po.View(pd2, np.ones(len(x2), dtype=bool)))  # fmt: skip
            np.testing.assert_array_equal(v2, o2, err_msg=key + " f64")
            np.testing.assert_array_equal(ps._data["ei"], pd2["ei"], err_msg=key + " f64")


@pytest.mark.parametrize("name", SCALAR_CASES)
def test_invdist_land_tracer_matches_oracle_and_reference(name, golden_dir):
    """XLinearInvdistLandTracer on the device (MODE 6 of agrid.cuh) on a field with land, samples exactly on nodes included."""
    g = np.load(os.path.join(golden_dir, "scalar_eval.npz"))
    c = load_case(name)
    ofs = oracle_fieldset(c)
    for T in (c["U"].shape[0], 1):
        P, tq, x, y = land_tracer_inputs(c, T)
        fs = make_fieldset(c)
        fs.add_field("P", P, interp_method="linear_invdist_land")
        ps = pb.ParticleSet(fs, x=x, y=y, z=c["z"], t=c["t"])
        val = fs.P.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
        pd = po.create_particle_data(x, y, c["z"], c["t"])
        oval = po.eval_scalar(ofs, P, "linear_invdist_land", tq, pd["z"], pd["y"], pd["x"], po.View(pd, np.ones(len(x), dtype=bool)))
        key = f"{name}/T{T}/linear_invdist_land"
        assert val.dtype == oval.dtype == g[f"{key}/value"].dtype, key
        np.testing.assert_array_equal(ps._data["ei"], pd["ei"], err_msg=key)
        np.testing.assert_array_equal(ps._data["state"], pd["state"], err_msg=key)
        np.testing.assert_array_equal(val, oval, err_msg=key)
        np.testing.assert_array_equal(val, g[f"{key}/value"], err_msg=key)


def test_user_sampling_kernel_in_a_mixed_list():
    """The common idiom `particles.p = fieldset.P[particles]` after an advection kernel: the built-in runs on the device,
    the sampling kernel's Field.eval too; compared with the oracle running the same list."""
    c = load_case("flat_f32c_f64d")
    P, _ = scalar_inputs(c, c["U"].shape[0])
    fs = make_fieldset(c)
    fs.add_field("P", P)
    pclass = pb.Particle.add_variable(pb.Variable("p", np.float32, initial=0))
    ps = pb.ParticleSet(fs, pclass=pclass, x=c["x"], y=c["y"], z=c["z"], t=c["t"])

    def SampleP(particles, fieldset):
        particles.p = fieldset.P[particles]

    def DeleteErr(particles, fieldset):
        particles[particles.state >= 50].state = 30

    ps.execute([pb.AdvectionRK4_3D, SampleP, DeleteErr], dt=c["dt"], runtime=50.0)

    ofs = oracle_fieldset(c)
    pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"])
    pd["p"] = np.zeros(len(pd["x"]), dtype=np.float32)

    def OSample(p, fs_):
        p.p = po.eval_scalar(fs_, P, "linear", p.t, p.z, p.y, p.x, p)

    po.pset_execute(pd, ofs, [po.AdvectionRK4_3D, OSample, po.DeleteOnError], c["dt"], runtime=50.0)
    assert len(ps) == len(pd["x"]) and len(ps) > 0
    for k in ("particle_id", "state", "t", "ei", "x", "y", "z", "p"):
        np.testing.assert_array_equal(ps._data[k], pd[k], err_msg=k)
    assert np.abs(ps._data["p"]).max() > 0


@pytest.mark.parametrize("name", ["curv_sph_2d", "curv_flat_2d", "curv_sph_3d", "curv_sph_f32", "curv_sph_dateline"])
def test_scalar_eval_on_curvilinear_grids(name, golden_dir):
    """CGrid_Tracer / XNearest on curvilinear C-grids (NEMO tracers on an ORCA grid): a fresh set -- the whole batch through the
    spatial hash, like the reference -- and a displaced float64 evaluation hinted by the cells just found; values, cells and
    states equal the oracle's and the reference's own (tests/golden/scalar_eval_curv.npz)."""
    g = np.load(os.path.join(golden_dir, "scalar_eval_curv.npz"))
    c = load_case(name)
    ofs = oracle_fieldset(c)
    for T in (c["U"].shape[0], 1):
        P, tq = scalar_inputs(c, T)
        for how in ("nearest", "cgrid_tracer"):
            fs = make_fieldset(c)
            fs.add_field("P", P, interp_method=how)
            ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
            v1 = fs.P.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
            ei1 = ps._data["ei"].copy()
            x2 = np.asarray(ps._data["x"], dtype=np.float64) + 0.3 * float(np.abs(np.diff(np.asarray(c["lon"], dtype=np.float64), axis=1)).mean())
            v2 = fs.P.eval(tq, ps._data["z"], np.asarray(ps._data["y"], dtype=np.float64), x2, ps)
            key = f"{name}/T{T}/{how}"
            assert v1.dtype == g[f"{key}/value"].dtype and v2.dtype == g[f"{key}/value2"].dtype, key
            np.testing.assert_array_equal(v1, g[f"{key}/value"], err_msg=key)
            np.testing.assert_array_equal(ei1, g[f"{key}/ei"], err_msg=key)
            np.testing.assert_array_equal(v2, g[f"{key}/value2"], err_msg=key + " second")
            np.testing.assert_array_equal(ps._data["ei"], g[f"{key}/ei2"], err_msg=key + " second")
            np.testing.assert_array_equal(ps._data["state"], g[f"{key}/state2"], err_msg=key + " second")
    with pytest.raises(NotImplementedError, match="cgrid_tracer"):
        make_fieldset(c).add_field("Q", P, interp_method="linear_invdist_land")


CURV_SCALAR = ["curv_sph_2d", "curv_flat_2d", "curv_sph_3d", "curv_sph_f32", "curv_sph_dateline"]


@pytest.mark.parametrize("name, exact", [pytest.param(n, False, id=n) for n in CURV_SCALAR] + [pytest.param(n, True, id=f"{n}-exact") for n in CURV_SCALAR])
def test_xlinear_scalar_eval_on_curvilinear_grids(name, exact, golden_dir):
    """XLinear behind the curvilinear search (an A-grid tracer on 2-D lon / lat), against the reference's own values
    (tests/golden/scalar_eval_curv_linear.npz): cells and states bit-exact; values within 64 float32 ulp of the field's range --
    the barycentric coordinates come out of the closed-form bilinear inverse (last-ulp trig differences amplified, hash hits
    rounded to float32: the curvilinear tolerance of the trajectory tests), and the reference's float32-TYPED coordinates after
    a hash hit (DESIGN.md waiver 4) are float32-rounded float64 values here, so the value is always float64.  `exact`: the values
    are compared bit for bit with the oracle in engine arithmetic instead (the scalar sampler's own trigonometry and waiver 4's
    resolution, tests/device_trig.py)."""
    g = np.load(os.path.join(golden_dir, "scalar_eval_curv_linear.npz"))
    c = load_case(name)
    for T in (c["U"].shape[0], 1):
        P, tq = scalar_inputs(c, T)
        fs = make_fieldset(c)
        fs.add_field("P", P, interp_method="linear")
        ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
        v1 = fs.P.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
        ei1 = ps._data["ei"].copy()
        x2 = np.asarray(ps._data["x"], dtype=np.float64) + 0.3 * float(np.abs(np.diff(np.asarray(c["lon"], dtype=np.float64), axis=1)).mean())
        v2 = fs.P.eval(tq, ps._data["z"], np.asarray(ps._data["y"], dtype=np.float64), x2, ps)
        key = f"{name}/T{T}/linear"
        tol = 64 * np.finfo(np.float32).eps * float(np.abs(P).max())
        np.testing.assert_array_equal(ei1, g[f"{key}/ei"], err_msg=key)
        np.testing.assert_array_equal(ps._data["ei"], g[f"{key}/ei2"], err_msg=key + " second")
        np.testing.assert_array_equal(ps._data["state"], g[f"{key}/state2"], err_msg=key + " second")
        if exact:
            ofs = oracle_fieldset(c)
            pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"], ngrids=ofs.ngrids)
            view = po.View(pd, np.ones(len(pd["x"]), dtype=bool))
            with trig.use(DeviceTrig(scalar_sampler=True)):
                o1 = po.eval_scalar(ofs, P, "linear", tq, pd["z"], pd["y"], pd["x"], view)
                np.testing.assert_array_equal(ei1, pd["ei"], err_msg=key)
                o2 = po.eval_scalar(ofs, P, "linear", tq, pd["z"], np.asarray(pd["y"], dtype=np.float64), x2, view)
            np.testing.assert_array_equal(ps._data["ei"], pd["ei"], err_msg=key + " second")
            np.testing.assert_array_equal(ps._data["state"], pd["state"], err_msg=key + " second")
            np.testing.assert_array_equal(v1, o1, err_msg=key)
            np.testing.assert_array_equal(v2, o2, err_msg=key + " second")
            continue
        np.testing.assert_allclose(v1, g[f"{key}/value"].astype(np.float64), rtol=0, atol=tol, err_msg=key)
        np.testing.assert_allclose(v2, g[f"{key}/value2"].astype(np.float64), rtol=0, atol=tol, err_msg=key + " second")
        assert np.abs(g[f"{key}/value"]).max() > 0
