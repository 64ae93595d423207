"""GPU parity of AdvectionRK45 (pb_advect_rk45: the Repeat / next_dt state machine in one device kernel) against the
oracle and against the reference's own outputs (tests/golden/rk45.npz): positions bit-exact on flat meshes and <= 2
float32 ulp on spherical ones; times, per-particle dt and next_dt, states and cell indices bit-exact; the number of
RK45 attempts (accepted + rejected) equal to the oracle's.  In engine arithmetic (``-exact`` ids: the oracle's sin / cos are the
device's own functions, tests/device_trig.py) the spherical and curvilinear cases are bit-exact as well, with the same number of
attempts and no particle left out of the comparison."""

import os

import numpy as np
import pytest

import cases
import parcels_b200 as pb
from device_trig import DeviceTrig
from oracle import parcels_oracle as po
from oracle import trig
from engine_run import make_fieldset, ulp_diff_f32
from oracle.make_golden import RK45_CASES
from oracle_run import load_case, oracle_fieldset
from test_rk45_cpu import run_oracle_rk45

pytestmark = pytest.mark.gpu
NEXT_DT = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0))


def _flat_rectilinear(name):
    return cases.CASES[name]["mesh"] == "flat" and not name.startswith("curv")


RK45_MODES = [pytest.param(n, False, id=n) for n in RK45_CASES] + [
    pytest.param(n, True, id=f"{n}-exact") for n in RK45_CASES if not _flat_rectilinear(n)
]


def _engine_rk45(name, kernels=None, exact=False):
    tol, min_dt, fmax, runtime, dt = RK45_CASES[name]
    attempts = [0]
    with trig.use(DeviceTrig() if exact else trig.NumpyTrig()):
        c, pd, steps, _ = run_oracle_rk45(name, attempts)
    c = dict(c, W=None)
    fs = make_fieldset(c)
    fs.add_context("RK45_tol", tol)  # metres: converted to degrees when the kernel list is built, like the reference
    fs.add_context("RK45_min_dt", min_dt)
    fs.add_context("RK45_max_dt", fmax * abs(dt))
    ps = pb.ParticleSet(fs, pclass=NEXT_DT, x=c["x"], y=c["y"], z=np.abs(np.asarray(c["z"])), t=c["t"])
    ps.execute(kernels or pb.AdvectionRK45, dt=dt, runtime=runtime)
    return c, ps, pd, steps, attempts[0]


@pytest.mark.parametrize("name, engine_arithmetic", RK45_MODES)
def test_rk45_matches_oracle_and_reference(name, engine_arithmetic, golden_dir):
    g = np.load(os.path.join(golden_dir, "rk45.npz"))
    c, ps, pd, steps, attempts = _engine_rk45(name, exact=engine_arithmetic)
    d = ps._data
    assert ps.last_report["particle_steps"] == steps
    curv = name.startswith("curv")
    if engine_arithmetic:
        for k in ("x", "y", "z", "t", "dt", "next_dt", "state", "ei"):
            np.testing.assert_array_equal(d[k], pd[k], err_msg=f"{name}:{k}")
        assert ps.last_report["cache_refills"] == 6 * attempts  # field evaluations: same accept / reject sequence
        return
    exact = _flat_rectilinear(name)
    for ref in (pd, {k: g[f"{name}/{k}"] for k in ("x", "y", "z", "t", "dt", "next_dt", "state", "ei")}):
        for k in ("state", "z") + (() if curv else ("ei",)):
            np.testing.assert_array_equal(d[k], ref[k], err_msg=f"{name}:{k}")
        if exact:
            for k in ("x", "y", "t", "dt", "next_dt"):
                np.testing.assert_array_equal(d[k], ref[k], err_msg=f"{name}:{k}")
    if exact:
        assert ps.last_report["cache_refills"] == 6 * attempts  # field evaluations: same accept / reject sequence
    else:
        # cos(lat) of libdevice vs glibc differs in the last ulp: positions to 2 ulp (curvilinear meshes: the 8 ulp of
        # test_gpu_parity.CURV_ULP); an error estimate sitting exactly on the tolerance may flip one accept/reject decision,
        # so step sizes (and, on curvilinear meshes, cells) are compared on (almost) all particles
        same_path = (d["next_dt"] == pd["next_dt"]) & (d["t"] == pd["t"])
        assert same_path.mean() > (0.95 if curv else 0.98)
        for k in ("x", "y"):
            floor = 0.01 * float(np.abs(np.asarray(c[k])).max())
            assert ulp_diff_f32(d[k][same_path], pd[k][same_path], floor=floor if curv else None).max() <= (8 if curv else 2)
        if curv:
            assert (d["ei"][same_path] == pd["ei"][same_path]).mean() > 0.99
        np.testing.assert_array_equal(d["t"], pd["t"])


def test_rk45_with_delete_handler_is_the_same_run():
    """[AdvectionRK45, DeleteParticle]: RK45 overwrites every error state it raised (_advection.py:140,154), so the handler
    never sees one -- nothing is deleted, same trajectories."""
    _, a, pd, _, _ = _engine_rk45("flat_f32c_f64d")
    _, b, _, _, _ = _engine_rk45("flat_f32c_f64d", kernels=[pb.AdvectionRK45, pb.DeleteParticle])
    assert len(a) == len(b) == len(pd["x"])
    for k in ("x", "y", "t", "dt", "next_dt", "state"):
        np.testing.assert_array_equal(a._data[k], b._data[k])


def test_rk45_to_endtime_forward_and_backward():
    """reference tests/test_particleset_execute.py:207-230 (zero velocities, run to the end of the time axis and back)."""
    lon, lat = np.linspace(0, 1, 5), np.linspace(0, 10, 6)
    time = np.arange(0, 31) * 86400.0
    U = np.zeros((31, 1, 6, 5), dtype=np.float32)
    for dt in (10 * 86400.0, 86400.0):
        fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, U=U, V=U, time=time, mesh="flat")
        fs.add_context("RK45_tol", 10)
        fs.add_context("RK45_min_dt", 1)
        fs.add_context("RK45_max_dt", 24 * 60 * 60)
        ps = pb.ParticleSet(fs, pclass=NEXT_DT, x=[0.2], y=[5.0], t=[0.0])
        ps.execute(pb.AdvectionRK45, endtime=time[-1], dt=dt)
        assert ps._data["t"][0] == time[-1]
        ps.execute(pb.AdvectionRK45, endtime=0.0, dt=-dt)
        assert ps._data["t"][0] == 0.0


def test_rk45_reports_particles_the_reference_would_spin_on():
    """Two output intervals, particles finishing the first one at different loop iterations: the reference clamps the dt
    of the early finishers to 0 (kernel.py:199-203) and then never terminates; the engine raises instead."""

    class Out:
        outputdt = 70.0

        def write(self, pset, t):
            pass

    tol, min_dt, fmax, runtime, dt = RK45_CASES["flat_f32c_f64d"]
    c = dict(__import__("oracle_run").load_case("flat_f32c_f64d"), W=None)
    fs = make_fieldset(c)
    fs.add_context("RK45_tol", tol)
    fs.add_context("RK45_min_dt", min_dt)
    fs.add_context("RK45_max_dt", fmax * abs(dt))
    ps = pb.ParticleSet(fs, pclass=NEXT_DT, x=c["x"], y=c["y"], z=np.abs(np.asarray(c["z"])), t=c["t"])
    with pytest.raises(RuntimeError, match="never terminates"):
        ps.execute(pb.AdvectionRK45, dt=dt, runtime=runtime, output_file=Out())
    assert np.any(ps._data["dt"] == 0)


@pytest.mark.parametrize("name", ["flat_f32c_f64d", "c1_peninsula"])
def test_rk45_in_a_mixed_list_matches_oracle(name):
    """[AdvectionRK45, user kernel] -- the reference's own Stommel test is written like this (tests/test_advection.py:354-387,
    `[kernel, UpdateP]`): the host drives the loop (dt clamp, position update, dt <- next_dt), every iteration's RK45 attempts run
    on the device (pb_advect_rk45 with kernels_only), the user kernel samples a scalar field there too."""
    tol, min_dt, fmax, runtime, dt = RK45_CASES[name]
    c = dict(load_case(name), W=None)
    z = np.abs(np.asarray(c["z"]))
    P = (c["U"] * 2 + 1).astype(c["U"].dtype)
    fs = make_fieldset(c)
    fs.add_field("P", P)
    for k_, v_ in (("RK45_tol", tol), ("RK45_min_dt", min_dt), ("RK45_max_dt", fmax * abs(dt))):
        fs.add_context(k_, v_)
    pclass = pb.Particle.add_variable([pb.Variable("next_dt", dtype=np.float32, initial=0), pb.Variable("p", dtype=np.float32, initial=0),
                                       pb.Variable("nsteps", dtype=np.int32, initial=0)])  # fmt: skip
    ps = pb.ParticleSet(fs, pclass=pclass, x=c["x"], y=c["y"], z=z, t=c["t"])

    def UpdateP(particles, fieldset):
        particles.p = fieldset.P[particles]
        particles.nsteps += 1

    def DeleteErr(particles, fieldset):  # particles the sampler finds outside the domain
        particles[particles.state >= 50].state = 30

    ps.execute([pb.AdvectionRK45, UpdateP, DeleteErr], dt=dt, runtime=runtime)

    ofs = oracle_fieldset(c)
    ofs.context.update(RK45_tol=tol, RK45_min_dt=min_dt, RK45_max_dt=fmax * abs(dt))  # flat meshes: no unit conversion
    pd = po.create_particle_data(c["x"], c["y"], z, c["t"])
    pd["next_dt"] = np.zeros(len(pd["x"]), dtype=np.float32)
    pd["p"] = np.zeros(len(pd["x"]), dtype=np.float32)
    pd["nsteps"] = np.zeros(len(pd["x"]), dtype=np.int32)

    def OUpdateP(p, fs_):
        p.p = po.eval_scalar(fs_, P, "linear", p.t, p.z, p.y, p.x, p)
        p.nsteps = p.nsteps + 1

    po.pset_execute(pd, ofs, [po.AdvectionRK45, OUpdateP, po.DeleteOnError], dt, runtime=runtime)
    d = ps._data
    assert len(d["x"]) == len(pd["x"]) > 0 and d["nsteps"].max() > 1
    for k in ("particle_id", "state", "t", "dt", "next_dt", "ei", "x", "y", "z", "p", "nsteps"):
        np.testing.assert_array_equal(d[k], pd[k], err_msg=k)


@pytest.mark.parametrize("name", ["cgrid_rect_sph", "curv_flat_2d", "curv_sph_2d"])
def test_rk45_on_cgrids_in_a_mixed_list_equals_the_fused_run(name):
    """CGrid_Velocity (rectilinear and curvilinear): [AdvectionRK45, user kernel] -- host loop control, every iteration's RK45
    attempts on the device with the batch-level hint rule of the curvilinear search passed per iteration -- walks the same
    accept / reject sequence as the single-launch run (which test_rk45_matches_oracle_and_reference pins to the reference)."""

    def Count(particles, fieldset):
        particles.nsteps += 1

    _, fused, pd, steps, _ = _engine_rk45(name)
    tol, min_dt, fmax, runtime, dt = RK45_CASES[name]
    c = dict(load_case(name), W=None)
    fs = make_fieldset(c)
    for k_, v_ in (("RK45_tol", tol), ("RK45_min_dt", min_dt), ("RK45_max_dt", fmax * abs(dt))):
        fs.add_context(k_, v_)
    pclass = NEXT_DT.add_variable(pb.Variable("nsteps", dtype=np.int32, initial=0))
    ps = pb.ParticleSet(fs, pclass=pclass, x=c["x"], y=c["y"], z=np.abs(np.asarray(c["z"])), t=c["t"])
    ps.execute([pb.AdvectionRK45, Count], dt=dt, runtime=runtime)
    assert ps.last_report["mode"] == "stepwise" and int(ps.nsteps.sum()) == steps
    for k in ("x", "y", "z", "t", "dt", "next_dt", "state", "ei"):
        np.testing.assert_array_equal(ps._data[k], fused._data[k], err_msg=f"{name}:{k}")
