"""GPU: time-slab streaming (``FieldSet.from_arrays(..., time_window=W)``) under every kernel list -- AdvectionRK45, fused and
mixed with user kernels; AdvectionDiffusionM1 / EM; lists with user Python kernels; lists without the DeleteParticle token --
gives the resident run bit for bit, the Wiener increments of M1 / EM included.  Sampling ``fieldset.UV`` at times outside the
resident levels brings those levels in; the C-ABI refuses such a sample instead of reading another level's ring slot."""

import numpy as np
import pytest

import parcels_b200 as pb
from cases import CASES, build
from parcels_b200._lib import EngineError

pytestmark = pytest.mark.gpu

NEXT_DT = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0))
COLUMNS = ("particle_id", "state", "t", "ei", "x", "y", "z")


def _case(name, nt, tstep, n=150, seed=None):
    spec = dict(CASES[name], nt=nt, tstep=tstep, n=n)
    if seed is not None:
        spec["seed"] = seed
    return build(spec)


def _fieldset(c, window, three_d=True):
    return pb.FieldSet.from_arrays(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"],
                                   W=c["W"] if three_d else None, mesh=c["mesh"], interp_method=c.get("interp", "linear"),
                                   padding=c.get("padding", ("low", "low", "high")), time_window=window)  # fmt: skip


def _release(c, mode, rng):
    tend = float(c["times"][-1])
    n = len(c["x"])
    if mode == "forward":
        return np.zeros(n), 1
    if mode == "backward":
        return np.full(n, tend), -1
    return np.round(rng.uniform(0, 0.4 * tend, n) / 100.0) * 100.0, 1  # delayed releases


def _assert_same(win, ref, columns=COLUMNS):
    assert len(win) == len(ref)
    for k in columns:
        np.testing.assert_array_equal(win._data[k], ref._data[k], err_msg=k)


# ---- AdvectionRK45 ----------------------------------------------------------------------------------------------------
RK45_GRIDS = {  # case of tests/cases.py, level spacing (s), nominal dt (s)
    "linear": ("flat_f32c_f64d", 50.0, 10.0),
    "freeslip": ("freeslip_3d", 200.0, 40.0),
    "cgrid_rect": ("cgrid_rect_sph", 3600.0, 600.0),
    "cgrid_curv_sph": ("curv_sph_2d", 7200.0, 900.0),
}


def _rk45_run(grid, mode, window, kernels=None, fixed_step=False):
    name, tstep, dt = RK45_GRIDS[grid]
    c = _case(name, nt=6, tstep=tstep)
    fs = _fieldset(c, window, three_d=False)
    if fixed_step:  # every step a quarter level interval: no step straddles a level, so two resident levels suffice
        fs.add_context("RK45_tol", 1e30)
        fs.add_context("RK45_min_dt", tstep / 4)
        fs.add_context("RK45_max_dt", tstep / 4)
        dt = tstep / 4
    else:
        fs.add_context("RK45_tol", 5.0)
        fs.add_context("RK45_min_dt", dt / 8)
        fs.add_context("RK45_max_dt", 2 * dt)
    t0, sign = _release(c, mode, np.random.default_rng(5))
    ps = pb.ParticleSet(fs, pclass=NEXT_DT, x=c["x"], y=c["y"], z=np.abs(c["z"]), t=t0)
    tend = float(c["times"][-1])
    ps.execute(kernels or [pb.AdvectionRK45], dt=sign * dt, endtime=0.1 * tend if sign < 0 else 0.9 * tend)
    return ps


@pytest.mark.parametrize("mode", ["forward", "backward", "delayed"])
@pytest.mark.parametrize("grid", list(RK45_GRIDS))
def test_rk45_windowed_equals_resident(grid, mode):
    ref = _rk45_run(grid, mode, None)
    win = _rk45_run(grid, mode, 3)
    assert win.last_report["particle_steps"] == ref.last_report["particle_steps"] > 0
    assert win.fieldset._win[0]["first"] == (0 if mode == "backward" else 3)  # the window has slid over the run
    _assert_same(win, ref, COLUMNS + ("dt", "next_dt"))


def test_rk45_two_level_window_with_steps_on_the_levels():
    ref = _rk45_run("linear", "forward", None, fixed_step=True)
    win = _rk45_run("linear", "forward", 2, fixed_step=True)
    _assert_same(win, ref, COLUMNS + ("dt", "next_dt"))


def _age(particles, fieldset):
    particles.age += particles.dt


AGE = NEXT_DT.add_variable(pb.Variable("age", dtype=np.float64, initial=0))


def test_rk45_mixed_with_a_user_kernel_windowed_equals_resident():
    """A mixed list runs step by step: every iteration needs the levels of all particles' steps, and adaptive steps drift
    apart in time -- the window is sized for that spread."""
    name, tstep, dt = RK45_GRIDS["cgrid_rect"]
    out = []
    for window in (None, 4):
        c = _case(name, nt=8, tstep=tstep, n=60)
        fs = _fieldset(c, window, three_d=False)
        fs.add_context("RK45_tol", 5.0)
        fs.add_context("RK45_min_dt", dt / 8)
        fs.add_context("RK45_max_dt", 2 * dt)
        ps = pb.ParticleSet(fs, pclass=AGE, x=c["x"], y=c["y"], z=np.abs(c["z"]), t=np.zeros(len(c["x"])))
        ps.execute([pb.AdvectionRK45, _age, pb.DeleteParticle], dt=dt, endtime=0.5 * float(c["times"][-1]))
        out.append(ps)
    _assert_same(out[1], out[0], COLUMNS + ("dt", "next_dt", "age"))


def test_rk45_step_wider_than_any_window_is_an_error():
    name, tstep, _ = RK45_GRIDS["linear"]
    c = _case(name, nt=6, tstep=tstep, n=20)
    fs = _fieldset(c, 2, three_d=False)
    fs.add_context("RK45_tol", 1e30)
    fs.add_context("RK45_min_dt", 1.0)
    fs.add_context("RK45_max_dt", 2 * tstep)
    ps = pb.ParticleSet(fs, pclass=NEXT_DT, x=c["x"], y=c["y"], z=np.abs(c["z"]), t=np.zeros(20))
    with pytest.raises(RuntimeError, match="widen time_window"):
        ps.execute([pb.AdvectionRK45], dt=1.5 * tstep, runtime=4 * tstep)


# ---- AdvectionDiffusionM1 / EM ------------------------------------------------------------------------------------------
def _advdiff_run(kernel, mesh, kh_time, window, extra=(), nt=6, n=120, delete=True, near_edge=False, raises=None, spread=1.5):
    rng = np.random.default_rng(11)
    nx, ny, tstep = 24, 20, 3600.0
    if mesh == "flat":
        lon, lat = np.linspace(-1e5, 1e5, nx), np.linspace(-8e4, 8e4, ny)
    else:
        lon, lat = np.linspace(-2.0, 2.0, nx), np.linspace(-1.5, 1.5, ny)
    shape = (nt, 1, ny, nx)
    U = (0.5 * rng.uniform(-1, 1, shape)).astype(np.float32)
    V = (0.5 * rng.uniform(-1, 1, shape)).astype(np.float32)
    kt = nt if kh_time else 1
    X = lon[None, None, None, :] / lon.max()
    Kz = (40.0 + 20.0 * X + 5.0 * rng.uniform(0, 1, (kt, 1, ny, nx))).astype(np.float64)
    Km = (30.0 + 10.0 * rng.uniform(0, 1, (kt, 1, ny, nx))).astype(np.float64)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, time=np.arange(nt) * tstep, U=U, V=V, mesh=mesh, time_window=window)
    fs.add_field("Kh_zonal", Kz)
    fs.add_field("Kh_meridional", Km)
    fs.add_context("dres", float(lon[1] - lon[0]) / 10)
    x = rng.uniform(0.97 * lon.max(), 0.995 * lon.max(), n) if near_edge else rng.uniform(0.6 * lon.min(), 0.6 * lon.max(), n)
    y = rng.uniform(0.6 * lat.min(), 0.6 * lat.max(), n)
    t0 = np.round(rng.uniform(0, spread * tstep, n) / 600.0) * 600.0
    ps = pb.ParticleSet(fs, pclass=AGE, x=x, y=y, t=t0, seed=77)
    kl = [getattr(pb, kernel), *extra] + ([pb.DeleteParticle] if delete else [])
    if raises is None:
        ps.execute(kl, dt=600.0, endtime=(nt - 1.5) * tstep)
    else:
        with pytest.raises(raises):
            ps.execute(kl, dt=600.0, endtime=(nt - 1.5) * tstep)
    return ps


@pytest.mark.parametrize("kh_time", [False, True])
@pytest.mark.parametrize("mesh", ["flat", "spherical"])
@pytest.mark.parametrize("kernel", ["AdvectionDiffusionM1", "AdvectionDiffusionEM"])
def test_advdiff_windowed_equals_resident(kernel, mesh, kh_time):
    ref = _advdiff_run(kernel, mesh, kh_time, None)
    win = _advdiff_run(kernel, mesh, kh_time, 2)
    assert win.last_report["particle_steps"] == ref.last_report["particle_steps"] > 0
    assert win.fieldset._win[0]["first"] == 4  # the window has slid to the last two of the six levels
    assert np.any(win.x != win.x[::-1]) and np.all(win.t == ref.t)
    _assert_same(win, ref)


def test_advdiff_mixed_with_a_user_kernel_windowed_equals_resident():
    """Step by step, every iteration needs the levels of all particles: releases spread over less than one level interval."""
    ref = _advdiff_run("AdvectionDiffusionM1", "flat", True, None, extra=(_age,), spread=0.5)
    win = _advdiff_run("AdvectionDiffusionM1", "flat", True, 3, extra=(_age,), spread=0.5)
    _assert_same(win, ref, COLUMNS + ("age",))


def test_advdiff_without_delete_handler_raises_like_the_resident_run():
    """Particles leave the domain: without DeleteParticle the run raises after the iteration of the first exit; the windowed
    call replays up to it with the same Wiener increments."""
    ref = _advdiff_run("AdvectionDiffusionEM", "flat", False, None, delete=False, near_edge=True, raises=pb.FieldOutOfBoundError)
    win = _advdiff_run("AdvectionDiffusionEM", "flat", False, 2, delete=False, near_edge=True, raises=pb.FieldOutOfBoundError)
    assert np.any(win.state == pb.StatusCode.ErrorOutOfBounds) and np.any(win.t > 0)
    _assert_same(win, ref)


# ---- user kernels -------------------------------------------------------------------------------------------------------
SAMPLER = pb.Particle.add_variable([pb.Variable("u0", dtype=np.float64), pb.Variable("v1", dtype=np.float64),
                                    pb.Variable("p", dtype=np.float64)])  # fmt: skip


def _sample(particles, fieldset):
    u0, _ = fieldset.UV.eval(particles.t, particles.z, particles.y, particles.x, particles)
    _, v1 = fieldset.UV[particles.t + particles.dt, particles.z, particles.y, particles.x]
    particles.u0 = u0
    particles.v1 = v1
    particles.p = fieldset.P[particles]


def _user_run(window, spread=0.15, n=120):
    c = _case("c2_small", nt=7, tstep=3600.0, n=n, seed=9)
    fs = _fieldset(c, window)
    fs.add_field("P", np.asarray(c["U"], dtype=np.float32) + np.float32(1.0))
    rng = np.random.default_rng(3)
    t0 = np.round(rng.uniform(0, spread * 6 * 3600.0, n) / 600.0) * 600.0
    ps = pb.ParticleSet(fs, pclass=SAMPLER, x=c["x"], y=c["y"], z=c["z"], t=t0)
    ps.execute([pb.AdvectionRK4_3D, _sample, pb.DeleteParticle], dt=600.0, endtime=5.5 * 3600.0)
    return ps


def test_user_kernel_list_windowed_equals_resident():
    ref = _user_run(None)
    win = _user_run(3)
    _assert_same(win, ref, COLUMNS + ("u0", "v1", "p"))
    assert np.any(win.u0 != 0) and np.any(win.p != 0)


def test_user_kernel_list_with_releases_wider_than_the_window_is_an_error():
    with pytest.raises(RuntimeError, match="widen time_window"):
        _user_run(2, spread=0.9, n=40)


# ---- lists without the DeleteParticle token ---------------------------------------------------------------------------
RAISING = {  # case, levels, seconds to run
    "out_of_bounds": ("raise_oob", 5, 1500.0),
    "through_surface": ("through_surface", 5, 4000.0),
    "outside_time_interval": ("raise_time", 5, 2500.0),
}


def _raising_run(kind, window):
    name, nt, runtime = RAISING[kind]
    spec = CASES[name]
    c = _case(name, nt=nt, tstep=spec["tstep"], n=spec["n"])
    fs = _fieldset(c, window)
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    with pytest.raises(RuntimeError) as e:
        ps.execute([pb.AdvectionRK4_3D], dt=spec["dt"], runtime=runtime)
    return ps, type(e.value)


@pytest.mark.parametrize("kind", list(RAISING))
def test_list_without_delete_handler_raises_like_the_resident_run(kind):
    ref, ref_err = _raising_run(kind, None)
    win, win_err = _raising_run(kind, 2)
    assert win_err is ref_err
    _assert_same(win, ref)


# ---- sampling -----------------------------------------------------------------------------------------------------------
def test_vector_field_eval_brings_in_the_levels_of_its_sample_times():
    c = _case("c2_small", nt=7, tstep=3600.0, n=50, seed=4)
    ref_fs, win_fs = _fieldset(c, None), _fieldset(c, 2)
    for fs in (ref_fs, win_fs):  # first use: the window holds the first levels
        pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=np.zeros(50)).execute([pb.AdvectionRK4_3D, pb.DeleteParticle], dt=600.0,
                                                                                   runtime=1800.0)  # fmt: skip
    for t in (5.25 * 3600.0, 0.5 * 3600.0, 6 * 3600.0, 3 * 3600.0):
        ts = np.full(50, t)
        for a, b in zip(win_fs.UVW.eval(ts, c["z"], c["y"], c["x"]), ref_fs.UVW.eval(ts, c["z"], c["y"], c["x"]), strict=True):
            np.testing.assert_array_equal(a, b)
    with pytest.raises(RuntimeError, match="widen time_window"):
        win_fs.UV.eval(np.array([0.0, 4 * 3600.0]), c["z"][:2], c["y"][:2], c["x"][:2])


def test_sample_velocity_at_a_time_that_is_not_resident_is_refused():
    c = _case("c2_small", nt=7, tstep=3600.0, n=10, seed=4)
    fs = _fieldset(c, 2)
    fs.UV.eval(np.zeros(10), c["z"], c["y"], c["x"])  # window: levels 0 and 1
    eng = fs.engine(0)
    with pytest.raises(EngineError, match="resident time levels"):
        eng.sample_velocity(np.full(10, 4 * 3600.0), c["z"], c["y"], c["x"], three_d=False)
    u, *_ = eng.sample_velocity(np.full(10, 1800.0), c["z"], c["y"], c["x"], three_d=False)
    assert np.all(np.isfinite(u))
    eng.sample_velocity(np.full(10, 99 * 3600.0), c["z"], c["y"], c["x"], three_d=False)  # outside the axis: OutsideTimeInterval
