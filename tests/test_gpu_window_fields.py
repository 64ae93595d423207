"""GPU: time-slab streaming of scalar fields (``FieldSet.add_field(..., time_window=W)``) and of fields on further grids gives the
run with every field resident bit for bit: a sampled tracer on the velocity grid (rectilinear and curvilinear), a windowed
Kh of AdvectionDiffusionM1 / EM, and a scalar and a vector field on a second grid with its own time axis.  Only the levels that
enter a window are ever read from the caller's array-like; the C-ABI refuses a sample of a level that is not resident."""

import numpy as np
import pytest

import parcels_b200 as pb
from cases import CASES, build
from parcels_b200._lib import EngineError
from parcels_b200.fieldset import XGrid

pytestmark = pytest.mark.gpu

COLUMNS = ("particle_id", "state", "t", "ei", "x", "y", "z")
SAMPLER = pb.Particle.add_variable(pb.Variable("p", dtype=np.float64, initial=0))


class Levels:
    """An array-like that hands out one time level per ``[level]`` and records which; materialising it whole fails."""

    def __init__(self, a):
        self._a, self.shape, self.dtype, self.reads = a, a.shape, a.dtype, []

    def __getitem__(self, level):
        assert isinstance(level, (int, np.integer)), level
        self.reads.append(int(level))
        return self._a[level]

    def __array__(self, *args, **kwargs):
        raise AssertionError("the whole time-windowed field was materialised")


def _case(name, nt, tstep, n, seed=None):
    spec = dict(CASES[name], nt=nt, tstep=tstep, n=n)
    if seed is not None:
        spec["seed"] = seed
    return build(spec)


def _fieldset(c, window, three_d=True):
    return pb.FieldSet.from_arrays(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"],
                                   W=c["W"] if three_d else None, mesh=c["mesh"], interp_method=c.get("interp", "linear"),
                                   padding=c.get("padding", ("low", "low", "high")), time_window=window)  # fmt: skip


def _tracer(c, land=False):
    """A float32 tracer that changes from level to level (zero on a block of land nodes for the land tracer)."""
    U = np.asarray(c["U"], dtype=np.float32)
    P = (10.0 * U + np.arange(U.shape[0], dtype=np.float32)[:, None, None, None]).astype(np.float32)
    if land:
        P[..., 3:9, 5:14] = 0
    return P


def _release(c, mode, n):
    tend = float(c["times"][-1])
    if mode == "forward":
        return np.zeros(n), 1
    if mode == "backward":
        return np.full(n, tend), -1
    return np.round(np.random.default_rng(3).uniform(0, 0.15 * tend, n) / 600.0) * 600.0, 1  # delayed releases


def _assert_same(win, ref, columns=COLUMNS + ("p",)):
    assert len(win) == len(ref)
    for k in columns:
        np.testing.assert_array_equal(win._data[k], ref._data[k], err_msg=k)


def _sample_p(particles, fieldset):
    particles.p = fieldset.P[particles]


# ---- a tracer on the velocity grid -------------------------------------------------------------------------------------------
GRIDS = {  # case, levels, level spacing (s), dt (s), advection kernel
    "rect": ("c2_small", 7, 3600.0, 600.0, pb.AdvectionRK4_3D),
    "curv": ("curv_sph_2d", 6, 7200.0, 900.0, pb.AdvectionRK4),
}


def _tracer_run(grid, method, mode, window, n=120):
    name, nt, tstep, dt, adv = GRIDS[grid]
    c = _case(name, nt, tstep, n, seed=9)
    fs = _fieldset(c, window, three_d=adv is pb.AdvectionRK4_3D)
    P = Levels(_tracer(c, land=method == "linear_invdist_land"))
    fs.add_field("P", P if window else P._a, interp_method=method, time_window=window)
    t0, sign = _release(c, mode, n)
    ps = pb.ParticleSet(fs, pclass=SAMPLER, x=c["x"], y=c["y"], z=c["z"], t=t0)
    tend = float(c["times"][-1])
    ps.execute([adv, _sample_p, pb.DeleteParticle], dt=sign * dt, endtime=0.1 * tend if sign < 0 else 0.9 * tend)
    return ps, P.reads


@pytest.mark.parametrize("mode", ["forward", "backward", "delayed"])
@pytest.mark.parametrize("method", ["linear", "nearest", "cgrid_tracer", "linear_invdist_land"])
def test_tracer_windowed_equals_resident(method, mode):
    ref, _ = _tracer_run("rect", method, mode, None)
    win, reads = _tracer_run("rect", method, mode, 3)
    _assert_same(win, ref)
    assert np.any(win.p != 0)
    assert set(reads) >= {1, 5}  # the window has slid over the run (levels 0 .. 6, three of them resident at a time)
    if mode != "backward":  # forward, each level enters the window once (backward, the first use loads levels 0 .. 2 first)
        assert sorted(reads) == sorted(set(reads))


@pytest.mark.parametrize("mode", ["forward", "backward"])
@pytest.mark.parametrize("method", ["linear", "cgrid_tracer"])
def test_tracer_on_a_curvilinear_cgrid_windowed_equals_resident(method, mode):
    ref, _ = _tracer_run("curv", method, mode, None)
    win, reads = _tracer_run("curv", method, mode, 3)
    _assert_same(win, ref)
    assert np.any(win.p != 0) and max(reads) >= 4


def test_only_the_levels_entering_the_window_are_read():
    """Forward from t = 0 with a window of 3: each level is read once, when it enters the window, and never the whole field."""
    c = _case("c2_small", 7, 3600.0, 60, seed=9)
    fs = _fieldset(c, 3)
    P = Levels(_tracer(c))
    fs.add_field("P", P, time_window=3)
    assert P.reads == []
    ps = pb.ParticleSet(fs, pclass=SAMPLER, x=c["x"], y=c["y"], z=c["z"], t=np.zeros(60))
    ps.execute([pb.AdvectionRK4_3D, _sample_p, pb.DeleteParticle], dt=600.0, endtime=2.5 * 3600.0)
    assert sorted(P.reads) == sorted(set(P.reads)) and set(P.reads) <= {0, 1, 2, 3, 4}
    assert set(P.reads) == set(fs._win[0]["resident"]) | set(range(3))
    assert np.all(ps.t == 2.5 * 3600.0)


# ---- a windowed Kh under AdvectionDiffusionM1 / EM ---------------------------------------------------------------------------
def _advdiff_run(kernel, mesh, window, delete=True, near_edge=False, raises=None, nt=6, n=120):
    rng = np.random.default_rng(11)
    nx, ny, tstep = 24, 20, 3600.0
    if mesh == "flat":
        lon, lat = np.linspace(-1e5, 1e5, nx), np.linspace(-8e4, 8e4, ny)
    else:
        lon, lat = np.linspace(-2.0, 2.0, nx), np.linspace(-1.5, 1.5, ny)
    shape = (nt, 1, ny, nx)
    U = (0.5 * rng.uniform(-1, 1, shape)).astype(np.float32)
    V = (0.5 * rng.uniform(-1, 1, shape)).astype(np.float32)
    X = lon[None, None, None, :] / lon.max()
    Kz = (40.0 + 20.0 * X + 5.0 * rng.uniform(0, 1, shape)).astype(np.float64)
    Km = (30.0 + 10.0 * rng.uniform(0, 1, shape)).astype(np.float64)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, time=np.arange(nt) * tstep, U=U, V=V, mesh=mesh, time_window=window)
    fs.add_field("Kh_zonal", Levels(Kz) if window else Kz, time_window=window)
    fs.add_field("Kh_meridional", Levels(Km) if window else Km, time_window=window)
    fs.add_context("dres", float(lon[1] - lon[0]) / 10)
    x = rng.uniform(0.97 * lon.max(), 0.995 * lon.max(), n) if near_edge else rng.uniform(0.6 * lon.min(), 0.6 * lon.max(), n)
    y = rng.uniform(0.6 * lat.min(), 0.6 * lat.max(), n)
    t0 = np.round(rng.uniform(0, 1.5 * tstep, n) / 600.0) * 600.0
    ps = pb.ParticleSet(fs, x=x, y=y, t=t0, seed=77)
    kl = [getattr(pb, kernel)] + ([pb.DeleteParticle] if delete else [])
    if raises is None:
        ps.execute(kl, dt=600.0, endtime=(nt - 1.5) * tstep)
    else:
        with pytest.raises(raises):
            ps.execute(kl, dt=600.0, endtime=(nt - 1.5) * tstep)
    return ps


@pytest.mark.parametrize("mesh", ["flat", "spherical"])
@pytest.mark.parametrize("kernel", ["AdvectionDiffusionM1", "AdvectionDiffusionEM"])
def test_advdiff_with_a_windowed_kh_equals_resident(kernel, mesh):
    ref = _advdiff_run(kernel, mesh, None)
    win = _advdiff_run(kernel, mesh, 2)
    assert win.last_report["particle_steps"] == ref.last_report["particle_steps"] > 0
    assert win.fieldset._win[0]["first"] == 4  # the window has slid to the last two of the six levels
    assert max(win.fieldset.Kh_zonal.data.reads) == 5
    _assert_same(win, ref, COLUMNS)


@pytest.mark.parametrize("kernel", ["AdvectionDiffusionM1", "AdvectionDiffusionEM"])
def test_advdiff_with_a_windowed_kh_without_delete_handler_raises_like_the_resident_run(kernel):
    ref = _advdiff_run(kernel, "flat", None, delete=False, near_edge=True, raises=pb.FieldOutOfBoundError)
    win = _advdiff_run(kernel, "flat", 2, delete=False, near_edge=True, raises=pb.FieldOutOfBoundError)
    assert np.any(win.state == pb.StatusCode.ErrorOutOfBounds) and np.any(win.t > 0)
    _assert_same(win, ref, COLUMNS)


# ---- fields on a second grid with its own time axis ------------------------------------------------------------------------
WIND = pb.Particle.add_variable([pb.Variable("w", dtype=np.float64), pb.Variable("u10", dtype=np.float64),
                                 pb.Variable("v10", dtype=np.float64)])  # fmt: skip


def _sample_wind(particles, fieldset):
    particles.w = fieldset.wind[particles]
    u, v = fieldset.wind10[particles]
    particles.u10 = u
    particles.v10 = v


def _second_grid_run(window, n=100):
    c = _case("c2_small", 7, 3600.0, n, seed=4)
    fs = _fieldset(c, None)
    rng = np.random.default_rng(8)
    g2 = XGrid(np.linspace(-12.0, 12.0, 13), np.linspace(28.0, 52.0, 11), None, mesh="spherical")
    t2 = np.arange(14) * 1800.0  # every half hour: a finer time axis than U's
    wind = rng.uniform(-5, 5, (14, 1, 11, 13))
    U10 = rng.uniform(-8, 8, (14, 1, 11, 13)).astype(np.float32)
    V10 = rng.uniform(-8, 8, (14, 1, 11, 13)).astype(np.float32)
    wrap = Levels if window else (lambda a: a)
    fs.add_vector_field("wind10", wrap(U10), wrap(V10), grid=g2, time=t2, time_window=window)
    fs.add_field("wind", wrap(wind), grid=g2, time=t2, time_window=window)
    ps = pb.ParticleSet(fs, pclass=WIND, x=c["x"], y=c["y"], z=c["z"], t=np.zeros(n))
    ps.execute([pb.AdvectionRK4_3D, _sample_wind, pb.DeleteParticle], dt=600.0, endtime=5.5 * 3600.0)
    return ps


def test_scalar_and_vector_field_on_a_second_grid_windowed_equals_resident():
    ref = _second_grid_run(None)
    win = _second_grid_run(3)
    _assert_same(win, ref, COLUMNS + ("w", "u10", "v10"))
    assert np.any(win.w != 0) and np.any(win.u10 != 0)
    host = win.fieldset._extra_grids[0]
    assert host.time_window == 3 and host._win[0]["first"] >= 9  # slid along its own axis, to 5.5 h = level 11
    assert win.fieldset.time_window is None and win.fieldset.wind.data.reads.count(11) == 1


# ---- Field.eval and the C-ABI ----------------------------------------------------------------------------------------------
def _eval_pair(window=2, n=40):
    c = _case("c2_small", 7, 3600.0, n, seed=4)
    out = []
    for w in (None, window):
        fs = _fieldset(c, w)
        fs.add_field("P", _tracer(c), time_window=w)
        out.append(fs)
    return c, out


def test_field_eval_brings_in_the_levels_of_its_sample_times():
    c, (ref_fs, win_fs) = _eval_pair()
    for t in (5.25 * 3600.0, 0.5 * 3600.0, 6 * 3600.0, 3 * 3600.0):
        ts = np.full(40, t)
        np.testing.assert_array_equal(win_fs.P.eval(ts, c["z"], c["y"], c["x"]), ref_fs.P.eval(ts, c["z"], c["y"], c["x"]))
        assert win_fs._time_s[win_fs._win[0]["first"]] <= t <= win_fs._time_s[win_fs._win[0]["first"] + 1]
    states = []
    for fs in (ref_fs, win_fs):  # outside the time axis: OutsideTimeInterval, nothing loaded
        ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=np.zeros(40))
        fs.P.eval(np.full(40, 99 * 3600.0), ps._data["z"], ps._data["y"], ps._data["x"], ps)
        states.append(np.array(ps.state))
    assert np.all(states[1] == pb.StatusCode.ErrorOutsideTimeInterval)
    np.testing.assert_array_equal(states[1], states[0])
    with pytest.raises(RuntimeError, match="widen time_window"):
        win_fs.P.eval(np.array([0.0, 4 * 3600.0]), c["z"][:2], c["y"][:2], c["x"][:2])


def test_sample_scalar_at_a_time_that_is_not_resident_is_refused():
    c, (_, fs) = _eval_pair()
    fs.P.eval(np.zeros(40), c["z"], c["y"], c["x"])  # window: levels 0 and 1
    eng = fs.engine(0)
    with pytest.raises(EngineError, match="resident time levels"):
        eng.sample_scalar(fs.P._slot, "linear", np.full(40, 4 * 3600.0), c["z"], c["y"], c["x"])
    val, _, _ = eng.sample_scalar(fs.P._slot, "linear", np.full(40, 1800.0), c["z"], c["y"], c["x"])
    assert np.all(np.isfinite(val))


# ---- validation --------------------------------------------------------------------------------------------------------------
def test_time_window_validation():
    c = _case("c2_small", 7, 3600.0, 10, seed=4)
    P = _tracer(c)
    with pytest.raises(ValueError, match="window of 3 levels"):
        _fieldset(c, 3).add_field("P", P, time_window=2)
    with pytest.raises(ValueError, match="built without one"):
        _fieldset(c, None).add_field("P", P, time_window=3)
    with pytest.raises(ValueError, match="no time dimension to stream"):
        _fieldset(c, 3).add_field("P", P[:1], time_window=3)
    g2 = XGrid(np.linspace(-12.0, 12.0, 13), np.linspace(28.0, 52.0, 11), None, mesh="spherical")
    fs = _fieldset(c, None)
    fs.add_field("A", np.zeros((7, 1, 11, 13)), grid=g2, time_window=3)
    with pytest.raises(ValueError, match="use 3"):
        fs.add_field("B", np.zeros((7, 1, 11, 13)), grid=g2, time_window=4)
