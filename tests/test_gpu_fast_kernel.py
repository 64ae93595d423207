"""The specialised RK4 kernel (csrc/afast.cu: float64 grid, float32 node-interleaved data, cached T-lerp; two schedules) against the generic
A-grid kernel (csrc/agrid.cuh) -- the SAME arithmetic in another schedule, so every array must agree BIT FOR BIT -- and against
the oracle.  `PB_DISABLE_FAST_KERNEL=1` (read by the library at every launch) selects the generic kernel."""

import os

import numpy as np
import pytest

import parcels_b200 as pb
from device_trig import DeviceTrig
from engine_run import ulp_diff_f32
from oracle import trig
from oracle_run import run_oracle

pytestmark = pytest.mark.gpu

KEYS = ("particle_id", "state", "t", "ei", "x", "y", "z", "dx", "dy", "dz", "dt")


def _field(rng, nx, ny, nz, nt, mesh, tstep, umax):
    if mesh == "spherical":
        lon, lat = np.linspace(-20.0, 25.0, nx), np.linspace(30.0, 62.0, ny)
    else:
        lon, lat = np.linspace(0.0, 4.0e4, nx), np.linspace(-1.0e4, 2.5e4, ny)
    lon = lon + rng.uniform(-0.2, 0.2, nx) * (lon[1] - lon[0])  # irregular spacing
    lat = lat + rng.uniform(-0.2, 0.2, ny) * (lat[1] - lat[0])
    depth = None if nz == 0 else (np.array([0.0]) if nz == 1 else 800.0 * np.linspace(0, 1, nz) ** 1.5)
    times = np.arange(nt) * tstep
    shape = (nt, max(nz, 1), ny, nx)
    scale = umax * (1.0 if mesh == "flat" else 1.0)
    U = (scale * rng.uniform(-1, 1, shape)).astype(np.float32)
    V = (scale * rng.uniform(-1, 1, shape)).astype(np.float32)
    W = (0.05 * rng.uniform(-1, 1, shape)).astype(np.float32)
    return dict(lon=lon, lat=lat, depth=depth, times=times, U=U, V=V, W=W, mesh=mesh)


def _case(seed):
    """One random configuration that qualifies for the fast kernel (float64 axes, float32 data, >= 2 time levels, RK4)."""
    rng = np.random.default_rng(seed)
    three_d = bool(rng.integers(0, 2))
    nz = int(rng.integers(2, 9)) if three_d else int(rng.choice([0, 1, 5]))
    mesh = str(rng.choice(["spherical", "flat"]))
    nt = int(rng.integers(2, 5))
    backward = bool(rng.integers(0, 2))
    dt = float(rng.choice([300.0, 450.0, 600.0])) * (-1 if backward else 1)
    tstep = float(rng.choice([1800.0, 3600.0]))
    nx, ny = int(rng.integers(6, 30)), int(rng.integers(5, 26))
    umax = 8.0 if mesh == "spherical" else 6.0  # crosses cells often (and leaves the domain sometimes)
    f = _field(rng, nx, ny, nz, nt, mesh, tstep, umax)
    n = int(rng.integers(50, 260))
    lon, lat = f["lon"], f["lat"]
    m = 0.04  # a few percent released outside the domain
    x = rng.uniform(lon[0] - m * (lon[-1] - lon[0]), lon[-1] + m * (lon[-1] - lon[0]), n)
    y = rng.uniform(lat[0] - m * (lat[-1] - lat[0]), lat[-1] + m * (lat[-1] - lat[0]), n)
    if f["depth"] is not None and len(f["depth"]) > 1:
        z = rng.uniform(-20.0, f["depth"][-1] * 1.02, n)
        z[rng.random(n) < 0.1] = f["depth"][0]           # exactly on the first level: zeta == 0, no Z-lerp
        z[rng.random(n) < 0.05] = f["depth"][-1]         # exactly on the last level
        z[rng.random(n) < 0.05] = f["depth"][int(len(f["depth"]) // 2)]  # exactly on an inner level
    else:
        z = np.zeros(n)
    x[rng.random(n) < 0.05] = lon[0]    # on the first / last / an inner node of an axis
    x[rng.random(n) < 0.05] = lon[-1]
    y[rng.random(n) < 0.05] = lat[0]
    y[rng.random(n) < 0.05] = lat[int(ny // 2)]
    total = f["times"][-1]
    span = abs(dt) * int(rng.integers(3, 10))
    t0 = total if backward else 0.0
    t = np.full(n, t0)
    late = rng.random(n) < 0.3  # delayed releases
    t[late] = t0 + (-1 if backward else 1) * abs(dt) * rng.integers(1, 4, late.sum())
    if rng.random() < 0.3:
        x[int(rng.integers(0, n))] = np.nan
    kernels = ["AdvectionRK4_3D" if three_d else "AdvectionRK4"]
    diffusion = bool(rng.random() < 0.25)
    delete = bool(rng.random() < 0.7)
    segs = [span] if rng.random() < 0.5 else [span / 2 if (span / 2) % abs(dt) == 0 else abs(dt) * 2, abs(dt) * 3]
    return dict(field=f, x=x, y=y, z=z, t=t, dt=dt, kernels=kernels, diffusion=diffusion, delete=delete, segments=segs,
                three_d=three_d, seed=seed)


def _run(c, fast: int):
    """fast: 0 = the generic kernel, 1 / 2 = afast.cu's schedule 1 (four-trip stage loop; the default of lists with diffusion) /
    2 (two-stage loop body; the default of advection-only lists)"""
    os.environ["PB_DISABLE_FAST_KERNEL"] = "0" if fast else "1"
    os.environ["PB_FAST_KERNEL"] = str(fast or 1)
    try:
        f = c["field"]
        fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"],
                                     W=f["W"] if c["three_d"] else None, mesh=f["mesh"])
        if c["diffusion"]:
            fs.add_constant_field("Kh_zonal", 40.0, mesh=f["mesh"])
            fs.add_constant_field("Kh_meridional", 25.0, mesh=f["mesh"])
        ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"], seed=77)
        kern = [getattr(pb, k) for k in c["kernels"]]
        if c["diffusion"]:
            kern.append(pb.DiffusionUniformKh)
        if c["delete"]:
            kern.append(pb.DeleteParticle)
        err = ""
        reps = []
        try:
            for seg in c["segments"]:
                ps.execute(kern, dt=c["dt"], runtime=seg)
                reps.append(dict(ps.last_report))
        except RuntimeError as e:
            if type(e).__module__.startswith("parcels_b200._lib"):
                raise
            err = type(e).__name__
        return {k: np.array(ps._data[k]) for k in KEYS}, err, reps
    finally:
        os.environ.pop("PB_DISABLE_FAST_KERNEL", None)
        os.environ.pop("PB_FAST_KERNEL", None)


@pytest.mark.parametrize("version", [1, 2])
@pytest.mark.parametrize("seed", range(60))
def test_fast_kernel_equals_generic_kernel_bit_for_bit(seed, version):
    c = _case(1000 + seed)
    a, ea, ra = _run(c, fast=version)
    b, eb, rb = _run(c, fast=0)
    assert ea == eb
    for k in KEYS:
        np.testing.assert_array_equal(a[k].view(np.uint8), b[k].view(np.uint8), err_msg=f"{k} (seed {seed})")
    for x_, y_ in zip(ra, rb, strict=True):
        for k in ("particle_steps", "n_error", "n_deleted", "first_error_iter", "n_out_of_time", "max_state"):
            assert x_[k] == y_[k], (k, x_[k], y_[k])
        assert x_["kernel_variant"] == version and y_["kernel_variant"] == 0


def test_fast_kernel_is_the_one_that_runs_and_refills_less_often_than_it_samples():
    """The qualifying configuration really takes the specialised kernel: its report counts corner-block refills, and on a
    coarse grid with slow flow there are far fewer refills than samples (the cache works)."""
    rng = np.random.default_rng(5)
    f = _field(rng, 12, 10, 4, 3, "flat", 3600.0, 0.5)
    f["W"] *= np.float32(0.1)
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"], mesh="flat")
    n = 300
    ps = pb.ParticleSet(fs, x=rng.uniform(5e3, 3.5e4, n), y=rng.uniform(-5e3, 2e4, n), z=rng.uniform(10, 700, n), t=np.zeros(n))
    ps.execute([pb.AdvectionRK4_3D, pb.DeleteParticle], dt=60.0, runtime=3600.0)
    rep = ps.last_report
    assert rep["kernel_variant"] == 2
    assert rep["particle_steps"] == n * 60
    assert 0 < rep["cache_refills"] < rep["particle_steps"] // 4


@pytest.mark.parametrize(
    "mesh, schedule",
    [pytest.param("spherical", None, id="spherical"), pytest.param("flat", None, id="flat")]
    + [pytest.param("spherical", v, id=f"spherical-exact-schedule{v}") for v in (1, 2)],
)
def test_fast_kernel_against_the_oracle(mesh, schedule):
    """Directly against the CPU oracle (bit-exact ids / states / times / cells; positions bit-exact on the flat mesh, <= 2 float32
    ulp on the spherical one, where CUDA's cos differs from libm's in the last place).  With a `schedule`, the spherical case
    runs in that schedule of afast.cu against the oracle in engine arithmetic (the device's cosf / cos_np in the unit conversion,
    tests/device_trig.py): positions bit-exact too, so the code afast.cu shares with the generic kernel is pinned by itself."""
    rng = np.random.default_rng(11)
    f = _field(rng, 24, 19, 7, 3, mesh, 3600.0, 3.0)
    n = 400
    lon, lat = f["lon"], f["lat"]
    c = dict(lon=lon, lat=lat, depth=f["depth"], times=f["times"], U=f["U"], V=f["V"], W=f["W"], mesh=mesh, constants=None,
             x=rng.uniform(lon[0], lon[-1], n), y=rng.uniform(lat[0], lat[-1], n), z=rng.uniform(0, 790.0, n), t=np.zeros(n),
             kernels=["AdvectionRK4_3D"], delete_on_error=True, dt=600.0, segments=[dict(runtime=7200.0)])  # fmt: skip
    from engine_run import run_engine

    if schedule is None:
        ps, err = run_engine(c)
        pd, oerr = run_oracle(c)
    else:
        os.environ["PB_DISABLE_FAST_KERNEL"] = "0"
        os.environ["PB_FAST_KERNEL"] = str(schedule)
        try:
            ps, err = run_engine(c)
        finally:
            os.environ.pop("PB_DISABLE_FAST_KERNEL", None)
            os.environ.pop("PB_FAST_KERNEL", None)
        assert ps.last_report["kernel_variant"] == schedule
        with trig.use(DeviceTrig()):
            pd, oerr = run_oracle(c)
    assert err == "" and oerr is None
    d = ps._data
    for key in ("particle_id", "state", "t", "ei"):
        np.testing.assert_array_equal(d[key], pd[key], err_msg=key)
    if schedule is not None:
        for k in "xyz":
            np.testing.assert_array_equal(d[k], pd[k], err_msg=k)
        return
    worst = max(int(ulp_diff_f32(d[k], pd[k]).max()) for k in "xyz")
    assert worst <= (0 if mesh == "flat" else 2), worst
