"""GPU parity (-m gpu) of AdvectionDiffusionM1 / AdvectionDiffusionEM (csrc/advdiff.cu, pb_advect_diffusion) against the
CPU oracle fed the engine's own Philox stream: ids, states, times, surviving set and cell indices bit-exact; positions
bit-exact on flat meshes, <= 4 float32 ulp on spherical meshes (CUDA cos / cosf vs glibc) -- ulps of max(|x|, D), D = the
largest displacement any particle made in the run: the longitudes of these cases cross zero, where a 1-ulp rounding flip made
while the particle was at |x| ~ 0.4 deg is 30 ulps of a final x = 0.02 deg (every particle agrees to <= 3 ulp except the one
that ends next to zero; and with the oracle alone: perturbing its float32 cos by 1 ulp moves a particle
ending at x = -0.0008 by 150 of ITS ulps).  The oracle itself is pinned to
the reference's outputs with the reference's RNG (tests/test_advdiff_cpu.py).  Statistical check against the reference's
own test (tests/test_diffusion.py:49-81): zero mean, zonal skew > meridional skew on a field with a zonal Kh gradient.
The spherical cases run once more against the oracle in engine arithmetic (``-exact`` ids: the device's cosf in the Kh metric and
its cos in the unit conversion, tests/device_trig.py): positions bit-exact there too."""

import numpy as np
import pytest

from advdiff_run import case_inputs, run_engine_advdiff, run_oracle_advdiff
from device_trig import DeviceTrig
from engine_run import ulp_diff_f32
from oracle import trig
from oracle.make_golden import ADVDIFF_CASES
from philox_ref import device_normals, wiener_normals

pytestmark = pytest.mark.gpu
ERR_NAME = {60: "FieldOutOfBoundError", 61: "FieldOutOfBoundSurfaceError", 70: "OutsideTimeInterval", 51: "FieldInterpolationError"}
FLAT = {"m1_flat", "em_f64_static", "em_raise", "m1_cgrid_flat"}
ADVDIFF_MODES = [pytest.param(n, False, id=n) for n in ADVDIFF_CASES] + [
    pytest.param(n, True, id=f"{n}-exact") for n in ADVDIFF_CASES if n not in FLAT
]


@pytest.mark.parametrize("name, exact", ADVDIFF_MODES)
def test_advdiff_matches_oracle_with_same_normals(name, exact):
    seed = 4242
    ps, err = run_engine_advdiff(name, seed=seed)
    state = {"it": 0}

    def normal(view):  # one Kernel.execute call (rng_call = 1), one normal pair per particle and loop iteration
        zx, zy = device_normals(seed, 1, state["it"], view.particle_id)
        state["it"] += 1
        return zx, zy

    with trig.use(DeviceTrig() if exact else trig.NumpyTrig()):
        pd, oerr = run_oracle_advdiff(name, normal=normal)
    assert err == (ERR_NAME[oerr] if oerr else "")
    d = ps._data
    c0 = case_inputs(name)[0]
    for key in ("particle_id", "state", "t", "dt", "ei"):
        np.testing.assert_array_equal(d[key], pd[key], err_msg=f"{name}:{key}")
    for key in ("x", "y", "z"):
        if exact or name in FLAT:
            np.testing.assert_array_equal(d[key], pd[key], err_msg=f"{name}:{key}")
        else:
            start = np.asarray(c0[key], dtype=np.float64)[pd["particle_id"]]
            ulps = ulp_diff_f32(d[key], pd[key], floor=max(float(np.abs(pd[key] - start).max()), 1e-30))
            assert ulps.max() <= 4, f"{name}:{key} differs by {ulps.max()} f32 ulp"


@pytest.mark.parametrize("kernel", ["AdvectionDiffusionM1", "AdvectionDiffusionEM"])
@pytest.mark.parametrize("mesh", ["spherical", "flat"])
def test_spatially_varying_diffusion_statistics(mesh, kernel):
    """Known answer for a diffusivity that is linear in x, K = K0 + g x (Ito drift towards larger K): after time T
    E[x] = g T, E[y] = 0, Var ~ 2 K0 T.  The reference's own test of these kernels (tests/test_diffusion.py:49-81) uses a
    gradient so weak that its skewness assertion is decided by the seed (effect 5e-3, sampling noise 2.4e-2); the
    moments below are 6 sigma effects."""
    import parcels_b200 as pb

    ydim, xdim = 100, 200
    conv = 1 / 1852.0 / 60 if mesh == "spherical" else 1
    lon, lat = np.linspace(-1e6, 1e6, xdim), np.linspace(-1e6, 1e6, ydim)
    K0, g, T, npart = 500.0, 0.02, 3 * 3600.0, 40000
    Kh = np.broadcast_to((K0 + g * lon)[None, None, None, :], (2, 1, ydim, xdim)).astype(np.float64)
    if mesh == "spherical":
        lon, lat = lon * conv, lat * conv
    Z = np.zeros((2, 1, ydim, xdim), dtype=np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, time=np.array([0.0, 86400.0]), U=Z, V=Z, mesh=mesh)
    fs.add_field("Kh_zonal", Kh.copy())
    fs.add_field("Kh_meridional", np.full_like(Kh, K0))
    fs.add_context("dres", float(lon[1] - lon[0]))
    ps = pb.ParticleSet(fs, x=np.zeros(npart), y=np.zeros(npart), seed=1636)
    ps.execute(getattr(pb, kernel), runtime=T, dt=3600.0)
    assert np.all(ps.state == 1) and len(ps) == npart
    x, y = np.asarray(ps.x, dtype=np.float64) / conv, np.asarray(ps.y, dtype=np.float64) / conv  # metres (cos(lat) ~ 1 at the equator)
    sigma = np.sqrt(2 * K0 * T)
    sem = sigma / np.sqrt(npart)
    assert abs(np.mean(x) - g * T) < 4 * sem, (np.mean(x), g * T, sem)
    assert abs(np.mean(y)) < 4 * sem
    assert abs(np.std(y) / sigma - 1) < 0.03 and abs(np.std(x) / sigma - 1) < 0.06


def test_advdiff_in_a_mixed_list_matches_oracle():
    """[AdvectionDiffusionEM, user kernel, user error handler]: the loop runs on the host (stepwise.py), the built-in still on the
    device -- one pb_advect_diffusion(kernels_only) launch per step, its Wiener increments keyed by the launch counter."""
    import parcels_b200 as pb
    from engine_run import make_fieldset
    from oracle import parcels_oracle as po
    from oracle_run import oracle_fieldset

    c, kern, kz, km, dres, dt, runtime, _, _ = case_inputs("em_f64_static")
    seed = 77
    fs = make_fieldset(c)
    fs.add_field("Kh_zonal", kz)
    fs.add_field("Kh_meridional", km)
    fs.add_context("dres", dres)
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"], seed=seed)

    def Drift(particles, fieldset):
        particles.dx += 1.5

    def DeleteErr(particles, fieldset):
        particles[particles.state >= 50].state = 30

    ps.execute([getattr(pb, kern), Drift, DeleteErr], dt=dt, runtime=runtime)

    ofs = oracle_fieldset(c)
    ofs.scalars = {"Kh_zonal": (kz, "linear"), "Kh_meridional": (km, "linear")}
    ofs.context["dres"] = dres
    pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"])
    launch = {"k": 0}

    def normal(view):
        launch["k"] += 1
        return device_normals(seed, launch["k"], 0, view.particle_id)

    def ODrift(p, fs_):
        p.dx = p.dx + 1.5

    po.pset_execute(pd, ofs, [getattr(po, kern)(normal), ODrift, po.DeleteOnError], dt, runtime=runtime)
    assert len(ps) == len(pd["x"]) > 0 and launch["k"] == int(round(runtime / dt))
    for key in ("particle_id", "state", "t", "ei", "x", "y", "z"):
        np.testing.assert_array_equal(ps._data[key], pd[key], err_msg=key)
