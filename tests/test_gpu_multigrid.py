"""FieldSets with more than one XGrid (reference: every Field has its own grid, the gridset lists the distinct ones and
``ei`` has one column per grid -- _core/field.py:102-134, _core/fieldset.py:225-235, _core/particle.py:182-222 -- while every
Field.eval hints with, and writes back, the LAST column: `igrid` stays -1, _core/field.py:101,173,311).  The velocity grid is
the engine's; a scalar field on another grid lives in its own device engine (fieldset.py _ExtraGrid)."""

import numpy as np
import pytest

import parcels_b200 as pb
from device_trig import DeviceTrig
from oracle import parcels_oracle as po
from oracle import trig
from parcels_b200.fieldset import XGrid

pytestmark = pytest.mark.gpu


def _setup(curvilinear_second):
    rng = np.random.default_rng(3)
    lon, lat, depth, times = np.linspace(0, 10, 21), np.linspace(40, 50, 17), np.linspace(0, 100, 5), np.arange(3) * 3600.0
    U = rng.uniform(-1, 1, (3, 5, 17, 21)).astype(np.float32)
    V = rng.uniform(-1, 1, (3, 5, 17, 21)).astype(np.float32)
    W = (1e-3 * rng.uniform(-1, 1, (3, 5, 17, 21))).astype(np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, depth=depth, time=times, U=U, V=V, W=W, mesh="spherical")
    if curvilinear_second:
        import cases

        lon2, lat2 = cases.curv_mesh(9, 11, True, np.dtype("f8"))
        lon2 = 5.0 + (lon2 - lon2.mean()) * (8.0 / np.ptp(lon2))  # over the velocity domain
        lat2 = 45.0 + (lat2 - lat2.mean()) * (8.0 / np.ptp(lat2))
        g2 = XGrid(lon2, lat2, None, mesh="spherical")
        shape = (3, 1, 9, 11)
    else:
        g2 = XGrid(np.linspace(-1, 11, 9), np.linspace(39, 51, 7), None, mesh="spherical")
        shape = (3, 1, 7, 9)
    wind = rng.uniform(-5, 5, shape)
    fs.add_field("wind", wind, grid=g2, interp_method="linear")
    n = 120
    x, y, z = rng.uniform(2, 8, n), rng.uniform(42, 48, n), rng.uniform(5, 90, n)
    og1 = po.OGrid(lon, lat, depth, mesh="spherical")
    ofs1 = po.OFieldSet(og1, U, V, W, time=times, interp="linear")
    og2 = po.OGrid(g2.lon, g2.lat, None, mesh="spherical")
    ofs2 = po.OFieldSet(og2, wind, wind, None, time=times, interp="linear")
    return fs, ofs1, ofs2, wind, (x, y, z), times


@pytest.mark.parametrize("curv, exact", [pytest.param(False, False, id="False"), pytest.param(True, False, id="True"),
                                         pytest.param(True, True, id="True-exact")])  # fmt: skip
def test_field_on_a_second_grid_samples_like_the_oracle(curv, exact):
    """`exact`: the curvilinear second grid against the oracle in engine arithmetic (the scalar sampler's trigonometry,
    tests/device_trig.py): values bit-exact instead of within 64 float32 ulp."""
    fs, ofs1, ofs2, wind, (x, y, z), times = _setup(curv)
    assert len(fs.gridset) == 2
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=np.zeros(len(x)))
    assert ps._data["ei"].shape == (len(x), 2)
    tq = np.full(len(x), 1234.5)
    v = fs.wind.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
    pd = po.create_particle_data(x, y, z, np.zeros(len(x)), ngrids=2)
    view = po.View(pd, np.ones(len(x), dtype=bool))
    with trig.use(DeviceTrig(scalar_sampler=True) if exact else trig.NumpyTrig()):
        ov = po.eval_scalar(ofs2, wind, "linear", tq, pd["z"], pd["y"], pd["x"], view)
    np.testing.assert_array_equal(ps._data["ei"][:, -1], pd["ei"][:, -1])
    np.testing.assert_array_equal(ps._data["state"], pd["state"])
    if curv and not exact:
        np.testing.assert_allclose(v, ov, rtol=0, atol=64 * np.finfo(np.float32).eps * 5.0)
    else:
        np.testing.assert_array_equal(v, ov)
    ps.populate_indices()  # one search per grid (reference _core/particleset.py:252-262)
    np.testing.assert_array_equal(ps._data["ei"][:, 1], pd["ei"][:, -1])
    assert np.any(ps._data["ei"][:, 0] != ps._data["ei"][:, 1])


def test_mixed_kernel_list_with_a_field_on_a_second_grid():
    """[AdvectionRK4_3D, a user kernel sampling the second grid's field]: the built-in runs on the device (velocity grid), the user
    kernel samples the other grid's engine; both share the last `ei` column like the reference's fields do."""
    fs, ofs1, ofs2, wind, (x, y, z), times = _setup(False)
    pclass = pb.Particle.add_variable(pb.Variable("w10", dtype=np.float64, initial=0.0))
    ps = pb.ParticleSet(fs, pclass=pclass, x=x, y=y, z=z, t=np.zeros(len(x)))

    def SampleWind(particles, fieldset):
        particles.w10 = fieldset.wind[particles]

    ps.execute([pb.AdvectionRK4_3D, SampleWind, pb.DeleteParticle], dt=600.0, runtime=3600.0)

    pd = po.create_particle_data(x, y, z, np.zeros(len(x)), ngrids=2)
    pd["w10"] = np.zeros(len(x))

    def OSample(p, fs_):
        p.w10 = po.eval_scalar(ofs2, wind, "linear", p.t, p.z, p.y, p.x, p)

    po.pset_execute(pd, ofs1, [po.AdvectionRK4_3D, OSample, po.DeleteOnError], 600.0, runtime=3600.0)
    assert len(ps) == len(pd["x"]) > 0
    for k in ("particle_id", "state", "t", "ei", "w10"):
        np.testing.assert_array_equal(ps._data[k], pd[k], err_msg=k)
    from engine_run import ulp_diff_f32

    for k in "xyz":
        assert ulp_diff_f32(ps._data[k], pd[k]).max() <= 2, k
    assert np.abs(ps._data["w10"]).max() > 0


def test_vector_field_on_a_second_grid_samples_like_the_oracle():
    """A wind-like VectorField on its own (coarser, 2-D) grid next to the ocean velocities: `fieldset.wind[particles]` in a user
    kernel, values / cells / states against the oracle's eval_uvw on that grid."""
    fs, ofs1, _, _, (x, y, z), times = _setup(False)
    rng = np.random.default_rng(9)
    g3 = XGrid(np.linspace(-2, 12, 8), np.linspace(38, 52, 6), None, mesh="spherical")
    U10 = rng.uniform(-8, 8, (3, 1, 6, 8)).astype(np.float32)
    V10 = rng.uniform(-8, 8, (3, 1, 6, 8)).astype(np.float32)
    fs.add_vector_field("wind10", U10, V10, grid=g3)
    assert len(fs.gridset) == 3
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=np.zeros(len(x)))
    tq = np.full(len(x), 2000.0)
    u, v = fs.wind10.eval(tq, ps._data["z"], ps._data["y"], ps._data["x"], ps)
    og = po.OGrid(g3.lon, g3.lat, None, mesh="spherical")
    ofs = po.OFieldSet(og, U10, V10, None, time=times, interp="linear")
    pd = po.create_particle_data(x, y, z, np.zeros(len(x)), ngrids=3)
    view = po.View(pd, np.ones(len(x), dtype=bool))
    ou, ov = po.eval_uvw(ofs, tq, pd["z"], pd["y"], pd["x"], view, False)
    np.testing.assert_array_equal(ps._data["ei"][:, -1], pd["ei"][:, -1])
    np.testing.assert_array_equal(ps._data["state"], pd["state"])
    scale = float(np.abs(ou).max())
    assert np.abs(u - ou).max() <= 4 * np.finfo(np.float32).eps * scale and np.abs(v - ov).max() <= 4 * np.finfo(np.float32).eps * scale
    ps.populate_indices()
    assert ps._data["ei"].shape[1] == 3 and np.array_equal(ps._data["ei"][:, 2], pd["ei"][:, -1])
