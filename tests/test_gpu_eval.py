"""GPU parity of ONE VectorField.eval (pb_sample_velocity) against the oracle's eval_uvw:
cell indices and error states bit-exact; velocities
  * bit-exact on flat rectilinear A-grid meshes (same operations, same dtypes, no transcendental function),
  * <= 32 float64 ulp on flat rectilinear C-grids: the reference's np.einsum("ij,ji->i", ...) (jacobian, mid-edge latitudes)
    is not reproducible to the last bit itself -- with float64 barycentric coordinates against float32 corner coordinates it
    takes NumPy's buffered (casting) inner loop, whose SIMD / FMA rounding differs from the same-dtype loop and changes with
    the batch size (measured here: einsum of the SAME rows gives different last bits for n = 1, 3 and n = 2, 5, 400);
    the engine sums left to right, which is what einsum does when the dtypes agree,
  * on spherical rectilinear meshes within a few ulp OF THE DTYPE THE ARITHMETIC RUNS IN (CUDA's cos / cosf against glibc's):
    <= 4 float32 ulp where NumPy's promotion makes the unit conversion float32 -- float32 positions -- or the whole value
    float32, <= 64 float64 ulp otherwise (a lerp done in the wrong dtype is a 1e-8 relative error, 4e7 float64 ulp, and fails),
  * <= 64 float32 ulp on curvilinear meshes (hash hits carry float32-rounded (xsi, eta); the closed-form bilinear inverse
    amplifies last-ulp trig differences),
all relative to the largest velocity of the batch (a sum of products has no better scale).

In engine arithmetic (``-exact`` ids: the oracle's sin / cos are the device's own functions and waivers 4 and 8 take the engine's
resolution, tests/device_trig.py) every case that has a tolerance above is compared bit for bit instead: float32 and float64
positions, un-hinted and hinted."""

import numpy as np
import pytest

import cases
from engine_run import make_fieldset
from oracle import parcels_oracle as po
from device_trig import DeviceTrig
from oracle import trig
from oracle_run import load_case, oracle_fieldset

pytestmark = pytest.mark.gpu

NAMES = ["c2_small", "flat_f32c_f64d", "all_f32", "c1_peninsula", "cgrid_rect_3d", "cgrid_rect_sph", "curv_flat_2d",
         "curv_sph_2d", "curv_sph_3d", "curv_sph_f32", "curv_lin_flat_2d", "curv_lin_sph_3d", "curv_lin_sph_f32", "freeslip_3d", "partialslip_sph", "nearest_3d", "freeslip_surface",
         "sph_equator", "sph_polar_f32", "cgrid_rect_sph_f32", "curv_sph_dateline"]  # fmt: skip


# the cases whose NumPy-trig comparison needs a tolerance get a second, bit-exact comparison in engine arithmetic
EVAL_MODES = [pytest.param(n, False, id=n) for n in NAMES] + [
    pytest.param(n, True, id=f"{n}-exact") for n in NAMES if n.startswith(("curv", "cgrid")) or cases.CASES[n]["mesh"] == "spherical"
]


def _assert_values(name, c, f32_positions, got, want, what, exact=False):
    want = np.asarray(want)
    if exact:
        np.testing.assert_array_equal(np.asarray(got, dtype=np.float64), want.astype(np.float64), err_msg=f"{name} {what}")
        return
    scale = float(np.abs(want[np.isfinite(want)]).max()) if np.isfinite(want).any() else 0.0
    if name.startswith("curv"):
        tol = 64 * np.finfo(np.float32).eps
    elif c["mesh"] == "spherical":
        tol = 4 * np.finfo(np.float32).eps if (f32_positions or want.dtype == np.float32) else 64 * np.finfo(np.float64).eps
    elif name.startswith("cgrid"):
        tol = 32 * np.finfo(np.float64).eps
    else:
        tol = 0.0
    err = np.abs(np.asarray(got, dtype=np.float64) - want.astype(np.float64))
    err = np.where(np.isnan(want) & np.isnan(got), 0.0, err)
    worst = float(np.nanmax(err)) if err.size else 0.0
    assert worst <= tol * scale, f"{name} {what}: max |diff| {worst:.3e} = {worst / max(scale, 1e-300):.3e} x scale, allowed {tol:.3e} x scale"


def _oracle_eval(ofs, t, z, y, x, three_d, hint):
    n = len(x)
    pd = po.create_particle_data(np.zeros(n), np.zeros(n), np.zeros(n), 0.0, ngrids=ofs.ngrids)
    pd["ei"][:, -1] = hint
    view = po.View(pd, np.ones(n, dtype=bool))
    out = po.eval_uvw(ofs, t, z, y, x, view, three_d)
    return out, pd["ei"][:, -1].copy(), pd["state"].copy()


@pytest.mark.parametrize("name, exact", EVAL_MODES)
@pytest.mark.parametrize("f32", [True, False])
def test_single_eval_matches_oracle(name, exact, f32):
    with trig.use(DeviceTrig() if exact else trig.NumpyTrig()):
        _single_eval_vs_oracle(name, f32, exact)


def _single_eval_vs_oracle(name, f32, exact):
    c = load_case(name)
    fs = make_fieldset(c)
    ofs = oracle_fieldset(c)
    three_d = c["W"] is not None
    dt = np.float32 if f32 else np.float64
    x, y, z = (np.asarray(c[k]).astype(dt) for k in "xyz")
    tmax = 0.0 if c["times"] is None else float(c["times"][-1])
    t = np.full(len(x), 0.37 * tmax)
    eng = fs.engine(0)
    # first eval of a fresh ParticleSet: ei = 0 for everyone => no hint (curvilinear), then with the found cells as hint
    (ou, ov, *ow), oei, ost = _oracle_eval(ofs, t, z, y, x, three_d, np.zeros(len(x), dtype=np.int32))
    u, v, w, ei, st = eng.sample_velocity(t, z, y, x, three_d=three_d, positions_are_f32=f32, ei_hint=np.zeros(len(x), np.int32),
                                          no_hint=True)  # fmt: skip
    np.testing.assert_array_equal(ei, oei)
    np.testing.assert_array_equal(st, ost)
    _assert_values(name, c, f32, u, ou, "u", exact)
    _assert_values(name, c, f32, v, ov, "v", exact)
    # second eval, slightly displaced, hinted with the cells just found
    x2 = (x + dt(0.01) * (x.max() - x.min()) / 30).astype(dt)
    (ou, ov, *ow), oei2, ost2 = _oracle_eval(ofs, t, z, y, x2, three_d, oei)
    u, v, w, ei2, st2 = eng.sample_velocity(t, z, y, x2, three_d=three_d, positions_are_f32=f32, ei_hint=oei)
    np.testing.assert_array_equal(ei2, oei2)
    np.testing.assert_array_equal(st2, ost2)
    _assert_values(name, c, f32, u, ou, "u (hinted)", exact)
    _assert_values(name, c, f32, v, ov, "v (hinted)", exact)
    if three_d:
        _assert_values(name, c, f32, w, ow[0], "w (hinted)", exact)


@pytest.mark.parametrize("name", ["c2_small", "flat_f32c_f64d", "curv_sph_2d", "diffusion"])
def test_populate_indices_matches_oracle_search(name):
    """ParticleSet.populate_indices (reference _core/particleset.py:252-262): ei[:, i] = ravel_index(grid_i.search(z, y, x))
    for every grid of the gridset, the search of the fieldset's grid done on the device."""
    import parcels_b200 as pb

    c = load_case(name)
    fs = make_fieldset(c)
    ofs = oracle_fieldset(c)
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    ps.populate_indices()
    d = ps._data
    (zi, _), (yi, _), (xi, _) = po.grid_search(ofs.grid, d["z"], d["y"], d["x"], None)
    np.testing.assert_array_equal(d["ei"][:, 0], po.ravel_index(ofs.grid, zi, yi, xi).astype(np.int32))
    assert d["ei"].shape[1] == ofs.ngrids and not d["ei"][:, 1:].any()
