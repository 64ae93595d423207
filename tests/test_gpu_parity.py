"""GPU parity tests (-m gpu): the product path (parcels_b200 -> ctypes C-ABI -> sm_90a CUDA)
against the CPU oracle on the same seeded inputs, and against the committed outputs of the
reference itself (tests/golden/).

Bar (stated tolerance):
* particle_id, state, t, and the set of surviving particles: bit-exact;
* cell indices ``ei``: bit-exact;
* x, y, z: bit-exact on flat rectilinear meshes (only IEEE +,-,*,/,sqrt are involved, evaluated in the
  reference's order and dtype with FMA contraction off); on spherical meshes <= 2 float32 ulp
  (``cos`` of CUDA libdevice vs glibc/NumPy is not bit-identical); on curvilinear meshes <= 8 float32
  ulp (see CURV_ULP).
"""

import os

import numpy as np
import pytest

import cases
from engine_run import make_fieldset, run_engine, ulp_diff_f32
from oracle import parcels_oracle as po
from oracle_run import load_case, run_oracle
from philox_ref import device_normals, wiener_normals

pytestmark = pytest.mark.gpu

ERR_NAME = {60: "FieldOutOfBoundError", 61: "FieldOutOfBoundSurfaceError", 70: "OutsideTimeInterval",
            51: "FieldInterpolationError", 52: "GridSearchingError", 50: "GeneralError"}  # fmt: skip
FLAT_EXACT = {"flat_f32c_f64d", "c1_peninsula", "delayed_partial", "raise_oob", "raise_time", "rk2_3d", "through_surface",
              "cgrid_rect_3d", "freeslip_3d", "freeslip_surface", "nearest_f32_static"}
# Curvilinear search: the reference's closed-form bilinear inverse amplifies last-ulp differences (np.dot's
# BLAS summation order, libm vs libdevice trig) by the cell's condition number, and spatial-hash hits are
# rounded to float32 (spatialhash.py:511) -- a flipped rounding moves a weight by 6e-8.  Stated tolerance:
CURV_ULP = 8
NON_DIFFUSION = [n for n in cases.CASES if "DiffusionUniformKh" not in cases.CASES[n]["kernels"]]


def _compare(name, d, ref, exact_xyz):
    for key in ("particle_id", "state", "t", "dt"):
        np.testing.assert_array_equal(d[key], ref[key], err_msg=f"{name}:{key}")
    np.testing.assert_array_equal(d["ei"], ref["ei"], err_msg=f"{name}:ei")
    for key in ("x", "y", "z"):
        if exact_xyz:
            np.testing.assert_array_equal(d[key], ref[key], err_msg=f"{name}:{key}")
        else:
            ulps = ulp_diff_f32(d[key], ref[key])
            tol = CURV_ULP if name.startswith("curv") else 2
            assert ulps.max() <= tol, f"{name}:{key} differs by {ulps.max()} f32 ulp"


@pytest.mark.parametrize("name", NON_DIFFUSION)
def test_engine_matches_oracle(name):
    c = load_case(name)
    ps, err = run_engine(c)
    pd, oerr = run_oracle(c)
    assert err == (ERR_NAME[oerr] if oerr else "")
    if name == "raise_time":
        # whole-view OutsideTimeInterval: states/positions/time pinned; dx/ei of the aborted step waived
        np.testing.assert_array_equal(ps._data["state"], pd["state"])
        for key in ("x", "y", "z", "t"):
            np.testing.assert_array_equal(ps._data[key], pd[key])
        return
    _compare(name, ps._data, pd, name in FLAT_EXACT)


@pytest.mark.parametrize("name", NON_DIFFUSION)
def test_engine_matches_reference_outputs(name, golden_dir):
    """Against outputs of the reference's own code (tests/golden/ref_cases.npz)."""
    g = np.load(os.path.join(golden_dir, "ref_cases.npz"))
    c = load_case(name)
    ps, err = run_engine(c)
    assert err == str(g[f"{name}/error"])
    ref = {k: g[f"{name}/{k}"] for k in ("particle_id", "state", "t", "dt", "ei", "x", "y", "z")}
    if name == "raise_time":
        np.testing.assert_array_equal(ps._data["state"], ref["state"])
        return
    _compare(name, ps._data, ref, name in FLAT_EXACT)


V3_FILES = {"linear": "v3_jit_linear.npz", "cgrid_velocity": "v3_jit_cgrid.npz", "freeslip": "v3_jit_freeslip.npz",
            "nearest": "v3_jit_nearest.npz"}  # fmt: skip


@pytest.mark.parametrize("interp", list(V3_FILES))
def test_engine_reproduces_v3_jit_goldens(golden_dir, interp):
    """The reference's own regression test (tests/test_interpolation.py:297-378), atol 1e-6."""
    import parcels_b200 as pb

    g = np.load(os.path.join(golden_dir, V3_FILES[interp]))
    lon, lat, depth = (g[k].astype(np.float32) for k in ("lon", "lat", "depth"))
    x, y, z = np.meshgrid(np.linspace(0, 1, 7), np.linspace(0, 1, 13), np.linspace(0, 1, 5))
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, depth=depth, time=g["time"], U=g["U"], V=g["V"], W=g["W"], mesh="flat",
                                 interp_method=interp, padding=("low", "low", "high"))  # fmt: skip
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=np.zeros(x.size))
    n = x.size
    obs = {k: np.full((n, 5), np.nan, dtype=np.float32) for k in "xyz"}

    class Recorder:
        outputdt = 1.0
        i = 0

        def write(self, pset, _time):
            for k in "xyz":
                obs[k][pset._data["particle_id"], self.i] = pset._data[k]
            self.i += 1

    ps.execute([pb.AdvectionRK4_3D, pb.DeleteParticle], dt=1.0, runtime=4.0, output_file=Recorder())
    for k, gk in (("x", "gold_lon"), ("y", "gold_lat"), ("z", "gold_z")):
        np.testing.assert_allclose(obs[k][:, :4], g[gk], atol=1e-6, equal_nan=True)


def test_device_philox_matches_numpy_restatement():
    from parcels_b200.engine import Engine

    eng = Engine(0)
    pid = np.array([0, 1, 2, 12345, 2**33 + 7, 10**12], dtype=np.int64)
    dev = eng.debug_normals(seed=0xDEADBEEFCAFE, rng_call=3, it=17, particle_id=pid)
    zx, zy = wiener_normals(0xDEADBEEFCAFE, 3, 17, pid)
    # float32 Box-Muller on both sides: logf / sincospif of CUDA against NumPy's float32 log / sin / cos
    np.testing.assert_allclose(dev[:, 0], zx, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(dev[:, 1], zy, rtol=2e-5, atol=2e-6)


def test_fused_diffusion_matches_oracle_with_same_normals():
    """DiffusionUniformKh: deterministic part compared with the oracle fed the engine's Philox
    stream; statistical parity with the reference's RNG is covered in test_gpu_properties."""
    c = load_case("diffusion")
    seed = 99
    ps, err = run_engine(c, seed=seed)
    assert err == ""
    calls = {"n": 0}

    # one Kernel.execute call per segment, one normal pair per particle per iteration
    state = {"call": 1, "it": 0}

    def normal(view):
        zx, zy = device_normals(seed, state["call"], state["it"], view.particle_id)
        state["it"] += 1
        calls["n"] += 1
        return zx, zy

    pd, oerr = run_oracle(c, normal=normal)
    assert oerr is None and calls["n"] > 0
    np.testing.assert_array_equal(ps._data["particle_id"], pd["particle_id"])
    np.testing.assert_array_equal(ps._data["state"], pd["state"])
    np.testing.assert_array_equal(ps._data["ei"], pd["ei"])
    for key in ("x", "y", "z"):
        ulps = ulp_diff_f32(ps._data[key], pd[key])
        assert ulps.max() <= 4, f"{key}: {ulps.max()} ulp"
