"""CPU tests of the boundary and the host logic (no GPU, no compute calls):
the C-ABI library loads and exports every symbol include/parcels_b200.h declares, the host
mirror validates arguments like the reference, and the product fails loudly without a GPU."""

import os
import re

import numpy as np
import pytest

import parcels_b200 as pb
from parcels_b200 import _lib
from parcels_b200.particleset import KernelPlan
from parcels_b200.plan import FixedStep, PythonStep
from philox_ref import philox4x32_10, wiener_normals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    from parcels_b200 import build

    build.build()


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "parcels_b200.h")).read()
    declared = set(re.findall(r"\b(pb_[a-z_0-9]+)\s*\(", header))
    assert declared, "no declarations parsed"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    assert lib.pb_abi_version() == 1


def test_struct_layouts_match_header():
    import ctypes

    assert ctypes.sizeof(_lib.AdvectArgs) == 4 * 4 + 5 * 8 + 2 * 8 + 8 + 4 * 4
    assert ctypes.sizeof(_lib.Report) == 11 * 8 + 2 * 4 + 2 * 4
    assert ctypes.sizeof(_lib.Rk45Args) == 5 * 8 + 8 + 6 * 4
    assert ctypes.sizeof(_lib.ParticleArrays) == 10 * 8
    assert ctypes.sizeof(_lib.AdvDiffArgs) == 4 * 4 + 4 * 8 + 2 * 8 + 8 + 4 * 4


def _fs(with_w=True):
    z = np.zeros((2, 3, 4, 5), np.float32)
    return pb.FieldSet.from_arrays(lon=np.linspace(0, 1, 5), lat=np.linspace(0, 1, 4), depth=np.linspace(0, 1, 3),
                                   time=np.array([0.0, 10.0]), U=z, V=z, W=z if with_w else None, mesh="flat")  # fmt: skip


def test_kernel_plan_lowering():
    fs = _fs()
    p = KernelPlan([pb.AdvectionRK4_3D, pb.DeleteParticle], fs)
    assert (p.kind, p.scheme, p.diffusion, p.delete_on_error) == ("fixed", 5, False, True)
    fs.add_constant_field("Kh_zonal", 100, mesh="flat")
    fs.add_constant_field("Kh_meridional", 50, mesh="flat")
    p = KernelPlan([pb.AdvectionRK4, pb.DiffusionUniformKh], fs)
    assert (p.scheme, p.diffusion, p.delete_on_error, p.kh) == (4, True, False, (100.0, 50.0))
    assert len(fs.gridset) == 2  # constant fields live on their own grid => ei has 2 columns


def test_kernel_plan_mixed_lists_lower_to_step_records_with_builtins_on_the_device():
    def MyKernel(particles, fieldset):
        pass

    def DeleteParticle(particles, fieldset):  # a USER function that merely shares the token's name
        pass

    fs = _fs()
    fs.add_constant_field("Kh_zonal", 1.0, mesh="flat")
    fs.add_constant_field("Kh_meridional", 1.0, mesh="flat")
    p = KernelPlan([pb.AdvectionRK4, pb.DiffusionUniformKh, MyKernel, DeleteParticle], fs)
    assert p.kind == "stepwise" and p.stepwise and [type(s) for s in p.items] == [FixedStep, PythonStep, PythonStep]
    assert p.items[0] == FixedStep(scheme=4, diffusion=True)  # AdvectionRK4 fused with DiffusionUniformKh in one device call
    assert p.items[2].func is DeleteParticle
    with pytest.raises(AttributeError):  # the records are immutable: fusing replaces the step, it never edits one
        p.items[0].diffusion = False
    alone = KernelPlan([MyKernel, pb.DiffusionUniformKh, MyKernel], fs)  # no advection step to fuse with: diffusion on its own
    assert alone.items == (PythonStep(MyKernel), FixedStep(scheme=0, diffusion=True), PythonStep(MyKernel))
    assert not KernelPlan([pb.AdvectionRK4, pb.DeleteParticle], fs).stepwise  # built-ins only: one fused launch
    with pytest.raises(TypeError):
        KernelPlan([1], _fs())
    with pytest.raises(ValueError):
        KernelPlan([], _fs())
    with pytest.raises(AttributeError):
        KernelPlan([pb.AdvectionRK4_3D], _fs(with_w=False))


def test_particlesetview_write_through_semantics():
    """reference _core/particlesetview.py: reads are masked copies, in-place ops / assignments write through"""
    from parcels_b200.particlesetview import ParticleSetView

    d = {"x": np.arange(5, dtype=np.float32), "state": np.array([10, 60, 10, 51, 10], np.int32), "ei": np.zeros((5, 1), np.int32),
         "dt": np.full(5, 2.0)}  # fmt: skip
    v = ParticleSetView(d, np.array([True, True, False, True, True]))
    v.x += 10
    np.testing.assert_array_equal(d["x"], [10, 11, 2, 13, 14])
    v[v.state >= 50].state = 30
    np.testing.assert_array_equal(d["state"], [10, 30, 10, 30, 10])
    assert (v.x + v.x * 0.5 * v.dt).dtype == np.float64 and len(v.x) == 4 and v.x.max() == 14
    v.ei[:, -1] = 7
    np.testing.assert_array_equal(d["ei"].ravel(), [7, 7, 0, 7, 7])
    v.x = v.x - 1
    np.testing.assert_array_equal(d["x"], [9, 10, 2, 12, 13])
    v[1:3].x = 0  # integer/slice indices are relative to the view
    np.testing.assert_array_equal(d["x"], [9, 0, 2, 0, 13])


def test_builtin_kernels_have_no_cpu_body():
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        pb.AdvectionRK4(None, None)


def test_particleset_layout_matches_reference_default_particle():
    ps = pb.ParticleSet(_fs(), x=[0.1, 0.2], y=[0.1, 0.2], z=[0.5, 0.5], t=np.array([0.0, 1.0]))
    d = ps._data
    assert {k: v.dtype for k, v in d.items()} == {
        "ei": np.int32, "t": np.float64, "z": np.float32, "y": np.float32, "x": np.float32, "particle_id": np.int64,
        "dz": np.float32, "dy": np.float32, "dx": np.float32, "dt": np.float64, "state": np.int32,
    }  # fmt: skip
    assert d["ei"].shape == (2, 1) and (d["state"] == pb.StatusCode.Evaluate).all()


def test_execute_argument_validation():
    ps = pb.ParticleSet(_fs(), x=[0.1], y=[0.1], z=[0.5], t=[0.0])
    with pytest.raises(ValueError, match="mutually exclusive"):
        ps.execute(pb.AdvectionRK4, dt=1.0, runtime=1.0, endtime=2.0)
    with pytest.raises(ValueError, match="non-zero"):
        ps.execute(pb.AdvectionRK4, dt=0.0, runtime=1.0)
    with pytest.raises(ValueError, match="Either runtime or endtime"):
        ps.execute(pb.AdvectionRK4, dt=1.0)
    with pytest.raises(ValueError, match="not in fieldset time interval"):
        ps.execute(pb.AdvectionRK4, dt=1.0, endtime=100.0)


def test_no_gpu_means_loud_failure_not_fallback():
    if _lib.load().pb_device_count() > 0:
        pytest.skip("a GPU is present")
    ps = pb.ParticleSet(_fs(), x=[0.1], y=[0.1], z=[0.5], t=[0.0])
    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        ps.execute(pb.AdvectionRK4, dt=1.0, runtime=2.0)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "parcels_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src and "parcels_oracle" not in src, f


def test_philox_known_answer():
    """Random123 known-answer vectors for philox4x32-10."""
    out = philox4x32_10([0], [0], [0], [0], 0, 0)
    assert [int(o[0]) for o in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    out = philox4x32_10([0xFFFFFFFF], [0xFFFFFFFF], [0xFFFFFFFF], [0xFFFFFFFF], 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(o[0]) for o in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    zx, zy = wiener_normals(7, 1, 0, np.arange(200000))
    assert abs(zx.mean()) < 0.01 and abs(zy.std() - 1) < 0.01


def test_host_spatial_hash_equals_oracle_table():
    """The product's host-side table build must give the reference's table (here: via the oracle
    restatement, itself pinned to the reference's own SpatialHash by tests/test_oracle_vs_reference.py)."""
    import cases
    from oracle import curvilinear_oracle as co
    from oracle import parcels_oracle as po
    from parcels_b200.spatialhash import build_spatial_hash

    for spherical, cd in ((False, "f8"), (True, "f8"), (True, "f4")):
        lon, lat = cases.curv_mesh(23, 31, spherical, np.dtype(cd))
        h = build_spatial_hash(lon, lat, spherical)
        o = co.OHash(po.OGrid(lon, lat, None, mesh="spherical" if spherical else "flat"))
        assert h["bitwidth"] == o.bitwidth
        np.testing.assert_array_equal(h["keys"], o.keys)
        np.testing.assert_array_equal(h["starts"], o.starts)
        np.testing.assert_array_equal(h["counts"], o.counts)
        np.testing.assert_array_equal(h["faces"], o.faces)
        np.testing.assert_array_equal(h["box"], np.array([float(b) for b in o.box]))


def test_window_range_policy():
    """time-slab streaming: which levels must be resident for a particle at time t (host logic only)"""
    from parcels_b200.fieldset import window_range

    t = np.arange(6) * 100.0  # levels at 0, 100, ..., 500
    assert window_range(t, 0.0, 1, 3) == (0, 3)
    assert window_range(t, 100.0, 1, 3) == (1, 3)  # on a level: that level starts the window
    assert window_range(t, 250.0, 1, 3) == (2, 3)
    assert window_range(t, 450.0, 1, 3) == (3, 3)  # clipped so that 3 levels still fit
    assert window_range(t, 500.0, 1, 2) == (4, 2)
    assert window_range(t, 500.0, -1, 3) == (3, 3)
    assert window_range(t, 250.0, -1, 3) == (1, 3)  # covers [100, 300]
    assert window_range(t, 200.0, -1, 3) == (0, 3)
    assert window_range(t, 50.0, -1, 3) == (0, 3)
    for sign in (1, -1):  # the particle's own time is always inside the window
        for tt in np.linspace(0, 500, 41):
            f, n = window_range(t, tt, sign, 3)
            assert t[f] <= tt <= t[f + n - 1] and n >= 2


def test_pset_add_iadd_iter():
    """reference tests/test_particleset.py:126-162,173-178 (test_pset_add_explicit / _implicit / _in_loop / merge / iterator)."""
    fs = _fs()
    npart = 11
    lon, lat = np.linspace(0, 1, npart), np.linspace(1, 0, npart)
    pset = pb.ParticleSet(fs, x=lon[0], y=lat[0])
    for i in range(1, npart):
        pset.add(pb.ParticleSet(fs, x=lon[i], y=lat[i]))
    assert len(pset) == npart
    assert np.allclose([p.x for p in pset], lon, atol=1e-7) and np.allclose([p.y for p in pset], lat, atol=1e-7)
    assert np.allclose(np.diff(pset._data["particle_id"]), np.ones(npart - 1))
    pset = pb.ParticleSet(fs, x=np.zeros(3), y=np.ones(3))
    pset += pb.ParticleSet(fs, x=np.ones(4), y=np.zeros(4))
    assert len(pset) == 7 and np.allclose(np.diff(pset._data["particle_id"]), np.ones(6))
    pset = pb.ParticleSet(fs, x=[], y=[])
    for _ in range(10):
        pset += pb.ParticleSet(fs, x=0.1, y=0.1)
    assert pset.size == 10 and pset._data["ei"].shape == (10, 1)
    for i, particle in enumerate(pb.ParticleSet(fs, x=np.zeros(5), y=np.ones(5))):
        assert particle.particle_id == i
    assert i == 4


def test_pset_warnings_and_index_helpers():
    """reference tests/test_particleset.py:100-103 (release outside the time domain warns), data_indices / error-particle helpers
    (_core/particleset.py:294-341), from_particlefile (not implemented in v4 either)."""
    fs = _fs()
    with pytest.warns(pb.ParticleSetWarning, match="Some particles are set to be released"):
        pb.ParticleSet(fs, x=[0.5] * 3, y=[0.5] * 3, t=[0.0, 5.0, 20.0])
    ps = pb.ParticleSet(fs, x=np.linspace(0, 1, 6), y=np.zeros(6))
    ps._data["state"][:] = [0, 10, 50, 60, 30, 1]
    np.testing.assert_array_equal(ps.data_indices("state", [50, 60]), [2, 3])
    np.testing.assert_array_equal(ps.data_indices("state", 30), [4])
    np.testing.assert_array_equal(ps._error_particles, [2, 3, 4, 5])
    assert ps._num_error_particles == 4
    with pytest.raises(NotImplementedError):
        pb.ParticleSet.from_particlefile(fs, pb.Particle, "x.parquet")


def test_kernel_object_and_signature_checks():
    """reference tests/test_kernel.py:54-165 (test_kernel_init / _merging / _from_list / _from_list_error_checking /
    test_RK45Kernel_error_no_next_dt / test_kernel_signature), against the host mirror's Kernel."""
    fs = _fs()
    pset = pb.ParticleSet(fs, x=[0.5], y=[0.5])

    def MoveEast(particles, fieldset):
        particles.dx += 0.1

    def MoveNorth(particles, fieldset):
        particles.dy += 0.1

    pb.Kernel(kernels=[pb.AdvectionRK4], pset=pset)
    merged = pb.Kernel(kernels=[pb.AdvectionRK4, MoveEast, MoveNorth], pset=pset)
    assert merged.funcname == "AdvectionRK4MoveEastMoveNorth" and merged._kernels == [pb.AdvectionRK4, MoveEast, MoveNorth]
    merged = pb.Kernel(kernels=[MoveEast, MoveNorth, pb.AdvectionRK4], pset=pset)
    assert merged.funcname == "MoveEastMoveNorthAdvectionRK4" and len(merged._kernels) == 3
    with pytest.raises(ValueError, match="List of `kernels` should have at least one function."):
        pb.Kernel(kernels=[], pset=pset)
    with pytest.raises(TypeError, match=r"Argument `kernels` should be a function or list of functions.*"):
        pb.Kernel(kernels=[pb.AdvectionRK4, "something else"], pset=pset)
    with pytest.raises(TypeError, match=r".* should be a function or list of functions.*"):
        pb.Kernel(kernels=[pb.Kernel(kernels=[pb.AdvectionRK4], pset=pset), MoveEast, MoveNorth], pset=pset)
    with pytest.raises(ValueError, match='ParticleClass requires a "next_dt" for AdvectionRK45 Kernel.'):
        pb.Kernel(kernels=[pb.AdvectionRK45], pset=pset)

    def good_kernel(particles, fieldset):
        pass

    def version_3_kernel(particle, fieldset, time):
        pass

    def version_3_kernel_without_time(particle, fieldset):
        pass

    def kernel_switched_args(fieldset, particle):
        pass

    def kernel_with_forced_kwarg(particles, *, fieldset=0):
        pass

    pb.Kernel(kernels=[good_kernel], pset=pset)
    with pytest.raises(ValueError, match="Kernel function must have 2 parameters, got 3"):
        pb.Kernel(kernels=[version_3_kernel], pset=pset)
    with pytest.raises(ValueError, match="Parameter 'particle' has incorrect name. Expected 'particles', got 'particle'"):
        pb.Kernel(kernels=[version_3_kernel_without_time], pset=pset)
    with pytest.raises(ValueError, match="Parameter 'fieldset' has incorrect name. Expected 'particles', got 'fieldset'"):
        pb.Kernel(kernels=[kernel_switched_args], pset=pset)
    with pytest.raises(ValueError, match="Parameter 'fieldset' has incorrect parameter kind. Expected POSITIONAL_OR_KEYWORD, got KEYWORD_ONLY"):
        pb.Kernel(kernels=[kernel_with_forced_kwarg], pset=pset)
    with pytest.raises(ValueError, match="2 parameters"):  # execute() checks the same
        pset.execute(version_3_kernel, dt=1.0, runtime=1.0)


def test_fieldset_context_is_an_attribute():
    """reference tests/test_kernel.py:27-51: `fieldset.add_context(name, v)` makes `fieldset.<name>` readable in kernels."""
    fs = _fs()
    fs.add_context("fix_lon", -0.5)
    fs.add_context("func", lambda x: 2 * x)
    assert fs.fix_lon == -0.5 and fs.func(3) == 6
    with pytest.raises(AttributeError, match="FieldSet has no attribute 'nope'"):
        fs.nope
    with pytest.raises(ValueError, match="already has a context"):
        fs.add_context("fix_lon", 1)
    with pytest.raises(ValueError, match="valid Python variable name"):
        fs.add_context("not a name", 1)


def test_pset_creation_like_the_reference():
    """reference tests/test_particleset.py:21-98 (create_lon_lat, create_empty, with_pids, customvars, custominit via attrgetter /
    on the pclass / overridden on the pset)."""
    from operator import attrgetter

    fs = _fs()
    npart = 100
    lon, lat = np.linspace(0, 1, npart, dtype=np.float32), np.linspace(1, 0, npart, dtype=np.float32)
    pset = pb.ParticleSet(fs, x=lon, y=lat, pclass=pb.Particle)
    assert np.allclose([p.x for p in pset], lon, rtol=1e-12) and np.allclose([p.y for p in pset], lat, rtol=1e-12)
    empty = pb.ParticleSet(fs, pclass=pb.Particle)
    empty.execute(pb.AdvectionRK4, endtime=1.0, dt=1.0)  # nothing to launch: no device needed
    assert empty.size == 0
    for offset in (0, 1, 200):
        ids = np.arange(offset, npart + offset)
        assert np.allclose([p.particle_id for p in pb.ParticleSet(fs, x=lon, y=lat, particle_ids=ids)], ids)
    two = pb.Particle.add_variable([pb.Variable("sample_var"), pb.Variable("sample_var2")])
    ps = pb.ParticleSet(fs, x=0, y=0, pclass=two, sample_var=5.0, sample_var2=10.0)
    assert [p.sample_var for p in ps] == [5.0] and [p.sample_var2 for p in ps] == [10.0]
    ps = pb.ParticleSet(fs, x=3, y=0, pclass=pb.Particle.add_variable(pb.Variable("sample_var", initial=attrgetter("x"))))
    assert np.allclose([p.sample_var for p in ps], 3.0)
    four = pb.Particle.add_variable(pb.Variable("sample_var", initial=4))
    assert [p.sample_var for p in pb.ParticleSet(fs, x=0, y=0, pclass=four)] == [4.0]
    assert [p.sample_var for p in pb.ParticleSet(fs, x=0, y=0, pclass=four, sample_var=5)] == [5.0]
    with pytest.raises(RuntimeError, match="Particle class does not have Variable nope"):
        pb.ParticleSet(fs, x=0, y=0, nope=3)
    # default z: the depth level closest to zero (reference :188-215)
    depths = np.concatenate([np.linspace(-9, -3, 3), np.linspace(2, 8, 3)])
    z6 = np.zeros((1, 6, 4, 5), np.float32)
    fsz = pb.FieldSet.from_arrays(lon=np.linspace(0, 1, 5), lat=np.linspace(0, 1, 4), depth=depths, U=z6, V=z6, mesh="flat")
    assert np.isclose(pb.ParticleSet(fsz, x=[0], y=[0]).z[0], 2.0)


def test_host_column_passes_match_numpy():
    """pb_host_fill_* / pb_host_min_max_f64 / pb_host_compact (multi-threaded host passes over particle columns; no device):
    the results NumPy gives for `a[:] = v`, `a.min()` / `a.max()` with NaN propagation and np.delete on every column."""
    import parcels_b200.particleset as P
    from parcels_b200.statuscodes import StatusCode

    rng = np.random.default_rng(0)
    n = (1 << 21) + 12345
    a = np.empty(n)
    P._fill(a, 600.0)
    assert a[0] == 600.0 and a[-1] == 600.0 and np.all(a == 600.0)
    s = np.empty(n, dtype=np.int32)
    P._fill(s, 10)
    assert np.all(s == 10)
    t = rng.uniform(-5.0, 7.0, n)
    assert P._min_or_max(t, True) == t.min() and P._min_or_max(t, False) == t.max()
    t[n // 3] = np.nan
    assert np.isnan(P._min_or_max(t, True)) and np.isnan(P._min_or_max(t, False))
    # compaction: every column of the SoA incl. the 2-D `ei` and an extra variable, order preserved
    d = {"x": rng.random(n, dtype=np.float32), "t": rng.random(n), "particle_id": np.arange(n, dtype=np.int64),
         "state": np.full(n, int(StatusCode.Evaluate), dtype=np.int32), "ei": rng.integers(0, 1000, (n, 2)).astype(np.int32),
         "age": rng.random(n).astype(np.float32)}  # fmt: skip
    dele = np.sort(rng.choice(n, 5000, replace=False))
    dele = np.concatenate([dele, [0, n - 1]])
    d["state"][dele] = int(StatusCode.Delete)
    want = {k: np.delete(v, np.where(d["state"] == int(StatusCode.Delete))[0], axis=0) for k, v in d.items()}
    ref = d
    removed = P._remove_deleted_host(d)
    assert removed == len(np.unique(dele)) and d is ref
    for k in want:
        assert d[k].shape == want[k].shape and np.array_equal(d[k], want[k]), k
    assert P._remove_deleted_host(d) == 0


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the driver's second arm: the oracle port of the reference path on the host cores, no GPU, no
    CUDA library): one JSON line with `impl`, the arm's own `cpu_baseline` and an `e2e` that repeats the value with zero copies."""
    import json
    import subprocess
    import sys

    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "c2_small", "--steps", "2",
                        "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)  # fmt: skip
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "particle-RK4-steps/sec" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"] and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["config"]["kernels"] == ["AdvectionRK4_3D", "DeleteParticle"]
