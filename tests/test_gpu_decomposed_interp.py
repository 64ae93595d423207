"""GPU tests of mode D (X-slab domain decomposition) on C-grids with CGrid_Velocity and on A-grids with XFreeslip, XPartialslip and
nearest-node sampling: fixed-step RK4 / RK4_3D, AdvectionRK45 and AdvectionDiffusionM1 / EM equal the single-engine run BIT FOR BIT
-- ids, x, y, z, t, state, ei, and for RK45 dt and next_dt.  The slip and nearest cases have land (U = V = W = 0) around the
interior slab edges.  Three slab engines of one process linked by address (in-kernel migration,
scripts/decomposed_threads_check.py) and two gloo ranks sharing the GPU (collective transport, scripts/decomposed_check.py), on the
cases of scripts/decomposed_kernels.py.  A halo too small for the step makes every rank raise, for fixed-step lists too."""

import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = "400"


def _threads(*extra):
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--particles", N, "--halo", "1", *extra]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)


def _gloo(port, *extra):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--transport", "collective",
           "--particles", N, "--halo", "1", *extra]  # fmt: skip
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)


def _passed(r):
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    assert " 0 migrations" not in r.stdout  # particles crossed slab edges


def _flags(mesh, direction, coords):
    return ["--mesh", mesh, *(["--backward"] if direction == "backward" else []), *(["--f32-coords"] if coords == "f32" else [])]


# (kernel, interp, mesh, direction, coordinate dtype): 2-D and 3-D on C-grids, every A-grid interpolator with land at the slab edges,
# both meshes, both directions, float32 and float64 coordinates
FIXED = [("rk4_3d", "cgrid", "spherical", "forward", "f64"), ("rk4", "cgrid", "flat", "backward", "f32"),
         ("rk4_3d", "freeslip", "spherical", "backward", "f32"), ("rk4", "partialslip", "flat", "forward", "f64"),
         ("rk4_3d", "nearest", "spherical", "forward", "f32"), ("rk4", "nearest", "flat", "backward", "f64")]  # fmt: skip


@pytest.mark.parametrize("kernel,interp,mesh,direction,coords", FIXED)
def test_fixed_step_in_kernel_migration_three_slabs(kernel, interp, mesh, direction, coords):
    _passed(_threads("--kernel", kernel, "--interp", interp, *_flags(mesh, direction, coords)))


def test_delayed_releases_on_a_float32_c_grid():
    """Releases in the order of the particle ids: the first shard holds only particles on the first time level, whose first
    evaluation is float64 in the single-engine batch only because other particles are not -- the bit comes from the whole set."""
    _passed(_threads("--kernel", "rk4_3d", "--interp", "cgrid", "--f32-coords", "--ordered-releases"))


@pytest.mark.parametrize("interp,mesh,direction,coords", [("cgrid", "spherical", "forward", "f32"), ("freeslip", "flat", "backward", "f64")])
def test_rk45_in_kernel_migration_three_slabs(interp, mesh, direction, coords):
    _passed(_threads("--kernel", "rk45", "--interp", interp, "--delayed", *_flags(mesh, direction, coords)))


@pytest.mark.parametrize("kernel,mesh,direction", [("m1", "spherical", "backward"), ("em", "flat", "forward")])
def test_advection_diffusion_on_c_grid_slabs(kernel, mesh, direction):
    _passed(_threads("--kernel", kernel, "--interp", "cgrid", "--delayed", *_flags(mesh, direction, "f64")))


@pytest.mark.parametrize("kernel,interp", [("rk4_3d", "cgrid"), ("rk45", "freeslip")])
def test_windowed_slabs_in_kernel_migration(kernel, interp):
    """3 of 6 time levels of each slab resident, windows slid in lock-step, delayed releases."""
    r = _threads("--kernel", kernel, "--interp", interp, "--nt", "6", "--runtime", "172800", "--time-window", "3")
    _passed(r)
    assert "time window 3 of 6" in r.stdout


def test_c_grid_full_inbox():
    """An inbox of 16 records makes most leavers wait for a later round."""
    _passed(_threads("--kernel", "rk4_3d", "--interp", "cgrid", "--inbox", "16", "--runtime", "172800"))


@pytest.mark.parametrize("kernel,interp,extra,port", [("rk45", "partialslip", [], 29672), ("em", "cgrid", ["--mesh", "flat", "--backward"], 29673)])
def test_collective_transport_two_ranks(kernel, interp, extra, port):
    _passed(_gloo(port, "--kernel", kernel, "--interp", interp, *extra))


def test_diffusion_uniform_kh_on_c_grid_slabs():
    """Fused DiffusionUniformKh on a C-grid at rest: Var = 2 K t, every particle accounted for once (3000 particles: the variance
    is held to 6 %)."""
    r = _gloo(29675, "--diffusion", "--interp", "cgrid", "--particles", "3000")
    assert r.returncode == 0 and "PASS statistics" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("kernel,interp,extra,port", [("rk4_3d", "linear", ["--dt", "86400"], 29676),
                                                      ("rk4_3d", "cgrid", ["--dt", "86400"], 29677),
                                                      ("rk45", "cgrid", ["--max-dt", "86400", "--rk45-tol", "1e7"], 29678)])  # fmt: skip
def test_halo_too_small_raises_on_every_rank(kernel, interp, extra, port):
    """A halo of one 3-degree cell cannot hold the stages of day-long RK4 steps at ~40 m/s (nor of RK45 steps that a loose tolerance
    lets grow towards a day): the lane stops with state 99 -- the DeleteParticle handler does not turn it into a deletion -- and
    every rank raises."""
    r = _gloo(port, "--kernel", kernel, "--interp", interp, *extra)
    assert r.returncode != 0
    assert r.stdout.count("RuntimeError: halo violation") == 2, r.stdout[-3000:] + r.stderr[-3000:]


def test_refusals():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]
    import decomposed_kernels

    import parcels_b200 as pb
    from parcels_b200 import distributed as D

    f = decomposed_kernels.make_case("rk4", n=10)["f"]
    lon2, lat2 = np.meshgrid(f["lon"], f["lat"])
    with pytest.raises(NotImplementedError, match="curvilinear"):
        D.DecomposedFieldSet(lon=lon2, lat=lat2, depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], interp_method="cgrid_velocity",
                             rank=0, world=2)  # fmt: skip
    case = decomposed_kernels.make_case("m1", n=10, interp="freeslip")
    dfs = decomposed_kernels.decomposed_fieldset(case, 0, 2)
    with pytest.raises(NotImplementedError, match="XLinear_Velocity or CGrid_Velocity"):
        D.decomposed_plan(dfs, case["kernels"], case["full"])
    case = decomposed_kernels.make_case("rk45", n=10, interp="nearest")
    dfs = decomposed_kernels.decomposed_fieldset(case, 0, 2)
    with pytest.raises(NotImplementedError, match="AdvectionRK45 is implemented for"):
        D.decomposed_plan(dfs, case["kernels"], case["full"])
    for interp in ("cgrid", "freeslip", "partialslip"):
        case = decomposed_kernels.make_case("rk45", n=10, interp=interp)
        plan = D.decomposed_plan(decomposed_kernels.decomposed_fieldset(case, 1, 2), case["kernels"], case["full"])
        assert plan.kind == "rk45" and plan.rk45 is not None
