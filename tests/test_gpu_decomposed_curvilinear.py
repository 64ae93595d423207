"""GPU tests of mode D on CURVILINEAR grids (column slabs, DecomposedFieldSet.from_curvilinear): fixed-step EE / RK4 / RK4_3D and
AdvectionRK45 with CGrid_Velocity and curvilinear XLinear_Velocity equal the single-engine run BIT FOR BIT -- ids, x, y, z, t,
state, ei, and for RK45 dt and next_dt.  Three slab engines of one process linked by address (in-kernel migration,
scripts/decomposed_threads_check.py) and two gloo ranks sharing the GPU (collective transport, scripts/decomposed_check.py), on the
curvilinear cases of scripts/decomposed_kernels.py.  A halo too small for the step makes every rank raise."""

import os
import subprocess
import sys

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
    assert " 0 migrations" not in r.stdout  # particles crossed column-slab edges
    print(r.stdout[-1500:])  # (the per-rank grid and field bytes of the case)


# (kernel, interp, extra): the small config-3 mesh (spherical, float32 nodes) in 2-D and 3-D, the flat warped mesh, both
# interpolators, both directions, delayed releases ordered by id with the first shards' hints all zero, an overflowing inbox
THREADS = [("rk4", "curv_cgrid", []), ("rk4_3d", "curv_cgrid", ["--ordered-releases"]), ("ee", "curv_linear", ["--backward"]),
           ("rk4", "curv_cgrid", ["--mesh", "flat", "--backward"]), ("rk4_3d", "curv_linear", ["--mesh", "flat", "--inbox", "16"]),
           ("rk45", "curv_cgrid", ["--delayed"]), ("rk45", "curv_cgrid", ["--ordered-releases", "--backward"]),
           ("rk4", "curv_cgrid", ["--time-window", "3", "--nt", "6", "--runtime", "172800"]),
           ("rk45", "curv_cgrid", ["--time-window", "3", "--nt", "6", "--runtime", "172800"])]  # fmt: skip


@pytest.mark.parametrize("kernel,interp,extra", THREADS)
def test_in_kernel_migration_three_column_slabs(kernel, interp, extra):
    _passed(_threads("--kernel", kernel, "--interp", interp, *extra))


@pytest.mark.parametrize("kernel,interp,extra,port", [("rk4_3d", "curv_cgrid", ["--ordered-releases"], 29694),
                                                      ("rk45", "curv_cgrid", ["--delayed", "--backward"], 29695),
                                                      ("rk4", "curv_linear", ["--mesh", "flat"], 29696)])  # fmt: skip
def test_collective_transport_two_ranks(kernel, interp, extra, port):
    _passed(_gloo(port, "--kernel", kernel, "--interp", interp, *extra))


def test_halo_too_small_raises_on_every_rank():
    r = _gloo(29697, "--kernel", "rk4", "--interp", "curv_cgrid", "--dt", "86400")
    assert r.returncode != 0
    assert r.stdout.count("RuntimeError: halo violation") == 2, r.stdout[-3000:] + r.stderr[-3000:]


def test_every_rank_holds_the_single_engine_hash_table():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")]
    import decomposed_kernels as K
    import numpy as np

    import parcels_b200 as pb

    case = K.make_case("rk4", n=10, interp="curv_cgrid")
    f = case["f"]
    one = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], time=f["times"], U=f["U"], V=f["V"], mesh="spherical", **case["fs_kw"])
    ref = one.engine(0).hash_table()
    for r in range(3):
        h = K.decomposed_fieldset(case, r, 3).engine.hash_table()
        assert all(np.array_equal(h[k], ref[k]) for k in ref), r
