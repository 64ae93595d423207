"""GPU tests of AdvectionRK45 and AdvectionDiffusionM1 / EM under mode D (X-slab domain decomposition): a lane that leaves its slab
stops mid-call and continues on its new owner with its dt, next_dt and iteration count, so the decomposed run equals the
single-engine run BIT FOR BIT -- ids, x, y, z, t, state, ei, and for RK45 dt and next_dt; M1 / EM draw the same Wiener increments.
Three slab engines of one process linked by address (in-kernel migration, scripts/decomposed_threads_check.py) and two gloo ranks
sharing the GPU (collective transport, scripts/decomposed_check.py), on the cases of scripts/decomposed_kernels.py."""

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


# (kernel, mesh, direction, delayed releases): every kernel on both meshes, both directions, with and without delayed releases
CASES = [("rk45", "spherical", "forward", True), ("rk45", "flat", "backward", False), ("m1", "spherical", "backward", True),
         ("m1", "flat", "forward", False), ("em", "spherical", "forward", False), ("em", "flat", "backward", True)]  # fmt: skip


@pytest.mark.parametrize("kernel,mesh,direction,delayed", CASES)
def test_in_kernel_migration_three_slabs(kernel, mesh, direction, delayed):
    r = _threads("--kernel", kernel, "--mesh", mesh, *(["--backward"] if direction == "backward" else []), *(["--delayed"] if delayed else []))
    _passed(r)


def test_m1_deletions_at_the_domain_edge_and_a_full_inbox():
    """M1 deletes the particles that leave the global domain; an inbox of 16 records makes most leavers wait for a later round."""
    r = _threads("--kernel", "m1", "--inbox", "16", "--runtime", "172800")
    _passed(r)
    left = int(r.stdout.split(" of ")[0].rsplit(" ", 1)[-1])
    assert left < int(N), r.stdout[-2000:]


@pytest.mark.parametrize("kernel", ["rk45", "em"])
def test_windowed_slabs_in_kernel_migration(kernel):
    """3 of 6 time levels of each slab resident (Kh of EM streams too; an RK45 step may straddle a level), windows slid in lock-step,
    delayed releases."""
    r = _threads("--kernel", kernel, "--nt", "6", "--runtime", "172800", "--time-window", "3")
    _passed(r)
    assert "time window 3 of 6" in r.stdout


@pytest.mark.parametrize("kernel,extra,port", [("rk45", [], 29651), ("m1", ["--mesh", "flat", "--backward", "--delayed"], 29652),
                                               ("em", ["--nt", "6", "--runtime", "172800", "--time-window", "3"], 29653)])  # fmt: skip
def test_collective_transport_two_ranks(kernel, extra, port):
    _passed(_gloo(port, "--kernel", kernel, *extra))


@pytest.mark.parametrize("kernel,extra,port", [("rk45", ["--max-dt", "86400", "--rk45-tol", "1e7"], 29654), ("m1", ["--dres", "20"], 29655)])
def test_halo_too_small_raises_on_every_rank(kernel, extra, port):
    """A halo of one cell cannot hold the stages of RK45 steps that a loose tolerance lets grow towards a day, nor a Kh sample 20
    degrees away: every rank raises."""
    r = _gloo(port, "--kernel", kernel, *extra)
    assert r.returncode != 0
    assert r.stdout.count("RuntimeError: halo violation") == 2, r.stdout[-3000:] + r.stderr[-3000:]


def test_refusals():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]
    import decomposed_kernels

    import parcels_b200 as pb
    from parcels_b200 import distributed as D

    case = decomposed_kernels.make_case("rk45", n=10)
    dfs = decomposed_kernels.decomposed_fieldset(case, 0, 2)
    with pytest.raises(NotImplementedError, match="DeleteParticle"):
        D.decomposed_plan(dfs, [pb.AdvectionRK45], case["full"])
    no_next_dt = {k: v for k, v in case["full"].items() if k != "next_dt"}
    with pytest.raises(ValueError, match="next_dt"):
        D.decomposed_plan(dfs, case["kernels"], no_next_dt)

    def user(particles, fieldset):
        pass

    with pytest.raises(NotImplementedError, match="one built-in kernel"):
        D.decomposed_plan(dfs, [pb.AdvectionRK45, user, pb.DeleteParticle], case["full"])
    plan = D.decomposed_plan(dfs, case["kernels"], case["full"])
    assert plan.kind == "rk45" and plan.rk45 is not None and plan.next_dt_dtype == np.float32
