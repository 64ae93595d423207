"""CPU (host simulation of the kernel sources, oracle/hostsim): AdvectionRK45 and AdvectionDiffusionM1 / EM under mode D reproduce
the undecomposed run bit for bit -- the peer-memory round loop on thread ranks (scripts/decomposed_threads_check.py) and the gloo
collective transport of two ranks (scripts/decomposed_check.py)."""

import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no C++ compiler for the host simulation")


def _env():
    from oracle.hostsim import build as hb

    return dict(os.environ, PB_LIB=hb.build(), PB_HOSTSIM_TEST="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))


@pytest.mark.parametrize("kernel,extra", [("rk45", ["--delayed"]), ("m1", ["--mesh", "flat", "--backward"]), ("em", ["--inbox", "16"])])
def test_thread_ranks_in_kernel_migration(kernel, extra):
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--kernel", kernel, "--particles", "300",
           "--halo", "1", *extra]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


@pytest.mark.parametrize("kernel,port", [("rk45", 29661), ("em", 29662)])
def test_gloo_collective_transport(kernel, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--transport", "collective",
           "--kernel", kernel, "--particles", "300", "--halo", "1"]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout
