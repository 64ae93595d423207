"""GPU test of time-slab streaming UNDER mode D (DESIGN.md 7b): 2 ranks on cuda:0, each with 2 of 6 time levels of its X-slab
resident, windows slid in lock-step -- bit-exact against the undecomposed run that keeps every level resident.  (The host
simulation runs it too, tests/test_hostsim_cpu.py; the file sorts last on purpose.)"""

import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WINDOWED = ["--same-gpu", "--particles", "6000", "--nt", "6", "--runtime", "345600", "--time-window", "2"]


def _run(extra, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "decomposed_check.py"), *WINDOWED, *extra]  # fmt: skip
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)


def test_windowed_slabs_collective_transport():
    r = _run(["--transport", "collective"], 29636)
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "time window 2 of 6" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


def test_windowed_slabs_in_kernel_migration_ipc():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("CUDA IPC needs a real device (thread ranks cover the loop under the host simulation)")
    r = _run(["--transport", "p2p", "--inbox", "256"], 29637)
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "peer memory" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout
