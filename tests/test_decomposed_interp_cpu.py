"""CPU (host simulation of the kernel sources, oracle/hostsim): mode D on C-grids with CGrid_Velocity and on A-grids with XFreeslip /
XPartialslip / nearest-node sampling (land around the interior slab edges) reproduces the undecomposed run bit for bit -- the
peer-memory round loop on thread ranks (scripts/decomposed_threads_check.py) and the gloo collective transport of two ranks
(scripts/decomposed_check.py) -- and a halo too small for a fixed-step list raises on every rank instead of deleting particles."""

import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

needs_cxx = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no C++ compiler for the host simulation")


def _env():
    from oracle.hostsim import build as hb

    return dict(os.environ, PB_LIB=hb.build(), PB_HOSTSIM_TEST="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))


def _gloo(port, *extra):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--transport", "collective",
           "--particles", "300", "--halo", "1", *extra]  # fmt: skip
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())


@needs_cxx
@pytest.mark.parametrize("kernel,interp,extra", [("rk4_3d", "cgrid", ["--f32-coords", "--ordered-releases"]),
                                                 ("rk4", "freeslip", ["--mesh", "flat", "--backward"]),
                                                 ("rk4_3d", "nearest", ["--f32-coords"]),
                                                 ("rk45", "partialslip", ["--delayed"]),
                                                 ("m1", "cgrid", ["--inbox", "16"])])  # fmt: skip
def test_thread_ranks_in_kernel_migration(kernel, interp, extra):
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--kernel", kernel, "--interp", interp,
           "--particles", "300", "--halo", "1", *extra]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


@needs_cxx
def test_gloo_collective_transport_c_grid():
    r = _gloo(29681, "--kernel", "rk45", "--interp", "cgrid")
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


@needs_cxx
@pytest.mark.parametrize("interp,port", [("linear", 29682), ("cgrid", 29683)])
def test_fixed_step_halo_violation_raises_on_every_rank(interp, port):
    """Day-long RK4_3D steps at ~40 m/s leave a halo of one 3-degree cell: every rank raises, no particle is silently deleted."""
    r = _gloo(port, "--kernel", "rk4_3d", "--interp", interp, "--dt", "86400")
    assert r.returncode != 0
    assert r.stdout.count("RuntimeError: halo violation") == 2, r.stdout[-2000:] + r.stderr[-2000:]


def test_curvilinear_slabs_are_refused():
    from parcels_b200 import distributed as D

    lon, lat = np.meshgrid(np.linspace(-180, 180, 12), np.linspace(-80, 80, 6))
    U = np.zeros((1, 1, 6, 12), dtype=np.float32)
    with pytest.raises(NotImplementedError, match="curvilinear"):
        D.DecomposedFieldSet(lon=lon, lat=lat, U=U, V=U, interp_method="cgrid_velocity", rank=0, world=2)
