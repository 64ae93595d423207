"""CPU (needs the reference's own Python package, oracle/ref_harness.py): ``parcels_b200.install()`` patches the reference's ``Kernel.execute`` so that an
unmodified reference script -- its own ``ParticleSet``, ``ParticleSet.execute``, kernel functions, exceptions -- runs its inner
loop on the engine.  The engine here is the host simulation of the kernel sources (oracle/hostsim); tests/install_run.py does the
same comparison on a real GPU when the reference travels there."""

import json
import os
import subprocess
import sys

import pytest

from oracle import ref_harness as rh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(not rh.reference_available(), reason="the reference's own Python package is not importable (PARCELS_REFERENCE_SRC)")


@pytest.fixture(scope="module")
def result():
    from oracle.hostsim import build as hb

    env = dict(os.environ, PB_LIB=hb.build(), PB_HOSTSIM_TEST="1", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "install_run.py")], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("INSTALL_RESULT ")][-1]
    return json.loads(line[len("INSTALL_RESULT "):])


def test_builtin_kernel_list_runs_on_the_engine_with_identical_data(result):
    r = result["builtins_flat"]
    assert r["patched"] and r["err"] == ["", ""] and r["n"][0] == r["n"][1] > 0
    assert all(r["same"].values()), r


def test_user_python_handler_in_the_list(result):
    r = result["user_handler"]
    assert r["err"] == ["", ""] and r["n"][0] == r["n"][1] > 0 and all(r["same"].values()), r


def test_errors_are_raised_as_the_references_own_classes(result):
    r = result["raises"]
    assert r["err"][0] == r["err"][1] == "parcels._core.statuscodes.FieldOutOfBoundError", r
    assert all(r["same"].values()), r


def test_config2_dtypes_take_the_specialised_kernel(result):
    r = result["c2_small"]
    assert r["variant"] == 2 and r["err"] == ["", ""] and all(r["same"].values()), r  # (afast.cu, schedule 2: advection only)


def test_output_intervals_of_the_references_outer_loop(result):
    r = result["output_intervals"]
    assert r["writes"][0] == r["writes"][1] >= 3 and r["rows_equal"] and all(r["same"].values()), r


def test_uninstall_restores_the_reference(result):
    assert result["uninstalled"]


def test_random_configurations_against_the_reference_itself():
    """140 random configurations -- mostly rectilinear (the generator of scripts/fuzz_hostsim.py: dtypes, meshes, 2-D / 3-D, five schemes, five
    interpolators, boundary releases, non-finite coordinates, releases outside the time interval, with and without an error handler)
    through the reference's own ParticleSet.execute, untouched and with install(): identical data, same exception classes
    (scripts/fuzz_install_vs_reference.py) -- the engine against the REFERENCE, not against the oracle.  The reference's outputs on 140
    such configurations are stored too: tests/test_hostsim_cpu.py replays them where the reference is absent."""
    from oracle.hostsim import build as hb

    env = dict(os.environ, PB_LIB=hb.build(), PB_HOSTSIM_TEST="1", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "fuzz_install_vs_reference.py"), "140", "2026"], capture_output=True,
                         text=True, timeout=900, env=env, cwd=ROOT)  # fmt: skip
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-2000:]
    assert res.stdout.strip().endswith("140 cases (140 through the engine), 0 with differences"), res.stdout[-3000:]
