"""CPU (no GPU needed): the keys of tests/instantiations.py launch every exported instantiation of the particle and sampling
kernels.  tests/test_gpu_instantiations.py runs on the host simulation of the kernel sources (oracle/hostsim) with its launch
trace on (PB_HOSTSIM_TRACE); the launched symbols, demangled, must cover every instantiation the library exports, apart from
the explicit exclusions of tests/instantiations.py.  Whoever adds a template instantiation has to add its key."""

import os
import re
import shutil
import subprocess
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = re.compile(r"^void (advect_kernel|rk45_kernel|advdiff_kernel|sample_kernel|sample_scalar_curv_kernel|classify_columns_kernel)<")

pytestmark = pytest.mark.skipif(any(shutil.which(t) is None for t in (os.environ.get("CXX", "g++"), "nm", "c++filt")),
                                reason="no C++ compiler or binutils for the host simulation")  # fmt: skip


def _demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {re.sub(r"\(.*$", "", s) for s in out if FAMILIES.match(s)}


def test_every_exported_instantiation_is_launched_or_excluded(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import instantiations as I
    from oracle.hostsim import build as hb

    lib = hb.build()
    nm = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    exported = _demangle([ln.split()[-1] for ln in nm.splitlines() if ln.strip()])
    assert len(exported) > 300, sorted(exported)[:10]
    trace = tmp_path / "launched.txt"
    env = dict(os.environ, PB_LIB=lib, PB_HOSTSIM_TEST="1", PB_HOSTSIM_TRACE=str(trace),
               PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))  # fmt: skip
    cmd = [sys.executable, "-m", "pytest", "tests/test_gpu_instantiations.py", "-m", "gpu", "-q", "-p", "no:cacheprovider"]
    # (the file also runs inside tests/test_hostsim_cpu.py's whole-suite run, whose limit it shares: a tight limit here shows growth)
    t0 = time.monotonic()
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=360)
    elapsed = time.monotonic() - t0
    assert res.returncode == 0, f"({elapsed:.0f} s on the simulation)\n" + res.stdout[-3000:] + res.stderr[-2000:]
    print(f"tests/test_gpu_instantiations.py: {elapsed:.0f} s on the simulation")
    launched = _demangle(sorted(set(trace.read_text().split())))
    excluded = {e[0] for e in I.EXCLUDED}
    stale = sorted(excluded - exported)
    assert not stale, f"the exclusion list names instantiations the library no longer exports: {stale}"
    missing = sorted(exported - launched - excluded)
    assert not missing, f"{len(missing)} exported instantiations no key of tests/instantiations.py launches:\n" + "\n".join(missing)
