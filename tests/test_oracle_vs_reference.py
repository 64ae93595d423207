"""CPU test: the oracle restatement is bit-identical to the reference's own code.  The reference's outputs on these cases are
stored in tests/golden/ref_cases.npz (oracle/make_golden.py); where the reference tree is importable through
oracle/ref_harness.py, the live reference is run as well and must still produce exactly the stored outputs."""

import os

import numpy as np
import pytest

from oracle import ref_harness as rh
from oracle_run import load_case, run_oracle

COLUMNS = ("particle_id", "state", "ei", "t", "x", "y", "z")


def _live_reference(c):
    fs = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"],
                           W=c["W"], mesh=c["mesh"], constants=c["constants"])  # fmt: skip
    ps = rh.make_pset(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    k = rh.kernels()

    def DeleteParticle(particles, fieldset):
        particles[particles.state >= 50].state = 30

    kern = [getattr(k, kn) for kn in c["kernels"]] + ([DeleteParticle] if c["delete_on_error"] else [])
    if c["rng_seed"] is not None:
        np.random.seed(c["rng_seed"])
    try:
        for seg in c["segments"]:
            ps.execute(kern, dt=c["dt"], verbose_progress=False, **seg)
    except RuntimeError:
        pass
    return ps._data


@pytest.mark.parametrize("name", ["c2_small", "all_f32", "delayed_partial", "diffusion", "raise_oob"])
def test_live_reference_equals_oracle(name, golden_dir):
    c = load_case(name)
    with np.load(os.path.join(golden_dir, "ref_cases.npz")) as g:
        ref = {key: g[f"{name}/{key}"] for key in COLUMNS}
    if rh.reference_available():
        live = _live_reference(c)
        for key in COLUMNS:
            np.testing.assert_array_equal(live[key], ref[key], err_msg=f"live reference vs stored: {key}")
    pd, _ = run_oracle(c)
    for key in COLUMNS:
        np.testing.assert_array_equal(pd[key], ref[key], err_msg=key)
