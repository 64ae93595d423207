"""Every template instantiation of the particle and sampling kernels on the device, bit for bit against the oracle in engine
arithmetic (the device's own sin / cos, tests/device_trig.py).

The kernels are templates over the coordinate dtype, the data dtype, a time axis, 2 or 3 components, the mesh, the interpolator,
fused diffusion and the Kh dtype / time axis of AdvectionDiffusionM1 / EM; nvcc compiles each combination on its own, and a
user's FieldSet picks one from its own dtypes.  tests/instantiations.py holds one key per combination the launchers can select,
each a small case of tests/cases.py run through the public API (ParticleSet.execute, column-slab engines, fs.UV / fs.UVW.eval,
Field.eval).  Trajectories compare particle_id, state, t, ei, x, y, z, dt (and next_dt for AdvectionRK45); samples compare the
value and its dtype.  The keys that run the per-lane shared-memory corner cache also run in reversed storage order, which must
give every particle the same bits.  tests/test_instantiations_cpu.py checks that the keys launch every exported instantiation.
"""

import numpy as np
import pytest

import instantiations as I

pytestmark = pytest.mark.gpu

TRAJ_KEYS = sorted(k for k, v in I.KEYS.items() if v["fam"] in ("advect", "rk45", "advdiff"))
SAMPLE_KEYS = sorted(k for k, v in I.KEYS.items() if v["fam"] in ("sample", "scalar"))


@pytest.mark.parametrize("name", TRAJ_KEYS)
def test_trajectories_equal_the_oracle(name):
    k = I.KEYS[name]
    c = I.build_case(k)
    n = len(c["x"])
    got, err = I.run_engine(c, k, np.arange(n))
    pd, oerr = I.run_oracle(c, k)
    assert (err != "") == (oerr is not None), (name, err, oerr)
    keys = I.TRAJ[1:] + (("next_dt",) if k["fam"] == "rk45" else ())
    I.assert_oracle(got, pd, keys, name)
    # (released outside the domain or NaN: deleted; AdvectionRK45 never errors.  The host simulation's sets are too small to say.)
    assert 0 < len(got["particle_id"]) and (len(got["particle_id"]) < n or k["fam"] == "rk45" or I.HOSTSIM), f"{name}: lost none"
    if I.uses_smem_cache(k) and not I.HOSTSIM:  # (the simulation runs every particle as lane 0 of its own block)
        rev, _ = I.run_engine(c, k, np.arange(n)[::-1].copy())
        I.assert_same(got, rev, f"{name}, reversed storage order")


@pytest.mark.parametrize("name", SAMPLE_KEYS)
def test_samples_equal_the_oracle(name):
    k = I.KEYS[name]
    c = I.build_case(k)
    t, z, y, x = I.samples(c)
    vals, ei, state = I.sample_engine(c, k, t, z, y, x)
    ovals, oei, ostate = I.sample_oracle(c, k, t, z, y, x)
    for i, (got, want) in enumerate(zip(vals, ovals, strict=True)):
        what = f"{name}, evaluation {i + 1}"
        assert len(got) == len(want), what
        for g, w in zip(got, want, strict=True):
            if k["fam"] == "scalar":  # (value_is_f32: the dtype NumPy's arithmetic gives; VectorField.eval returns float64)
                assert g.dtype == w.dtype, f"{what}: value dtype {g.dtype}, the oracle's {w.dtype}"
            np.testing.assert_array_equal(g, w, err_msg=what)
        assert any(np.any(g != 0) for g in got), f"{what}: every sample is 0"
    np.testing.assert_array_equal(ei, oei, err_msg=f"{name}: ei")
    np.testing.assert_array_equal(state, ostate, err_msg=f"{name}: state")
    assert np.any(state != 0) or I.HOSTSIM, f"{name}: no sample left the domain"
    if I.uses_smem_cache(k) and not I.HOSTSIM:
        r = slice(None, None, -1)
        rvals, rei, rstate = I.sample_engine(c, k, t[r], z[r], y[r], x[r])
        flat = lambda vs, ei, st: {**{f"{i}.{j}": a for i, v in enumerate(vs) for j, a in enumerate(v)}, "ei": ei, "state": st}  # noqa: E731
        rev = flat(rvals, rei, rstate)
        I.assert_same(flat(vals, ei, state), {key: v[r] for key, v in rev.items()}, f"{name}, reversed order")


@pytest.mark.parametrize("symbol, refusal, call", I.EXCLUDED)
def test_excluded_instantiations_are_refused(symbol, refusal, call):
    with pytest.raises(refusal):
        call()
