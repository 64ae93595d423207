"""What happens BETWEEN lanes of the device kernels: a particle's result must not depend on the lane, warp or block it runs in.

The host simulation of the kernel sources (oracle/hostsim) runs one thread at a time, every thread lane 0 of its own warp and
block: per-lane shared-memory columns collapse into one, cp.async is a plain copy and __shfl_xor_sync a stand-in.  So a wrong
lane stride, two lanes sharing a column, a dropped shuffle step of a warp-reduced launch report or of the batch-level lenT /
lenZ pre-pass all pass it.  This file checks those on the device:

1. lane-order invariance at multi-block scale: the same set of particles (same ids, so the same Philox increments) in storage
   order, reversed and randomly permuted -- every column bit-identical per id, every launch report equal -- for every
   particle kernel family, plus a stratified subset (storage positions 0, 31, 32, B - 1, B, 3 B - 1, 3 B and N - 1 of both
   orders; B = the launch block) against the oracle -- within the trigonometry's tolerance against NumPy's sin / cos, and bit
   for bit against the oracle evaluating the device's own (tests/device_trig.py);
2. lane placement of the rare path: one particle that takes the side path (fast flow, released outside the domain, NaN,
   released later) in a set that never does -- and one hit-path particle among missing lanes -- at lanes 0, 1 and 31 of a
   warp, in the first and last warp of a block and in the first and last block: bit-identical wherever it sits, its
   neighbours unchanged, and equal to the oracle (bit for bit in engine arithmetic);
3. warp-reduced reports against a recount from the returned arrays (the headline RK4 kernel and AdvectionDiffusionM1);
4. the batch flags (`any(tau > 0)`, `any(zeta > 0)`) of pb_sample_velocity / pb_sample_scalar when the one sample that sets
   them sits at a lane / warp / block boundary of the pre-pass.

Block sizes come from the library (Engine.debug_launch_block), not from an assumption.  Under the host simulation
(PB_HOSTSIM_TEST=1) the sets are a few thousand particles instead of 2e5: a logic check only.
"""

import os
import zlib

import numpy as np
import pytest

import cases
import parcels_b200 as pb
from device_trig import DeviceTrig
from engine_run import ulp_diff_f32
from oracle import parcels_oracle as po
from oracle import trig
from philox_ref import device_normals

pytestmark = pytest.mark.gpu

HOSTSIM = os.environ.get("PB_HOSTSIM_TEST") == "1"
N_BIG = 3001 if HOSTSIM else 200_003  # odd: a partial last warp and block
SEED = 4321
KEYS = ("particle_id", "state", "t", "ei", "x", "y", "z", "dx", "dy", "dz", "dt", "next_dt")
REPORT_KEYS = ("particle_steps", "n_error", "n_deleted", "first_error_iter", "n_out_of_time", "max_state", "max_iters_done",
               "cache_refills")  # fmt: skip
CURV_ULP = 8  # tests/test_gpu_parity.py: curvilinear positions against the oracle
NEXT_DT = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0))


@pytest.fixture(scope="module")
def blocks():
    from parcels_b200.engine import Engine

    eng = Engine(0)
    return {f: eng.debug_launch_block(f) for f in Engine.LAUNCH_FAMILIES}


# ------------------------------------------------------------------------------------------------
# configurations: a tests/cases.py case at N particles, made to diverge
# ------------------------------------------------------------------------------------------------
def _diverge(c, rng, n, sign=1.0):
    """Particles for case `c`: n of them, a slow half of the domain (cell changes every few steps on one side, never on the
    other), 3 % released outside the domain, a few NaN releases, a third released one to three steps later."""
    lon, lat = np.asarray(c["lon"], dtype=np.float64), np.asarray(c["lat"], dtype=np.float64)
    curv = lon.ndim == 2
    if curv:
        x, y = cases.points_in_mesh(rng, lon, lat, n)
        ny, nx = lon.shape
        slow = np.zeros((ny, nx), dtype=bool)
        slow[:, : nx // 2] = True
    else:
        lx, ly = lon[-1] - lon[0], lat[-1] - lat[0]
        x = rng.uniform(lon[0] - 0.03 * lx, lon[-1] + 0.03 * lx, n)
        y = rng.uniform(lat[0] + 0.02 * ly, lat[-1] - 0.02 * ly, n)
        slow = np.zeros((len(lat), len(lon)), dtype=bool)
        slow[:, : len(lon) // 2] = True
    for k in ("U", "V", "W"):
        if c.get(k) is not None:
            a = np.array(c[k])
            a[..., slow] *= a.dtype.type(0.02)
            c[k] = a
    if curv:
        out = rng.random(n) < 0.03
        x[out] = lon.max() + 0.05 * (lon.max() - lon.min())
    if c["depth"] is not None and len(c["depth"]) > 1:
        d = np.asarray(c["depth"], dtype=np.float64)
        z = rng.uniform(d[0] + 0.01 * (d[-1] - d[0]), d[-1] - 0.01 * (d[-1] - d[0]), n)
    else:
        z = np.zeros(n)
    x[rng.random(n) < 0.002] = np.nan
    t0 = float(np.asarray(c["t"])[0])
    t = np.full(n, t0)
    late = rng.random(n) < 0.3
    t[late] = t0 + sign * abs(c["dt"]) * rng.integers(1, 4, late.sum())
    c.update(x=x, y=y, z=z, t=t)
    return c


def _config(name):
    """name -> (case dict at N_BIG particles, kernel family, environment / FieldSet options, oracle tolerance in float32 ulp
    (0: bit-exact; None: invariance only))."""
    env = {}
    kind, _, variant = name.partition(":")
    if kind == "afast":
        sched, diff, mesh = variant.split("-")
        spec = dict(cases.CASES["c2_small"], mesh=mesh, umax=8.0 if mesh == "flat" else 12.0, segments=[dict(runtime=2400.0)])
        if diff == "kh":
            spec.update(kernels=["AdvectionRK4_3D", "DiffusionUniformKh"], kh=(40.0, 25.0) if mesh == "flat" else (100.0, 50.0))
        env = {"PB_DISABLE_FAST_KERNEL": "0", "PB_FAST_KERNEL": sched[-1]}
        tol = 0 if mesh == "flat" else 2
    elif kind == "agrid":  # the generic A-grid kernel: coordinate / data dtypes
        cd, dd = variant.split("-")
        spec = dict(cases.CASES["flat_f32c_f64d"], cdtype=cd, ddtype=dd, umax=6.0, segments=[dict(runtime=60.0), dict(runtime=50.0)])
        env = {"PB_DISABLE_FAST_KERNEL": "1"}
        tol = 0
    elif kind == "slip":
        base = {"freeslip": "freeslip_3d", "partialslip": "partialslip_sph", "nearest": "nearest_3d"}[variant]
        spec = dict(cases.CASES[base])
        spec["segments"] = [dict(runtime=4 * abs(spec["dt"]))]
        tol = 0 if spec["mesh"] == "flat" else 2
    elif kind == "cgrid":
        spec = dict(cases.CASES["cgrid_rect_3d"], segments=[dict(runtime=200.0)])
        tol = 0
    elif kind == "curv":
        base = {"cgrid-flat": "curv_flat_2d", "cgrid-sph": "curv_sph_2d", "agrid-flat": "curv_lin_flat_2d"}[variant]
        spec = dict(cases.CASES[base])
        spec["segments"] = [dict(runtime=4 * abs(spec["dt"]))]
        tol = CURV_ULP
    elif kind == "window":
        spec = dict(cases.CASES["c2_small"], nt=4, tstep=1800.0, umax=12.0, segments=[dict(runtime=3000.0), dict(runtime=2400.0)])
        env = {"time_window": 2}
        tol = 2
    elif kind == "rk45":
        spec = dict(cases.CASES["flat_f32c_f64d"], kernels=["AdvectionRK45"], umax=6.0, segments=[dict(runtime=100.0)])
        tol = None  # (against the oracle and the reference: tests/test_gpu_rk45.py)
    elif kind == "advdiff":
        spec = dict(cases.CASES["flat_f32c_f64d"], kernels=[variant], umax=6.0, segments=[dict(runtime=80.0)])
        tol = None  # (against the oracle fed the same normals: tests/test_gpu_advdiff.py)
    else:
        raise KeyError(name)
    spec["n"] = 8
    c = cases.build(spec)
    if kind in ("rk45", "advdiff"):
        c["W"] = None
    c = _diverge(c, np.random.default_rng(zlib.crc32(name.encode())), N_BIG, sign=np.sign(c["dt"]))
    return c, kind, env, tol


CONFIGS = ["afast:s1-adv-flat", "afast:s2-adv-flat", "afast:s2-adv-spherical", "afast:s1-kh-flat", "afast:s2-kh-flat",
           "agrid:f4-f4", "agrid:f4-f8", "agrid:f8-f8", "slip:freeslip", "slip:partialslip", "slip:nearest", "cgrid:rect",
           "curv:cgrid-flat", "curv:cgrid-sph", "curv:agrid-flat", "rk45:flat", "advdiff:AdvectionDiffusionM1",
           "advdiff:AdvectionDiffusionEM", "window:c2"]  # fmt: skip


def _fieldset(c, kind, env):
    fs = pb.FieldSet.from_arrays(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"], W=c["W"],
                                 mesh=c["mesh"], interp_method=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")),
                                 **({"time_window": env["time_window"]} if "time_window" in env else {}))  # fmt: skip
    for k, v in (c["constants"] or {}).items():
        fs.add_constant_field(k, v, mesh=c["mesh"])
    if kind == "rk45":
        fs.add_context("RK45_tol", 1e-4)
        fs.add_context("RK45_min_dt", 0.5)
        fs.add_context("RK45_max_dt", 4 * abs(c["dt"]))
    if kind == "advdiff":
        from oracle.make_golden import advdiff_inputs

        kz, km, dres = advdiff_inputs(c, "f8", True)
        fs.add_field("Kh_zonal", kz)
        fs.add_field("Kh_meridional", km)
        fs.add_context("dres", dres)
    return fs


def _run(c, kind, env, order, ids=None, fs=None):
    """Run the particles `order` (storage order = that index array; ids = order unless given).  Returns (columns sorted by
    particle id, error class name or '', one report per execute call)."""
    kenv = {k: v for k, v in env.items() if k.startswith("PB_")}
    os.environ.update(kenv)
    try:
        fs = fs or _fieldset(c, kind, env)
        pclass = NEXT_DT if kind == "rk45" else pb.Particle
        ps = pb.ParticleSet(fs, pclass=pclass, x=c["x"][order], y=c["y"][order], z=c["z"][order], t=c["t"][order],
                            particle_ids=order if ids is None else ids, seed=SEED)  # fmt: skip
        kern = [getattr(pb, k) for k in c["kernels"]]
        if c["delete_on_error"]:
            kern.append(pb.DeleteParticle)
        err, reps = "", []
        try:
            for seg in c["segments"]:
                ps.execute(kern, dt=c["dt"], **seg)
                reps.append(dict(ps.last_report))
        except RuntimeError as e:
            if type(e).__module__.startswith("parcels_b200._lib"):
                raise
            err = type(e).__name__
            reps.append(dict(ps.last_report))
        d = ps._data
        o = np.argsort(np.asarray(d["particle_id"]), kind="stable")
        return {k: np.ascontiguousarray(np.asarray(d[k])[o]) for k in KEYS if k in d}, err, reps
    finally:
        for k in kenv:
            os.environ.pop(k, None)


def _assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert a[k].shape == b[k].shape, f"{what}: {k}: {a[k].shape} vs {b[k].shape} particles"
        if a[k].size == 0:
            continue
        bad = np.flatnonzero((a[k].view(np.uint8).reshape(len(a[k]), -1) != b[k].view(np.uint8).reshape(len(b[k]), -1)).any(axis=1))
        assert bad.size == 0, (f"{what}: {k} differs for {bad.size} particles, ids {a['particle_id'][bad[:8]]}: "
                               f"{a[k][bad[:4]]} vs {b[k][bad[:4]]}")  # fmt: skip


def _oracle(c, ids):
    """The oracle on the particles `ids` only (their own ids: the engine's Philox increments for DiffusionUniformKh)."""
    pad = c.get("padding", ("low", "low", "high"))
    g = po.OGrid(c["lon"], c["lat"], c["depth"], mesh=c["mesh"], offsets=tuple(int(p == "low") for p in pad))
    ofs = po.OFieldSet(g, c["U"], c["V"], c["W"], time=c["times"], constants=c["constants"], interp=c.get("interp", "linear"))
    pd = po.create_particle_data(c["x"][ids], c["y"][ids], c["z"][ids], c["t"][ids], ngrids=ofs.ngrids, particle_ids=ids)
    state = {"call": 0, "it": 0}

    def normal(view):
        zx, zy = device_normals(SEED, state["call"], state["it"], view.particle_id)
        state["it"] += 1
        return zx, zy

    kern = [po.DiffusionUniformKh(normal) if k == "DiffusionUniformKh" else getattr(po, k) for k in c["kernels"]]
    if c["delete_on_error"]:
        kern.append(po.DeleteOnError)
    err = None
    try:
        for seg in c["segments"]:
            state["call"] += 1
            state["it"] = 0
            po.pset_execute(pd, ofs, kern, c["dt"], **seg)
    except po.OracleParticleError as e:
        err = e.code
    return pd, err


def _assert_oracle(c, got, ids, tol, what):
    """Against the oracle with NumPy's trigonometry within `tol`; where tol > 0 (spherical or curvilinear), also against the
    oracle in engine arithmetic (the device's own sin / cos, tests/device_trig.py) bit for bit."""
    if tol:
        with trig.use(DeviceTrig()):
            _assert_oracle_within(c, got, ids, 0, what + " (engine arithmetic)")
    return _assert_oracle_within(c, got, ids, tol, what)


def _assert_oracle_within(c, got, ids, tol, what):
    pd, oerr = _oracle(c, ids)
    sel = np.isin(got["particle_id"], ids)
    mine = {k: v[sel] for k, v in got.items()}
    o = np.argsort(pd["particle_id"], kind="stable")
    np.testing.assert_array_equal(mine["particle_id"], pd["particle_id"][o], err_msg=f"{what}: surviving ids")
    for k in ("state", "t", "ei"):
        np.testing.assert_array_equal(mine[k], pd[k][o], err_msg=f"{what}: {k}")
    for k in "xyz":
        if tol == 0:
            np.testing.assert_array_equal(mine[k], pd[k][o], err_msg=f"{what}: {k}")
        else:
            floor = 0.01 * float(np.nanmax(np.abs(np.asarray(c[k], dtype=np.float64)))) if tol == CURV_ULP else None
            u = ulp_diff_f32(mine[k], pd[k][o], floor=floor)
            fin = np.isfinite(pd[k][o])
            np.testing.assert_array_equal(np.isfinite(mine[k]), fin, err_msg=f"{what}: {k} finite")
            assert u[fin].max(initial=0) <= tol, f"{what}: {k} {u[fin].max()} float32 ulp from the oracle"
    return oerr, len(ids)


def _family(kind, env, c):
    if kind == "afast":
        return "agrid_fast"
    if kind == "curv":
        return "curv_agrid" if c.get("interp", "linear") == "linear" else "cgrid"
    if kind == "cgrid":
        return "cgrid"
    return "agrid"


def _stratified(n, block):
    pos = np.array([0, 31, 32, block - 1, block, 3 * block - 1, 3 * block, n - 1])
    return pos[(pos >= 0) & (pos < n)]


# ------------------------------------------------------------------------------------------------
# 1. lane-order invariance
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CONFIGS)
def test_result_does_not_depend_on_the_lane_a_particle_runs_in(name, blocks):
    c, kind, env, tol = _config(name)
    n = len(c["x"])
    ident = np.arange(n)
    perm = np.random.default_rng(7).permutation(n)
    rev = ident[::-1].copy()
    fs = _fieldset(c, kind, env)
    a, ea, ra = _run(c, kind, env, ident, fs=fs)
    assert 0 < len(a["particle_id"]) < n or kind in ("rk45",), f"{name}: the set must lose some particles and keep most"
    for what, order in (("permuted", perm), ("reversed", rev)):
        b, eb, rb = _run(c, kind, env, order, fs=_fieldset(c, kind, env) if "time_window" in env else fs)
        assert ea == eb, (what, ea, eb)
        _assert_same(a, b, f"{name}, {what} storage order")
        for x_, y_ in zip(ra, rb, strict=True):
            for k in REPORT_KEYS:
                assert x_[k] == y_[k], f"{name}, {what} storage order: report {k} {x_[k]} vs {y_[k]}"
    if kind == "afast":
        assert all(r["kernel_variant"] == int(env["PB_FAST_KERNEL"]) for r in ra), "the specialised kernel did not run"
    assert ra[-1]["particle_steps"] > 0
    if tol is None:
        return
    block = blocks[_family(kind, env, c)]
    pos = _stratified(n, block)
    ids = np.unique(np.concatenate([ident[pos], perm[pos], rev[pos]]))
    _assert_oracle(c, a, ids, tol, f"{name} vs the oracle")


# ------------------------------------------------------------------------------------------------
# 2. lane placement of the rare path
# ------------------------------------------------------------------------------------------------
def _placement_set(kind_name, block):
    """A set in which no particle takes the side path after its first evaluation (slow field, inside the domain, one release
    time) -- or, for 'hit', where every particle crosses cells all the time -- and the odd particles to put into it."""
    if kind_name == "curv":
        spec = dict(cases.CASES["curv_flat_2d"], n=8, segments=[dict(runtime=360.0)])
    else:
        spec = dict(cases.CASES["c2_small"], mesh="flat", umax=8.0, n=8, segments=[dict(runtime=2400.0)])
    c = cases.build(spec)
    lon, lat = np.asarray(c["lon"], dtype=np.float64), np.asarray(c["lat"], dtype=np.float64)
    n = 8 * block + 37
    rng = np.random.default_rng(3)
    for k in ("U", "V", "W"):  # the left half of the domain (columns): slow; the right half: fast
        if c.get(k) is not None:
            a = np.array(c[k])
            a[..., : a.shape[-1] // 2] *= a.dtype.type(0.002)
            a[..., a.shape[-1] // 2 :] *= a.dtype.type(3.0)
            c[k] = a
    if lon.ndim == 2:
        ny, nx = lon.shape
        jj, ii = rng.uniform(3, ny - 4, n + 2), rng.uniform(3, nx // 2 - 4, n + 2)
        fast_ii = rng.uniform(nx // 2 + 3, nx - 4, n + 2)

        def at(j, i):
            j0, i0 = int(j), int(i)
            fj, fi = j - j0, i - i0
            return [((1 - fj) * (1 - fi) * a[j0, i0] + (1 - fj) * fi * a[j0, i0 + 1] + fj * fi * a[j0 + 1, i0 + 1] + fj * (1 - fi) * a[j0 + 1, i0])
                    for a in (lon, lat)]  # fmt: skip

        slow_xy = np.array([at(j, i) for j, i in zip(jj, ii)])
        fast_xy = np.array([at(j, i) for j, i in zip(jj, fast_ii)])
        outside = (float(lon.max()) + 0.1 * float(np.ptp(lon)), float(lat.mean()))
    else:
        lx, ly = lon[-1] - lon[0], lat[-1] - lat[0]
        sy = rng.uniform(lat[0] + 0.2 * ly, lat[-1] - 0.2 * ly, n + 2)
        slow_xy = np.stack([rng.uniform(lon[0] + 0.1 * lx, lon[0] + 0.4 * lx, n + 2), sy], axis=1)
        fast_xy = np.stack([rng.uniform(lon[0] + 0.6 * lx, lon[0] + 0.9 * lx, n + 2), sy], axis=1)
        outside = (float(lon[-1] + 0.05 * lx), float(lat.mean()))
    if c["depth"] is not None and len(c["depth"]) > 1:
        d = np.asarray(c["depth"], dtype=np.float64)
        z = rng.uniform(d[0] + 0.3 * (d[-1] - d[0]), d[-1] - 0.3 * (d[-1] - d[0]), n + 2)
    else:
        z = np.zeros(n + 2)
    t0 = float(np.asarray(c["t"])[0])
    return c, n, slow_xy, fast_xy, z, outside, t0


ODD = ["fast", "leaves", "nan", "late", "hit"]


@pytest.mark.parametrize("kernel", ["afast:1", "afast:2", "curv"])
def test_the_odd_particle_of_a_warp_is_the_same_wherever_it_sits(kernel, blocks):
    kname, _, sched = kernel.partition(":")
    env = {"PB_DISABLE_FAST_KERNEL": "0", "PB_FAST_KERNEL": sched} if kname == "afast" else {}
    block = blocks["agrid_fast" if kname == "afast" else "cgrid"]
    c, n, slow_xy, fast_xy, z, outside, t0 = _placement_set(kname, block)
    nb = (n + block - 1) // block
    positions = sorted({0, 1, 31, block - 32, block - 1, block + 33, (nb - 1) * block, n - 1})
    dt = c["dt"]
    ODD_ID = 10 * n
    fs = _fieldset(c, "afast" if kname == "afast" else "curv", env)
    for odd in ODD:
        base_xy = fast_xy if odd == "hit" else slow_xy
        x, y, t = base_xy[:n, 0].copy(), base_xy[:n, 1].copy(), np.full(n, t0)
        ox, oy, ot = {"fast": (fast_xy[n, 0], fast_xy[n, 1], t0), "leaves": (outside[0], outside[1], t0),
                      "nan": (np.nan, slow_xy[n, 1], t0), "late": (slow_xy[n, 0], slow_xy[n, 1], t0 + 2 * dt),
                      "hit": (slow_xy[n, 0], slow_xy[n, 1], t0)}[odd]  # fmt: skip
        base = dict(c, x=x, y=y, z=z[:n].copy(), t=t)
        ref, err0, rep0 = _run(base, kname, env, np.arange(n), fs=fs)
        assert err0 == ""
        first = None
        for p in positions:
            cc = dict(base, x=np.insert(x, p, ox), y=np.insert(y, p, oy), z=np.insert(base["z"], p, z[n]), t=np.insert(t, p, ot))
            ids = np.insert(np.arange(n), p, ODD_ID)
            got, err, rep = _run(cc, kname, env, np.arange(n + 1), ids=ids, fs=fs)
            assert err == "", (odd, p, err)
            what = f"{kernel}: odd particle '{odd}' at storage position {p} (lane {p % 32}, warp {p % block // 32}, block {p // block})"
            odd_sel = got["particle_id"] == ODD_ID
            rest = {k: v[~odd_sel] for k, v in got.items()}
            _assert_same(rest, ref, what + ": its neighbours")
            mine = {k: v[odd_sel] for k, v in got.items()}
            if first is None:
                first = mine
                # the oracle: the odd particle with two neighbours (>= 2 rows, waiver 8)
                nbr = [0, n - 1]
                oc = dict(base, x=np.append(x[nbr], ox), y=np.append(y[nbr], oy), z=np.append(base["z"][nbr], z[n]),
                          t=np.append(t[nbr], ot))  # fmt: skip
                oids = np.array([0, n - 1, ODD_ID])
                sub = {k: np.concatenate([ref[k][np.isin(ref["particle_id"], oids[:2])], mine[k]]) for k in mine}
                _assert_oracle_ids(oc, sub, oids, 0 if c["mesh"] == "flat" and kname == "afast" else CURV_ULP, what + " vs the oracle")
            else:
                _assert_same(mine, first, what)
            if odd in ("leaves", "nan"):
                assert not odd_sel.any(), what + ": deleted"


def _assert_oracle_ids(c, got, ids, tol, what):
    """_assert_oracle for a set whose inputs are given in `c` in the order of `ids` (arbitrary ids)."""
    if tol:
        with trig.use(DeviceTrig()):
            _assert_oracle_ids_within(c, got, ids, 0, what + " (engine arithmetic)")
    _assert_oracle_ids_within(c, got, ids, tol, what)


def _assert_oracle_ids_within(c, got, ids, tol, what):
    pd, _ = _oracle_with_ids(c, ids)
    o = np.argsort(pd["particle_id"], kind="stable")
    g = np.argsort(got["particle_id"], kind="stable")
    mine = {k: v[g] for k, v in got.items()}
    np.testing.assert_array_equal(mine["particle_id"], pd["particle_id"][o], err_msg=f"{what}: surviving ids")
    for k in ("state", "t", "ei"):
        np.testing.assert_array_equal(mine[k], pd[k][o], err_msg=f"{what}: {k}")
    for k in "xyz":
        u = ulp_diff_f32(mine[k], pd[k][o], floor=0.01 * float(np.nanmax(np.abs(np.asarray(c["lon"], dtype=np.float64)))) if tol else None)
        assert u.max(initial=0) <= tol, f"{what}: {k} {u.max()} float32 ulp from the oracle"


def _oracle_with_ids(c, ids):
    pad = c.get("padding", ("low", "low", "high"))
    g = po.OGrid(c["lon"], c["lat"], c["depth"], mesh=c["mesh"], offsets=tuple(int(p == "low") for p in pad))
    ofs = po.OFieldSet(g, c["U"], c["V"], c["W"], time=c["times"], constants=c["constants"], interp=c.get("interp", "linear"))
    pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"], ngrids=ofs.ngrids, particle_ids=ids)
    kern = [getattr(po, k) for k in c["kernels"]] + ([po.DeleteOnError] if c["delete_on_error"] else [])
    err = None
    try:
        for seg in c["segments"]:
            po.pset_execute(pd, ofs, kern, c["dt"], **seg)
    except po.OracleParticleError as e:
        err = e.code
    return pd, err


# ------------------------------------------------------------------------------------------------
# 3. warp-reduced reports against a per-particle recount
# ------------------------------------------------------------------------------------------------
# kernel family -> (case, environment, end time): the headline RK4 kernel and AdvectionDiffusionM1 both warp-reduce their
# reports and take fixed steps, so the same recount holds
REPORT_KERNELS = {"afast": ("c2_small", {"PB_DISABLE_FAST_KERNEL": "0", "PB_FAST_KERNEL": "2"}, 2400.0),
                  "advdiff": ("flat_f32c_f64d", {}, 100.0)}  # fmt: skip


def _report_case(n, delete, rng, kind):
    base, _, endtime = REPORT_KERNELS[kind]
    spec = dict(cases.CASES[base], mesh="flat", umax=8.0, n=8, segments=[dict(endtime=endtime)], delete=delete)
    if kind == "advdiff":
        spec.update(kernels=["AdvectionDiffusionM1"], umax=6.0)
    c = cases.build(spec)
    if kind == "advdiff":
        c["W"] = None
    lon, lat = np.asarray(c["lon"]), np.asarray(c["lat"])
    lx, ly = lon[-1] - lon[0], lat[-1] - lat[0]
    d = np.asarray(c["depth"], dtype=np.float64)
    m = 0.01 if delete else 0.3  # with the delete handler some leave the domain; without it none does
    c["U"] = c["U"] * np.float32(1.0 if delete else 0.05)
    c["V"] = c["V"] * np.float32(1.0 if delete else 0.05)
    x = rng.uniform(lon[0] + m * lx, lon[-1] - m * lx, n)
    y = rng.uniform(lat[0] + m * ly, lat[-1] - m * ly, n)
    z = rng.uniform(d[0] + 0.3 * (d[-1] - d[0]), d[-1] - 0.3 * (d[-1] - d[0]), n)
    # every lane its own iteration count: releases at 0 .. 5 steps, and some after the end of the run (no step at all)
    t = c["dt"] * rng.integers(0, 6, n).astype(np.float64)
    t[rng.random(n) < 0.05] = 1.25 * endtime
    t[0] = 0.0
    c.update(x=x, y=y, z=z, t=t)
    return c


def _recount_steps(t0, t1, dt, endtime):
    """A lane's iterations of one execute call from its start and end times: the last step clamped to the end time, and a lane
    released exactly at the end time makes one step of length 0 (kernel.py:191-203); one released after it makes none."""
    t0 = np.asarray(t0, dtype=np.float64)
    steps = np.ceil((np.minimum(t1, endtime) - t0) / dt)
    return np.where(t0 > endtime, 0, np.where(t0 == endtime, 1, steps)).astype(np.int64)


@pytest.mark.parametrize("n", [1, 31, 33, "block-1", "block+1", "3block-1", "3block+1", "big"])
def test_warp_reduced_reports_equal_a_recount_from_the_arrays(n, blocks):
    block = blocks["agrid_fast"]
    n = {"block-1": block - 1, "block+1": block + 1, "3block-1": 3 * block - 1, "3block+1": 3 * block + 1,
         "big": 9_999 if HOSTSIM else 1_000_001}.get(n, n)  # fmt: skip
    for kind in REPORT_KERNELS:
        _check_reports(n, kind)


def _check_reports(n, kind):
    _, env, endtime = REPORT_KERNELS[kind]
    rng = np.random.default_rng(n)
    # (a) no errors: the steps of every lane
    c = _report_case(n, False, rng, kind)
    got, err, rep = _run(c, kind, env, np.arange(n))
    assert err == "" and len(got["particle_id"]) == n
    t_in = c["t"][got["particle_id"]]
    steps = _recount_steps(t_in, got["t"], c["dt"], endtime)
    assert np.all(got["t"][t_in <= endtime] == endtime)
    assert rep[0]["particle_steps"] == int(steps.sum()), (rep[0]["particle_steps"], int(steps.sum()))
    assert rep[0]["max_iters_done"] == int(steps.max())
    assert rep[0]["n_deleted"] == 0 and rep[0]["n_error"] == 0 and rep[0]["first_error_iter"] < 0 or rep[0]["n_error"] == 0
    assert rep[0]["max_state"] == int(got["state"].max())
    # (b) with the delete handler: what was deleted is what is missing
    c = _report_case(n, True, rng, kind)
    c["U"] = c["U"] * np.float32(4.0)
    got, err, rep = _run(c, kind, env, np.arange(n))
    assert err == ""
    gone = n - len(got["particle_id"])
    assert rep[0]["n_deleted"] == gone and rep[0]["n_error"] == 0
    assert rep[0]["max_state"] == max(int(got["state"].max(initial=0)), 30 if gone else 0)
    # (c) no handler: the run raises; the report counts the errored lanes and the first iteration any of them errored in
    c = _report_case(n, True, rng, kind)
    c["U"] = c["U"] * np.float32(4.0)
    c["delete_on_error"] = False
    got, err, rep = _run(c, kind, env, np.arange(n))
    assert err or n < 100, "the run was meant to raise"
    if err:
        errored = got["state"] >= 50
        assert rep[-1]["n_error"] >= 1 and rep[-1]["max_state"] == int(got["state"].max())
        it_err = np.round((got["t"][errored] - c["t"][got["particle_id"][errored]]) / c["dt"]).astype(np.int64)
        assert rep[-1]["first_error_iter"] == int(it_err.min()), (rep[-1]["first_error_iter"], int(it_err.min()))
    else:
        assert rep[-1]["n_error"] == 0


# ------------------------------------------------------------------------------------------------
# 4. batch flags across warp and block boundaries of the pre-pass
# ------------------------------------------------------------------------------------------------
def _flag_case(interp, blk):
    """A float32 grid (lenT decides float32 -> float64 promotion) or a slip interpolator with land next to the first depth
    level (lenZ decides where it looks for land), and a batch of samples spanning several pre-pass blocks."""
    if interp == "linear":
        c = cases.build(dict(seed=5, kind="smooth", cdtype="f4", ddtype="f4", mesh="flat", nx=20, ny=15, nz=4, nt=4, tstep=600.0,
                             n=8, kernels=["AdvectionRK4_3D"], dt=100.0, segments=[dict(runtime=100.0)], delete=True, margin=0.1))  # fmt: skip
    else:
        c = cases.build(dict(cases.CASES["freeslip_surface"], interp=interp, n=8, land=False))
        U, V = c["U"].copy(), c["V"].copy()
        U[:, 0, : U.shape[2] // 2, :] = 0
        V[:, 0, : U.shape[2] // 2, :] = 0
        c["U"], c["V"] = U, V
    n = 4 * blk + 77
    rng = np.random.default_rng(11)
    lon, lat = np.asarray(c["lon"], dtype=np.float64), np.asarray(c["lat"], dtype=np.float64)
    x = rng.uniform(lon[0], lon[-1], n).astype(np.float32)
    y = rng.uniform(lat[0], lat[-1], n).astype(np.float32)
    depth = np.asarray(c["depth"], dtype=np.float64)
    z = np.full(n, depth[0], dtype=np.float32)  # every sample on the first depth level (zeta == 0) ...
    t = np.zeros(n)  # ... and on the first time level (tau == 0)
    return c, x, y, z, t, depth


@pytest.mark.parametrize("flag, interp", [("t", "linear"), ("z", "freeslip"), ("z", "partialslip"),
                                          ("none", "linear"), ("none", "freeslip")])  # fmt: skip
def test_batch_flags_reach_every_sample_from_any_lane(flag, interp, blocks):
    from engine_run import make_fieldset
    from oracle_run import oracle_fieldset

    blk = blocks["sample_flags"]
    c, x, y, z, t, depth = _flag_case(interp, blk)
    n = len(x)
    fs, ofs = make_fieldset(c), oracle_fieldset(c)
    three_d = c["W"] is not None
    vec = fs.UVW if three_d else fs.UV
    P = (c["U"] + np.float32(0.25) * c["V"]).astype(c["U"].dtype)
    if interp == "linear":
        fs.add_field("P", P)
    promoted = []
    for p in ([None] if flag == "none" else [0, 31, 32, blk - 1, blk, n - 1]):
        tt, zz = t.copy(), z.copy()
        if flag == "t":
            tt[p] = 0.5 * float(c["times"][1])  # the one sample with tau > 0
        elif flag == "z":
            zz[p] = np.float32(0.5 * (depth[0] + depth[1]))  # the one sample with zeta > 0
        what = f"{interp}: flag {flag} set by sample {p} (lane {None if p is None else p % 32}, block {None if p is None else p // blk})"
        got = vec.eval(tt, zz, y, x)
        want = po.eval_uvw(ofs, tt, zz, y, x, None, three_d)
        for a, b in zip(got, want):
            np.testing.assert_array_equal(np.asarray(a), np.asarray(b, dtype=np.float64), err_msg=what)
        if interp == "linear":
            val = fs.P.eval(tt, zz, y, x)
            ref = po.eval_scalar(ofs, P, "linear", tt, zz, y, x, None)
            assert val.dtype == np.asarray(ref).dtype, f"{what}: scalar dtype {val.dtype} vs the oracle's {np.asarray(ref).dtype}"
            np.testing.assert_array_equal(val, ref, err_msg=what)
            promoted.append(val.dtype == np.float64)
        # ... and not a no-op: the first-level samples alone would be evaluated otherwise
        if p is not None and p != 0:
            rest = np.arange(n) != p
            alone = po.eval_uvw(ofs, tt[rest], zz[rest], y[rest], x[rest], None, three_d)
            assert any(np.any(np.asarray(a) != np.asarray(b)[rest]) for a, b in zip(alone, want)), what + ": the flag changes nothing"
    if interp == "linear":
        assert all(promoted) == (flag != "none") and any(promoted) == (flag != "none"), promoted
