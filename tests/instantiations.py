"""The dispatch keys of the particle and sampling kernels: one small case per template instantiation the launchers can select,
run through the public API and compared bit for bit with the oracle in engine arithmetic (tests/test_gpu_instantiations.py).

A key names what picks the instantiation: the launcher family, the coordinate dtype ``a``, the data dtype ``d``, a time axis
(``ht``: nt > 1), the number of velocity components (``nc``), the mesh, the interpolator, fused DiffusionUniformKh, and for
AdvectionDiffusionM1 / EM the Kh dtype and Kh time axis; the comments of ``_table`` name the launcher each group goes through.
tests/test_instantiations_cpu.py checks on the host simulation that the keys together launch every exported instantiation.
"""

from __future__ import annotations

import contextlib
import os
import sys
import zlib

import numpy as np

import cases
from device_trig import DeviceTrig
from oracle import parcels_oracle as po
from oracle import trig
from philox_ref import device_normals

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import thread_ranks  # noqa: E402  (scripts/: ranks as threads of one process)

HOSTSIM = os.environ.get("PB_HOSTSIM_TEST") == "1"
# an odd count over several blocks of every launcher (A-grid blocks of 128 / 256 lanes, curvilinear 128); a logic check only on
# the host simulation, which runs one thread at a time
N = 23 if HOSTSIM else 4001
SEED = 9876
DT = ("f4", "f8")
BOOL = (False, True)
TRAJ = ("particle_id", "state", "t", "ei", "x", "y", "z", "dt")


# ------------------------------------------------------------------------------------------------
# the key table
# ------------------------------------------------------------------------------------------------
def _k(fam, **kw):
    kw["fam"] = fam
    return kw


def _name(k):
    return "-".join(f"{v}" if not isinstance(v, bool) else (f"{key}" if v else f"no{key}") for key, v in k.items() if key != "fam")


def _table():
    keys = {}

    def add(fam, **kw):
        k = _k(fam, **kw)
        keys[f"{fam}:{_name({x: y for x, y in k.items() if x != 'fam'})}"] = k

    # the specialised A-grid RK4 kernel (afast.cu: float64 nodes, float32 data, a time axis), both schedules, fused diffusion
    for nc, hz in ((2, False), (2, True), (3, True)):
        for sched in (1, 2):
            for diff in BOOL:
                add("advect", path="afast", interp="linear", a="f8", d="f4", ht=True, nc=nc, hz=hz, sched=sched, diff=diff, mesh="flat")
    for a in DT:
        for d in DT:
            for ht in BOOL:
                for nc in (2, 3):
                    mesh = "spherical" if ht != (nc == 3) else "flat"
                    # launch_agrid (MODE 0), launch_agrid_alt (MODE 1: XFreeslip / XPartialslip, MODE 2: nearest node)
                    add("advect", path="agrid", interp="linear", a=a, d=d, ht=ht, nc=nc, mesh=mesh)
                    add("advect", path="agrid", interp="freeslip" if mesh == "flat" else "partialslip", a=a, d=d, ht=ht, nc=nc, mesh=mesh)
                    add("advect", path="agrid", interp="nearest", a=a, d=d, ht=ht, nc=nc, mesh="flat")
                    # launch_sample_agrid / launch_sample_agrid_alt: fs.UV / fs.UVW.eval
                    for interp in ("linear", "partialslip", "nearest"):
                        add("sample", path="agrid", interp=interp, a=a, d=d, ht=ht, nc=nc, mesh="flat" if interp == "nearest" else mesh)
                # launch_sample_scalar: Field.eval, every scalar interpolator
                for method in ("linear", "nearest", "cgrid_tracer", "linear_invdist_land"):
                    add("scalar", path="agrid", method=method, a=a, d=d, ht=ht, mesh="flat")
                # launch_rk45 (XLinear_Velocity), launch_rk45_slip (XFreeslip / XPartialslip)
                for interp in ("linear", "freeslip"):
                    add("rk45", path="agrid", interp=interp, a=a, d=d, ht=ht, mesh="flat")
            for nc in (2, 3):
                # launch_cgrid / launch_sample_cgrid on rectilinear grids
                add("advect", path="cgrid", interp="cgrid_velocity", a=a, d=d, ht=True, nc=nc, mesh="spherical" if nc == 2 else "flat")
                add("sample", path="cgrid", interp="cgrid_velocity", a=a, d=d, ht=True, nc=nc, mesh="flat")
                for sph in BOOL:
                    mesh = "spherical" if sph else "flat"
                    # launch_cgrid (curvilinear C-grid, with and without fused DiffusionUniformKh), launch_curv_agrid
                    for diff in BOOL:
                        add("advect", path="curv", interp="cgrid_velocity", a=a, d=d, nc=nc, mesh=mesh, diff=diff)
                        add("advect", path="columns", interp="cgrid_velocity", a=a, d=d, nc=nc, mesh=mesh, diff=diff)
                    add("advect", path="curv", interp="linear", a=a, d=d, nc=nc, mesh=mesh, diff=False)
                    add("advect", path="columns", interp="linear", a=a, d=d, nc=nc, mesh=mesh, diff=False)
                    # launch_sample_cgrid / launch_sample_curv_agrid on curvilinear grids
                    add("sample", path="curv", interp="cgrid_velocity", a=a, d=d, ht=True, nc=nc, mesh=mesh)
                    add("sample", path="curv", interp="linear", a=a, d=d, ht=True, nc=nc, mesh=mesh)
            # launch_rk45_cgrid: rectilinear and curvilinear (single engine and column slabs)
            add("rk45", path="cgrid", interp="cgrid_velocity", a=a, d=d, ht=True, mesh="flat")
            for sph in BOOL:
                mesh = "spherical" if sph else "flat"
                add("rk45", path="curv", interp="cgrid_velocity", a=a, d=d, mesh=mesh)
                add("rk45", path="columns", interp="cgrid_velocity", a=a, d=d, mesh=mesh)
                # launch_sample_scalar_curv
                for ht in BOOL:
                    add("scalar", path="curv", method="cgrid_tracer" if ht else "nearest", a=a, d=d, ht=ht, mesh=mesh)
            # launch_advdiff: Kh dtype, (U/V time, Kh time) of the A-grid, and the C-grid with and without a Kh time axis
            for dk in DT:
                for ht, kht in ((False, False), (True, False), (True, True)):
                    add("advdiff", path="agrid", interp="linear", a=a, d=d, dk=dk, ht=ht, kht=kht, mesh="spherical" if kht else "flat",
                        scheme="AdvectionDiffusionEM" if ht == kht else "AdvectionDiffusionM1")  # fmt: skip
                for kht in BOOL:
                    add("advdiff", path="cgrid", interp="cgrid_velocity", a=a, d=d, dk=dk, ht=True, kht=kht, mesh="flat",
                        scheme="AdvectionDiffusionM1" if kht else "AdvectionDiffusionEM")  # fmt: skip
    return keys


KEYS = _table()

# Exported instantiations that no public path can select: (demangled symbol, the refusal that makes it unreachable, a callable that
# must raise it).  Empty: every instantiation the launchers can select is reachable through the public API.
EXCLUDED = []

# the keys that run the per-lane shared-memory corner cache (PB_SMEM_CACHE): one reversed-storage-order run each
SMEM_PATHS = {("advect", "agrid"), ("advect", "afast"), ("rk45", "agrid"), ("advdiff", "agrid"), ("advdiff", "cgrid"), ("sample", "agrid"), ("scalar", "agrid")}


def uses_smem_cache(k):
    return (k["fam"], k["path"]) in SMEM_PATHS


# ------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------
def _rect_spec(k, kernels, nt):
    if k["mesh"] == "spherical":
        spec = dict(seed=61, kind="smooth", mesh="spherical", nx=21, ny=17, nz=5, tstep=3600.0, dt=600.0,
                    segments=[dict(runtime=2400.0)], margin=-0.02, umax=10.0)  # fmt: skip
    else:
        spec = dict(seed=62, kind="smooth", mesh="flat", nx=20, ny=17, nz=6, tstep=50.0, dt=10.0, segments=[dict(runtime=40.0)],
                    margin=-0.03, umax=6.0)  # fmt: skip
    spec.update(cdtype=k["a"], ddtype=k["d"], nt=nt, n=8, kernels=kernels, delete=True, interp=k.get("interp", "linear"),
                no_depth=not k.get("hz", True))  # fmt: skip
    if k.get("interp") in ("freeslip", "partialslip", "nearest") or k["fam"] == "scalar":
        spec["land"] = True
    if k.get("interp") == "nearest" or k["fam"] == "scalar":
        spec["umax"] = 3.0 / spec["dt"]  # nearest node converts no units: cells per step on a flat mesh
    return spec


def _curv_spec(k, kernels):
    nz = 6 if kernels[0].endswith("_3D") else 1
    if k["mesh"] == "spherical":
        spec = dict(seed=63, mesh="spherical", tstep=7200.0, dt=900.0, segments=[dict(runtime=2700.0)], umax=15.0)
    else:
        spec = dict(seed=64, mesh="flat", tstep=600.0, dt=60.0, segments=[dict(runtime=180.0)], umax=1.5)
    # (30 cell columns, cut at column 15 into column slabs; fewer rows on the simulation, whose spatial-hash build is slow)
    spec.update(kind="curv", interp=k.get("interp", "cgrid_velocity"), cdtype=k["a"], ddtype=k["d"], nx=31, ny=9 if HOSTSIM else 23, nz=nz, nt=3, n=8, kernels=kernels,
                delete=True)  # fmt: skip
    return spec


def build_case(k, n=N):
    """The case of key ``k``: tests/cases.py with overrides, n particles made to diverge (cell changes on one side of the domain
    only, some released outside it, a few NaN, a third released later)."""
    fam = k["fam"]
    nc = k.get("nc", 2)
    kernels = {"rk45": ["AdvectionRK45"], "advdiff": [k.get("scheme")]}.get(fam, ["AdvectionRK4_3D" if nc == 3 else "AdvectionRK4"])
    if k.get("diff"):
        kernels = kernels + ["DiffusionUniformKh"]
    curv = k["path"] in ("curv", "columns")
    nt = 3 if k.get("ht", True) else 1
    # (nearest node: the oracle samples W with the 2-D kernels too, so the 2-D keys keep the W of a 3-D case)
    spec = _curv_spec(k, kernels) if curv else _rect_spec(k, ["AdvectionRK4_3D"] if k.get("interp") == "nearest" else kernels, nt)
    c = cases.build(spec)
    c["kernels"] = kernels
    if fam in ("rk45", "advdiff"):
        c["W"] = None
    if k.get("diff"):
        c["constants"] = {"Kh_zonal": 100.0, "Kh_meridional": 50.0} if k["mesh"] == "spherical" else {"Kh_zonal": 0.5, "Kh_meridional": 0.25}
    rng = np.random.default_rng(zlib.crc32(repr(sorted(k.items())).encode()))
    return _diverge(c, rng, n, avoid=EDGE_COLUMNS if k["path"] == "columns" and k.get("diff") else None)


def _points_avoiding(rng, lon, lat, n, avoid):
    """cases.points_in_mesh without the cell columns [avoid[0], avoid[1])."""
    ny, nx = lon.shape
    gap = avoid[1] - avoid[0]
    jj = rng.uniform(0.5, ny - 1.5, n)
    ii = rng.uniform(0.5, nx - 1.5 - gap, n)
    ii = np.where(ii >= avoid[0], ii + gap, ii)
    j0, i0 = jj.astype(int), ii.astype(int)
    fj, fi = jj - j0, ii - i0
    return tuple((1 - fj) * (1 - fi) * a[j0, i0] + (1 - fj) * fi * a[j0, i0 + 1] + fj * fi * a[j0 + 1, i0 + 1] + fj * (1 - fi) * a[j0 + 1, i0]
                 for a in (lon, lat))  # fmt: skip


def _diverge(c, rng, n, avoid=None):
    lon, lat = np.asarray(c["lon"], dtype=np.float64), np.asarray(c["lat"], dtype=np.float64)
    curv = lon.ndim == 2
    if curv:
        x, y = cases.points_in_mesh(rng, lon, lat, n) if avoid is None else _points_avoiding(rng, lon, lat, n, avoid)
        slow = np.zeros(lon.shape, dtype=bool)
        slow[:, : lon.shape[1] // 2] = True
        x[rng.random(n) < 0.03] = lon.max() + 0.05 * (lon.max() - lon.min())
    else:
        lx, ly = lon[-1] - lon[0], lat[-1] - lat[0]
        x = rng.uniform(lon[0] - 0.03 * lx, lon[-1] + 0.03 * lx, n)
        y = rng.uniform(lat[0] + 0.02 * ly, lat[-1] - 0.02 * ly, n)
        slow = np.zeros((len(lat), len(lon)), dtype=bool)
        slow[:, : len(lon) // 2] = True
    for key in ("U", "V", "W"):
        if c.get(key) is not None:
            a = np.array(c[key])
            a[..., slow] *= a.dtype.type(0.02)
            c[key] = a
    if c["depth"] is not None and len(c["depth"]) > 1:
        d = np.asarray(c["depth"], dtype=np.float64)
        z = rng.uniform(d[0] + 0.01 * (d[-1] - d[0]), d[-1] - 0.01 * (d[-1] - d[0]), n)
    else:
        z = np.zeros(n)
    x[rng.random(n) < 0.01] = np.nan
    t = np.zeros(n)
    late = rng.random(n) < 0.3
    t[late] = abs(c["dt"]) * rng.integers(1, 3, late.sum())
    c.update(x=x, y=y, z=z, t=t)
    return c


def _kh(c, k):
    from oracle.make_golden import advdiff_inputs

    return advdiff_inputs(c, k["dk"], k["kht"])


def _rk45_context(c):
    return {"RK45_tol": 1e-2 if c["mesh"] == "flat" else 200.0, "RK45_min_dt": 0.5, "RK45_max_dt": 4 * abs(c["dt"])}


# ------------------------------------------------------------------------------------------------
# the engine: trajectories
# ------------------------------------------------------------------------------------------------
def _fieldset(c, k):
    import parcels_b200 as pb

    fs = pb.FieldSet.from_arrays(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"], W=c["W"],
                                 mesh=c["mesh"], interp_method=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")))  # fmt: skip
    _setup(fs, c, k)
    return fs


def _setup(fs, c, k):
    for name, v in (c["constants"] or {}).items():
        fs.add_constant_field(name, v, mesh=c["mesh"])
    if k["fam"] == "rk45":
        for name, v in _rk45_context(c).items():
            fs.add_context(name, v)
    if k["fam"] == "advdiff":
        kz, km, dres = _kh(c, k)
        fs.add_field("Kh_zonal", kz)
        fs.add_field("Kh_meridional", km)
        fs.add_context("dres", dres)


def _pclass(k):
    import parcels_b200 as pb

    return pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0)) if k["fam"] == "rk45" else pb.Particle


def _kernels(c, k, columns=False):
    import parcels_b200 as pb

    kern = [getattr(pb, name) for name in c["kernels"]]
    return kern + ([pb.DeleteParticle] if (c["delete_on_error"] and k["fam"] != "rk45") or columns else [])


def _env(k):
    if k["path"] == "afast":
        return {"PB_DISABLE_FAST_KERNEL": "0", "PB_FAST_KERNEL": str(k["sched"])}
    # the generic A-grid kernel: the specialised one (afast.cu) would take some of its keys otherwise
    return {"PB_DISABLE_FAST_KERNEL": "1"} if k["fam"] == "advect" and k["path"] == "agrid" else {}


def _sorted(d, keys):
    o = np.argsort(np.asarray(d["particle_id"]), kind="stable")
    return {key: np.ascontiguousarray(np.asarray(d[key])[o]) for key in keys if key in d}


def run_engine(c, k, order):
    """The particles in storage order ``order`` (ids = order) through ParticleSet.execute, or through column-slab engines for the
    column keys.  Returns the columns sorted by particle id and the error class name ('' when none)."""
    import parcels_b200 as pb

    keys = TRAJ + (("next_dt",) if k["fam"] == "rk45" else ())
    if k["path"] == "columns":
        return _sorted(_run_columns(c, k, order), keys), ""
    env = _env(k)
    os.environ.update(env)
    try:
        fs = _fieldset(c, k)
        ps = pb.ParticleSet(fs, pclass=_pclass(k), x=c["x"][order], y=c["y"][order], z=c["z"][order], t=c["t"][order],
                            particle_ids=order, seed=SEED)  # fmt: skip
        err = ""
        try:
            for seg in c["segments"]:
                ps.execute(_kernels(c, k), dt=c["dt"], **seg)
        except RuntimeError as e:
            if type(e).__module__.startswith("parcels_b200._lib"):
                raise
            err = type(e).__name__
        return _sorted(ps._data, keys), err
    finally:
        for key in env:
            os.environ.pop(key, None)


# Column slabs: two slab engines of one process with in-kernel migration (scripts/decomposed_threads_check.py); the curvilinear
# cases have 30 cell columns, cut at column 15.  Fused DiffusionUniformKh keys its Wiener increments by the launch (every migration
# round is a new RNG call, distributed._advect_args), so its keys keep their particles off the cell columns next to that edge: a
# particle moves less than a cell in these runs, the call is one launch (round 0 of call 1) and the oracle draws its increments.
WORLD = 2
EDGE_COLUMNS = (13, 17)


@contextlib.contextmanager
def _engine_calls_serialised():
    """thread_ranks.serialise_engine_calls for the duration of a column-slab run: the Engine methods are restored afterwards."""
    from parcels_b200.engine import Engine

    saved = dict(vars(Engine))
    thread_ranks.serialise_engine_calls()
    try:
        yield
    finally:
        for name, method in saved.items():
            if vars(Engine).get(name) is not method:
                setattr(Engine, name, method)
        thread_ranks._serialised = False


def _run_columns(c, k, order):
    from parcels_b200 import distributed as D
    from parcels_b200.particle import create_particle_data

    world = WORLD
    n = len(order)
    slabs = []
    for r in range(world):
        dfs = D.DecomposedFieldSet.from_curvilinear(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"],
                                                    W=c["W"], mesh=c["mesh"], rank=r, world=world, halo_cells=3, device=0,
                                                    interp_method=c["interp"], padding=c.get("padding", ("low", "low", "high")))  # fmt: skip
        _setup(dfs.fs, c, k)
        slabs.append(dfs)
    full = create_particle_data(nparticles=n, ngrids=len(slabs[0].fs.gridset), initial=dict(x=c["x"][order], y=c["y"][order], z=c["z"][order], t=c["t"][order],
                                                                       particle_id=np.asarray(order)))  # fmt: skip
    full["dt"][:] = c["dt"]
    if k["fam"] == "rk45":
        full["next_dt"] = np.zeros(n, dtype=np.float32)
    bases = [s.engine.migrate_p2p_init(n)[1] for s in slabs]
    for s in slabs:
        s.engine.migrate_p2p_connect(local_bases=bases)
        s.p2p = True
    endtime = float(c["segments"][0]["runtime"]) * np.sign(c["dt"])
    with _engine_calls_serialised():
        res = thread_ranks.run_ranks(world, lambda r, dist: D.execute_decomposed(slabs[r], D.shard_particles(full, r, world),
                                                                                 _kernels(c, k, True), c["dt"], endtime, dist, seed=SEED))  # fmt: skip
    outs = [o for o, _ in res]
    rounds = {s["rounds"] for _, s in res}
    if k.get("diff"):
        assert rounds == {1}, f"a particle crossed the column-slab edge: {rounds} rounds"
    else:
        assert max(rounds) > 1 or HOSTSIM, "no particle crossed a column-slab edge"  # (the simulation runs too few to say)
    return {key: np.concatenate([o[key] for o in outs], axis=0) for key in outs[0]}


# ------------------------------------------------------------------------------------------------
# the oracle (in engine arithmetic: the device's own sin / cos)
# ------------------------------------------------------------------------------------------------
def _ofs(c):
    pad = c.get("padding", ("low", "low", "high"))
    g = po.OGrid(c["lon"], c["lat"], c["depth"], mesh=c["mesh"], offsets=tuple(int(p == "low") for p in pad))
    return po.OFieldSet(g, c["U"], c["V"], c["W"], time=c["times"], constants=c["constants"], interp=c.get("interp", "linear"))


def run_oracle(c, k):
    """The oracle on every particle (ids 0 .. n-1); the Wiener increments are the engine's (philox_ref.device_normals)."""
    ids = np.arange(len(c["x"]))
    with trig.use(DeviceTrig()):
        ofs = _ofs(c)
        pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"], ngrids=ofs.ngrids, particle_ids=ids)
        rng_call = (1 << 20) if k["path"] == "columns" else 1  # (column slabs: round 0 of call 1, distributed._advect_args)
        it = [0]

        def normal(view):
            zx, zy = device_normals(SEED, rng_call, it[0], view.particle_id)
            it[0] += 1
            return zx, zy

        if k["fam"] == "rk45":
            ctx = _rk45_context(c)
            if ofs.grid.spherical:
                ctx["RK45_tol"] = ctx["RK45_tol"] / ofs.grid.deg2m
            ofs.context.update(ctx)
            pd["next_dt"] = np.zeros(len(ids), dtype=np.float32)
        if k["fam"] == "advdiff":
            kz, km, dres = _kh(c, k)
            ofs.scalars = {"Kh_zonal": (kz, "linear"), "Kh_meridional": (km, "linear")}
            ofs.context["dres"] = dres
        kern = []
        for name in c["kernels"]:
            if name == "DiffusionUniformKh":
                kern.append(po.DiffusionUniformKh(normal))
            elif name in ("AdvectionDiffusionM1", "AdvectionDiffusionEM"):
                kern.append(getattr(po, name)(normal))
            else:
                kern.append(getattr(po, name))
        if (c["delete_on_error"] and k["fam"] != "rk45") or k["path"] == "columns":
            kern.append(po.DeleteOnError)
        err = None
        try:
            for seg in c["segments"]:
                po.pset_execute(pd, ofs, kern, c["dt"], **seg)
        except po.OracleParticleError as e:
            err = e.code
    return pd, err


# ------------------------------------------------------------------------------------------------
# sampling: fs.UV / fs.UVW.eval and Field.eval
# ------------------------------------------------------------------------------------------------
def samples(c, n=N):
    """n sample positions and times: the case's particles (NaN dropped: eval raises on a NaN time only, but the reference's
    search of a NaN position is not defined; positions outside the domain kept: their state is ErrorOutOfBounds) at times
    spread over the time axis."""
    ok = np.isfinite(c["x"])
    x, y, z = c["x"][ok][:n], c["y"][ok][:n], c["z"][ok][:n]
    times = c["times"]
    t = np.zeros(len(x)) if times is None else np.random.default_rng(5).uniform(times[0], times[-1], len(x))
    return t, z, y, x


def scalar_data(c, k):
    P = np.asarray(c["U"], dtype=np.float64) + 0.25 * np.asarray(c["V"], dtype=np.float64) + 1.0
    if not k["ht"]:
        P = P[:1]
    return P.astype(k["d"])


def _shifted(c, z, y, x):
    """float64 positions a little off the first ones (an RK stage position), for the second evaluation, hinted by the first."""
    step = 1e-3 if c["mesh"] == "spherical" else 0.5
    return np.asarray(z, dtype=np.float64), np.asarray(y, dtype=np.float64) + step, np.asarray(x, dtype=np.float64) + step


def sample_engine(c, k, t, z, y, x):
    """fs.UV / fs.UVW.eval or Field.eval with a ParticleSet at the sample positions, twice: at its float32 positions, then at
    float64 positions hinted by the cells the first evaluation wrote back.  Returns (values of each evaluation, ei, state)."""
    import parcels_b200 as pb

    fs = _fieldset(c, k)
    if k["fam"] == "scalar":
        fs.add_field("P", scalar_data(c, k), interp_method=k["method"])
        f = fs.P
    else:
        f = fs.UVW if k["nc"] == 3 else fs.UV
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=t)
    d = ps._data
    vals = []
    for zz, yy, xx in ((d["z"], d["y"], d["x"]), _shifted(c, d["z"], d["y"], d["x"])):
        v = f.eval(t, zz, yy, xx, ps)
        vals.append(tuple(np.asarray(a) for a in (v if isinstance(v, tuple) else (v,))))
    return vals, np.asarray(d["ei"]).copy(), np.asarray(d["state"]).copy()


def sample_oracle(c, k, t, z, y, x):
    """sample_engine's two evaluations on the oracle (its own dtypes: nothing is cast)."""
    with trig.use(DeviceTrig()):
        ofs = _ofs(c)
        pd = po.create_particle_data(x, y, z, t)
        view = po.View(pd, np.ones(len(pd["x"]), dtype=bool))
        vals = []
        for zz, yy, xx in ((pd["z"], pd["y"], pd["x"]), _shifted(c, pd["z"], pd["y"], pd["x"])):
            if k["fam"] == "scalar":
                vals.append((np.asarray(po.eval_scalar(ofs, scalar_data(c, k), k["method"], t, zz, yy, xx, view)),))
            else:
                vals.append(tuple(np.asarray(v) for v in po.eval_uvw(ofs, t, zz, yy, xx, view, k["nc"] == 3)))
    return vals, pd["ei"], pd["state"]


# ------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------
def assert_same(a, b, what):
    """Bit-identical columns (a and b: dicts of arrays in the same particle order)."""
    assert a.keys() == b.keys(), what
    for key in a:
        x, y = np.ascontiguousarray(a[key]), np.ascontiguousarray(b[key])
        assert x.shape == y.shape and x.dtype == y.dtype, f"{what}: {key}: {x.shape} {x.dtype} vs {y.shape} {y.dtype}"
        if x.size == 0:
            continue
        bad = np.flatnonzero((x.view(np.uint8).reshape(len(x), -1) != y.view(np.uint8).reshape(len(y), -1)).any(axis=1))
        assert bad.size == 0, f"{what}: {key} differs for {bad.size} of {len(x)}, first at {bad[:4]}: {x[bad[:4]]} vs {y[bad[:4]]}"


def assert_oracle(got, pd, keys, what):
    o = np.argsort(pd["particle_id"], kind="stable")
    np.testing.assert_array_equal(got["particle_id"], pd["particle_id"][o], err_msg=f"{what}: surviving ids")
    for key in keys:
        np.testing.assert_array_equal(got[key], np.asarray(pd[key])[o], err_msg=f"{what}: {key}")
