"""Cases of mode D beyond the default XLinear_Velocity RK4_3D run, shared by scripts/decomposed_check.py (gloo / NCCL ranks) and
scripts/decomposed_threads_check.py (thread ranks, in-kernel migration): the fixed-step RK4 / RK4_3D, AdvectionRK45 and
AdvectionDiffusionM1 / EM on the config-2 field shape at 3-degree resolution, fast enough that particles cross slab edges several
times a day, with any of the vector interpolators a slab can run (``INTERP``), and the undecomposed single-engine run the
decomposed one must equal bit for bit (ids, x, y, z, t, state, ei; RK45 also dt and next_dt)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np

import bench
import parcels_b200 as pb
from parcels_b200.particle import create_particle_data

KERNELS = {"ee": pb.AdvectionEE, "rk4": pb.AdvectionRK4, "rk4_3d": pb.AdvectionRK4_3D, "rk45": pb.AdvectionRK45, "m1": pb.AdvectionDiffusionM1,
           "em": pb.AdvectionDiffusionEM}  # fmt: skip
# --interp of the scripts -> FieldSet.from_arrays' interp_method; C-grids take the SGRID padding of NEMO-like output.  curv_*: the
# same interpolators on a CURVILINEAR grid cut into column slabs (DecomposedFieldSet.from_curvilinear)
INTERP = {"linear": "linear", "cgrid": "cgrid_velocity", "freeslip": "freeslip", "partialslip": "partialslip", "nearest": "nearest",
          "curv_cgrid": "cgrid_velocity", "curv_linear": "linear"}  # fmt: skip
# land (U = V = W = 0) for the slip and nearest-node cases: blocks of columns around the interior slab edges of 2 and 3 slabs
# (nodes 60; 40 and 79 of 120), so that the slip factors act where particles cross from one slab to the next
LAND_COLUMNS = [slice(36, 45), slice(56, 65), slice(75, 84)]
LAND_ROWS = slice(20, 41)


def fieldset_kwargs(interp):
    kw = dict(interp_method=INTERP[interp])
    if interp in ("cgrid", "curv_cgrid"):
        kw["padding"] = ("low", "low", "high")
    return kw


def curvilinear_field(kernel, mesh, nt, f32_coords):
    """A small config-3 field (bench.c3_field: rotated-pole ORCA-like mesh, float32 nodes) on a spherical mesh, or the warped
    mesh of tests/cases.curv_mesh on a flat one, fast enough that particles cross several cell columns a day."""
    from cases import curv_mesh

    nz = 6 if kernel == "rk4_3d" else 1
    f = bench.c3_field(nx=72, ny=48, nt=nt, nz=nz)
    if mesh == "flat":
        f["lon"], f["lat"] = curv_mesh(48, 72, False, np.float32 if f32_coords else np.float64)
        f["mesh"] = "flat"
        if f["depth"] is not None:
            f["depth"] = f["depth"].astype(f["lon"].dtype)
    scale = np.float32(40.0 if mesh == "spherical" else 0.02)
    f["U"] *= scale
    f["V"] *= scale
    if f["W"] is not None:
        f["W"] *= np.float32(10.0)
    # a strong meridional shear across the first-column cell next to the node closest to the equator (where particles_in puts
    # particles hinted by that cell): a float32 rounding of its eta coordinate moves the step by more than the float32 ulp of y there
    j0 = max(int(np.argmin(np.abs(np.asarray(f["lat"], dtype=np.float64)[:, 0]))), 1)
    f["V"][:, :, j0 - 1, :3] = np.float32(3.0) * scale
    f["V"][:, :, j0, :3] = np.float32(-3.0) * scale
    return f


def particles_in(f, n, rng):
    """n positions inside the mesh (random cells, bilinear blends of their corners), every 50th one outside it, and every 10th
    (ids 3, 13, ...) inside a cell of the first column, (row, 0): with the hint (row, 0) -- xi = 0 -- the hint test finds it, so
    whether its first evaluation skips the hint (the hash path, float32-rounded coordinates) or not shows in its bits.  Returns x, y, z
    and the hint rows (-1: none)."""
    from cases import points_in_mesh

    lon, lat = f["lon"].astype(np.float64), f["lat"].astype(np.float64)
    x, y = points_in_mesh(rng, lon, lat, n, margin=2.0)
    out = np.arange(n) % 50 == 49
    x[out] = float(f["lon"].max()) + 5.0 * (np.abs(float(f["lon"].max())) if f["mesh"] == "flat" else 1.0)
    rows = np.full(n, -1)
    edge = np.arange(n) % 10 == 3
    k = int(edge.sum())
    # next to the node of the first column closest to the equator (the origin on a flat mesh): the float32 ulp of y is small there,
    # so the float32 rounding of the hash path's coordinates shows in the positions
    j0 = int(np.argmin(np.abs(lat[:, 0])))
    row, fj = (j0 - 1, rng.uniform(0.8, 0.98, k)) if j0 > 0 else (0, rng.uniform(0.02, 0.2, k))
    rows[edge] = row
    fi = rng.uniform(0.02, 0.5, k)
    j = rows[edge]
    for a, dst in ((lon, x), (lat, y)):
        dst[edge] = (1 - fj) * (1 - fi) * a[j, 0] + (1 - fj) * fi * a[j, 1] + fj * fi * a[j + 1, 1] + fj * (1 - fi) * a[j + 1, 0]
    depth = f.get("depth")
    z = np.zeros(n) if depth is None else rng.uniform(float(depth[1]), float(depth[-2]), n)
    return x, y, z, rows


NEXT_DT = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0))


def make_case(kernel, *, mesh="spherical", n=1000, nt=3, runtime=86400.0, backward=False, delayed=False, max_dt=3600.0, dres=0.05,
              tol=100.0, seed=7, interp="linear", f32_coords=False, dt=600.0, ordered=False):  # fmt: skip
    """``ordered``: delayed releases in the order of the particle ids, so that the first shards hold only particles on the first
    time level and the batch-level bits of the call's first evaluation must come from the whole set."""
    if interp.startswith("curv_"):
        return make_curvilinear_case(kernel, mesh=mesh, n=n, nt=nt, runtime=runtime, backward=backward, delayed=delayed,
                                     max_dt=max_dt, tol=tol, seed=seed, interp=interp, f32_coords=f32_coords, dt=dt, ordered=ordered)  # fmt: skip
    f = bench.c2_field(nx=120, ny=60, nz=12, nt=nt)
    # ~40 m/s on the sphere (~30 degrees a day); the same displacement in mesh units on a flat mesh -- and with nearest-node
    # sampling, which converts no units: its values are degrees per second on the sphere too
    scale = np.float32(40.0 if mesh == "spherical" and interp != "nearest" else 40.0 / 111319.49)
    f["U"] *= scale
    f["V"] *= scale
    if interp in ("freeslip", "partialslip", "nearest"):
        for k in "UVW":
            for cols in LAND_COLUMNS:
                f[k][:, :, LAND_ROWS, cols] = 0
    if f32_coords:
        for k in ("lon", "lat", "depth"):
            f[k] = f[k].astype(np.float32)
    rng = np.random.default_rng(seed)
    x, y, z = rng.uniform(-175, 175, n), rng.uniform(-70, 70, n), rng.uniform(5, 5000, n)
    dt = -abs(dt) if backward else abs(dt)
    t_start = float(f["times"][-1]) if backward else 0.0
    delays = rng.choice([0.0, 7200.0, 40000.0], n) if delayed or ordered else np.zeros(n)
    t = t_start + np.sign(dt) * (np.sort(delays) if ordered else delays)
    endtime = t_start + np.sign(dt) * runtime
    context = {"dres": float(dres)}
    if kernel == "rk45":
        # a step of max_dt moves a particle ~1.3 degrees at 40 m/s: inside a halo of one 3-degree cell
        context = {"RK45_tol": tol if mesh == "spherical" else tol / 111319.49, "RK45_min_dt": 1.0, "RK45_max_dt": float(max_dt)}
    Z = np.linspace(0, 1, 12, dtype=np.float32)[None, :, None, None]
    Y = np.linspace(-1, 1, 60, dtype=np.float32)[None, None, :, None]
    X = np.linspace(0, 6.283, 120, dtype=np.float32)[None, None, None, :]
    T = np.arange(nt, dtype=np.float32)[:, None, None, None]
    kh = (2000.0 + 1500.0 * np.sin(X + 0.5 * T) * np.cos(2 * Y) + 500.0 * Z).astype(np.float32)
    if mesh == "flat":
        kh *= np.float32(1.0 / 111319.49**2)
    full = create_particle_data(nparticles=n, ngrids=1, initial=dict(x=x, y=y, z=z, t=t, particle_id=np.arange(n)))
    full["dt"][:] = dt  # ParticleSet.execute's `particles.dt = dt`
    if kernel == "rk45":
        full["next_dt"] = np.zeros(n, dtype=np.float32)
    kernels = [KERNELS[kernel], pb.DeleteParticle]
    return dict(kernel=kernel, f=f, mesh=mesh, x=x, y=y, z=z, t=t, dt=dt, endtime=endtime, full=full, kernels=kernels,
                context=context, kh=(kh, np.ascontiguousarray(kh[..., ::-1])), seed=11, fs_kw=fieldset_kwargs(interp))  # fmt: skip


def make_curvilinear_case(kernel, *, mesh, n, nt, runtime, backward, delayed, max_dt, tol, seed, interp, f32_coords, dt, ordered):
    """``make_case`` on a curvilinear grid (column slabs).  Every hinted xi is 0 (``particles_in``: some particles sit in, and are
    hinted by, cells of the first column), so the whole set skips the hint at its first evaluation -- also the particles that
    start on another rank than the owner of their cell.  ``ordered`` also gives the particles of the second half of the ids a
    non-zero hint (ei = 1): the first shards' hints are all zero while the whole set's are not, and the first-column particles
    of those shards take the hint -- the reference's `if np.any(xi)` must be decided over the whole set."""
    f = curvilinear_field(kernel, mesh, nt, f32_coords)
    rng = np.random.default_rng(seed)
    x, y, z, rows = particles_in(f, n, rng)
    dt = -abs(dt) if backward else abs(dt)
    t_start = float(f["times"][-1]) if backward else 0.0
    delays = rng.choice([0.0, 7200.0, 40000.0], n) if delayed or ordered else np.zeros(n)
    t = t_start + np.sign(dt) * (np.sort(delays) if ordered else delays)
    endtime = t_start + np.sign(dt) * runtime
    context = {}
    if kernel == "rk45":
        context = {"RK45_tol": tol if mesh == "spherical" else tol / 111319.49, "RK45_min_dt": 1.0, "RK45_max_dt": float(max_dt)}
    full = create_particle_data(nparticles=n, ngrids=1, initial=dict(x=x, y=y, z=z, t=t, particle_id=np.arange(n)))
    full["dt"][:] = dt
    full["ei"][rows >= 0, 0] = rows[rows >= 0] * (f["lon"].shape[1] - 1)  # hints (row, 0): every hinted xi is still 0
    if ordered:
        full["ei"][n // 2 :, 0] = 1
    if kernel == "rk45":
        full["next_dt"] = np.zeros(n, dtype=np.float32)
    return dict(kernel=kernel, f=f, mesh=mesh, x=x, y=y, z=z, t=t, dt=dt, endtime=endtime, full=full, kernels=[KERNELS[kernel], pb.DeleteParticle],
                context=context, seed=11, fs_kw=fieldset_kwargs(interp), curvilinear=True)  # fmt: skip


def setup(fs, case, time_window=None):
    """The context values and the Kh_zonal / Kh_meridional fields of ``case`` on a FieldSet or a DecomposedFieldSet."""
    for k, v in case["context"].items():
        fs.add_context(k, v)
    if case["kernel"] in ("m1", "em"):
        fs.add_field("Kh_zonal", case["kh"][0], time_window=time_window)
        fs.add_field("Kh_meridional", case["kh"][1], time_window=time_window)


def decomposed_fieldset(case, rank, world, halo=1, time_window=None, device=0):
    from parcels_b200 import distributed as D

    f = case["f"]
    if case.get("curvilinear"):
        dfs = D.DecomposedFieldSet.from_curvilinear(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"],
                                                    W=f["W"] if case["kernel"] == "rk4_3d" else None, mesh=case["mesh"], rank=rank,
                                                    world=world, halo_cells=halo, device=device, time_window=time_window, **case["fs_kw"])  # fmt: skip
        grid_b, field_b = dfs.engine.memory_bytes()
        print(f"rank {rank}: column slab {dfs.plan['lo']}..{dfs.plan['hi']} of {f['lon'].shape[1]} node columns, "
              f"grid {grid_b} B, fields {field_b} B on the device")
    else:
        dfs = D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                                   mesh=case["mesh"], rank=rank, world=world, halo_cells=halo, device=device, time_window=time_window,
                                   **case["fs_kw"])  # fmt: skip
    setup(dfs, case, time_window)
    return dfs


def reference(case, device=0) -> dict:
    """The single-engine run with every time level resident."""
    f = case["f"]
    W = None if case.get("curvilinear") and case["kernel"] != "rk4_3d" else f["W"]
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=W,
                                 mesh=case["mesh"], **case["fs_kw"])  # fmt: skip
    setup(fs, case)
    pclass = NEXT_DT if case["kernel"] == "rk45" else pb.Particle
    ps = pb.ParticleSet(fs, pclass=pclass, x=case["x"], y=case["y"], z=case["z"], t=case["t"], device=device, seed=case["seed"])
    if case.get("curvilinear"):
        ps._data["ei"][:] = case["full"]["ei"]  # (the hints of the decomposed run's set)
    ps.execute(case["kernels"], dt=case["dt"], endtime=case["endtime"])
    return ps._data


def compare(merged, ref, kernel):
    """Bit-exact comparison of the merged decomposed result (any order) with the reference; returns (ok, messages)."""
    order = np.argsort(merged["particle_id"], kind="stable")
    merged = {k: v[order] for k, v in merged.items()}
    keys = ["particle_id", "state", "t", "ei", "x", "y", "z"] + (["dt", "next_dt"] if kernel == "rk45" else [])
    ok, msgs = True, []
    for k in keys:
        same = merged[k].shape == ref[k].shape and merged[k].dtype == ref[k].dtype and np.array_equal(merged[k], ref[k])
        ok &= same
        if not same:
            msgs.append(f"MISMATCH {k}: {merged[k].shape} {merged[k].dtype} vs {ref[k].shape} {ref[k].dtype}")
    return ok, msgs
