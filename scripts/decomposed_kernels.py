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

KERNELS = {"rk4": pb.AdvectionRK4, "rk4_3d": pb.AdvectionRK4_3D, "rk45": pb.AdvectionRK45, "m1": pb.AdvectionDiffusionM1,
           "em": pb.AdvectionDiffusionEM}  # fmt: skip
# --interp of the scripts -> FieldSet.from_arrays' interp_method; C-grids take the SGRID padding of NEMO-like output
INTERP = {"linear": "linear", "cgrid": "cgrid_velocity", "freeslip": "freeslip", "partialslip": "partialslip", "nearest": "nearest"}
# land (U = V = W = 0) for the slip and nearest-node cases: blocks of columns around the interior slab edges of 2 and 3 slabs
# (nodes 60; 40 and 79 of 120), so that the slip factors act where particles cross from one slab to the next
LAND_COLUMNS = [slice(36, 45), slice(56, 65), slice(75, 84)]
LAND_ROWS = slice(20, 41)


def fieldset_kwargs(interp):
    kw = dict(interp_method=INTERP[interp])
    if interp == "cgrid":
        kw["padding"] = ("low", "low", "high")
    return kw


NEXT_DT = pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0))


def make_case(kernel, *, mesh="spherical", n=1000, nt=3, runtime=86400.0, backward=False, delayed=False, max_dt=3600.0, dres=0.05,
              tol=100.0, seed=7, interp="linear", f32_coords=False, dt=600.0, ordered=False):  # fmt: skip
    """``ordered``: delayed releases in the order of the particle ids, so that the first shards hold only particles on the first
    time level and the batch-level bits of the call's first evaluation must come from the whole set."""
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
    dfs = D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                               mesh=case["mesh"], rank=rank, world=world, halo_cells=halo, device=device, time_window=time_window,
                               **case["fs_kw"])  # fmt: skip
    setup(dfs, case, time_window)
    return dfs


def reference(case, device=0) -> dict:
    """The single-engine run with every time level resident."""
    f = case["f"]
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                                 mesh=case["mesh"], **case["fs_kw"])  # fmt: skip
    setup(fs, case)
    pclass = NEXT_DT if case["kernel"] == "rk45" else pb.Particle
    ps = pb.ParticleSet(fs, pclass=pclass, x=case["x"], y=case["y"], z=case["z"], t=case["t"], device=device, seed=case["seed"])
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
