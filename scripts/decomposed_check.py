"""Mode D check (launch with torchrun, N ranks): domain-decomposed execution with particle migration
reproduces the single-GPU trajectories BIT-EXACTLY.  With --same-gpu all ranks share cuda:0 and the
exchange goes through gloo (host-staged) -- this is how the 1-GPU `pytest -m gpu` run covers the path;
on a multi-GPU box the records travel over NCCL."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import numpy as np
import torch
import torch.distributed as dist

import bench
import decomposed_kernels
import parcels_b200 as pb
from parcels_b200 import distributed as D
from parcels_b200.particle import create_particle_data

ap = argparse.ArgumentParser()
ap.add_argument("--same-gpu", action="store_true")
ap.add_argument("--particles", type=int, default=20000)
ap.add_argument("--halo", type=int, default=3)
ap.add_argument("--umax", type=float, default=40.0, help="velocity scale: large => many slab crossings")
ap.add_argument("--transport", default="auto", choices=["auto", "p2p", "collective"],
                help="p2p: in-kernel migration over peer memory (CUDA IPC; default over NCCL); collective: classify / pack / all-to-all")
ap.add_argument("--inbox", type=int, default=0, help="p2p: records per inbox slot (default: the particle count; small values exercise the overflow path)")
ap.add_argument("--time-window", type=int, default=0, help="time-slab streaming under mode D: W levels of each slab resident, windows slid in "
                "lock-step (the undecomposed comparison run keeps every level resident)")
ap.add_argument("--nt", type=int, default=3, help="time levels of the synthetic field (one day apart)")
ap.add_argument("--runtime", type=float, default=86400.0)
ap.add_argument("--diffusion", action="store_true", help="fused DiffusionUniformKh on a field at rest: statistical check (Var = 2 K t)")
ap.add_argument("--kernel", default="rk4_3d", choices=list(decomposed_kernels.KERNELS),
                help="[AdvectionRK4 | RK4_3D | RK45 | AdvectionDiffusionM1 | EM, DeleteParticle]; anything but the default XLinear_Velocity "
                "RK4_3D run on a spherical mesh takes its case from scripts/decomposed_kernels.py")
ap.add_argument("--interp", default="linear", choices=list(decomposed_kernels.INTERP),
                help="vector interpolator of the slabs: XLinear_Velocity, CGrid_Velocity, XFreeslip, XPartialslip, nearest node")
ap.add_argument("--dt", type=float, default=600.0, help="time step in seconds (RK45: the initial one)")
ap.add_argument("--f32-coords", action="store_true", help="float32 lon / lat / depth")
ap.add_argument("--ordered-releases", action="store_true", help="delayed releases in the order of the particle ids")
ap.add_argument("--mesh", default="spherical", choices=["spherical", "flat"])
ap.add_argument("--backward", action="store_true")
ap.add_argument("--delayed", action="store_true", help="releases at three different times")
ap.add_argument("--max-dt", type=float, default=3600.0, help="RK45_max_dt")
ap.add_argument("--dres", type=float, default=0.05, help="fieldset.dres of M1 / EM (degrees or mesh units)")
ap.add_argument("--rk45-tol", type=float, default=100.0, help="RK45_tol in metres")
a = ap.parse_args()
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = 0 if a.same_gpu else int(os.environ.get("LOCAL_RANK", rank))
if torch.cuda.is_available():  # (not under the host simulation of the test suite, oracle/hostsim)
    torch.cuda.set_device(dev)
dist.init_process_group("gloo" if a.same_gpu else "nccl")
p2p = a.transport == "p2p" or (a.transport == "auto" and not a.same_gpu)

f = bench.c2_field(nx=120, ny=60, nz=12, nt=a.nt)
f["U"] *= np.float32(a.umax)
f["V"] *= np.float32(a.umax)
n = a.particles
rng = np.random.default_rng(7)
x, y, z = rng.uniform(-175, 175, n), rng.uniform(-70, 70, n), rng.uniform(5, 5000, n)
dt, runtime = 600.0, a.runtime
if a.diffusion:
    # a field at rest and a large constant diffusivity: particles released on the slab boundary (lon 0, equator) diffuse across it
    K, runtime = 1.0e5, 28800.0
    for k in "UVW":
        f[k] *= np.float32(0)
    x, y, z = np.zeros(n), np.zeros(n), np.full(n, 100.0)
    full = create_particle_data(nparticles=n, ngrids=2, initial=dict(x=x, y=y, z=z, t=np.zeros(n), particle_id=np.arange(n)))
    dfs = D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                               mesh="spherical", rank=rank, world=world, halo_cells=a.halo, device=dev,
                               **decomposed_kernels.fieldset_kwargs(a.interp))  # fmt: skip
    dfs.fs.add_constant_field("Kh_zonal", K, mesh="spherical")
    dfs.fs.add_constant_field("Kh_meridional", K, mesh="spherical")
    if p2p:
        D.connect_p2p(dfs, dist, a.inbox or n)
    out, stats = D.execute_decomposed(dfs, D.shard_particles(full, rank, world), [pb.AdvectionRK4_3D, pb.DiffusionUniformKh, pb.DeleteParticle],
                                      dt, runtime, dist, seed=11)
    tot = D.allreduce_sum(stats["migrated"], dist, device="cpu" if a.same_gpu else f"cuda:{dev}")
    merged = D.gather_particles(out, dist, dst=0)
    ok = True
    if rank == 0:
        sigma = np.sqrt(2 * K * runtime) / dfs.fs.grid.deg2m  # degrees (cos(lat) ~ 1 at the equator)
        sx, sy = float(np.std(merged["x"])), float(np.std(merged["y"]))
        ok = (len(merged["x"]) == n and len(np.unique(merged["particle_id"])) == n and abs(sx / sigma - 1) < 0.06 and abs(sy / sigma - 1) < 0.06
              and abs(float(np.mean(merged["x"]))) < 5 * sigma / np.sqrt(n) and tot > n / 4)  # fmt: skip
        print(f"decomposed diffusion ({world} ranks): {len(merged['x'])} particles, {int(tot)} migrations, rounds={stats['rounds']}, "
              f"std x {sx:.4f} y {sy:.4f} expected {sigma:.4f} -> {'PASS statistics' if ok else 'FAIL'}")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)
if (a.kernel != "rk4_3d" or a.interp != "linear" or a.mesh != "spherical" or a.backward or a.delayed or a.f32_coords
        or a.ordered_releases or a.dt != 600.0):  # fmt: skip
    case = decomposed_kernels.make_case(a.kernel, mesh=a.mesh, n=n, nt=a.nt, runtime=a.runtime, backward=a.backward,
                                        delayed=a.delayed or bool(a.time_window), max_dt=a.max_dt, dres=a.dres, tol=a.rk45_tol,
                                        interp=a.interp, f32_coords=a.f32_coords, dt=a.dt, ordered=a.ordered_releases)  # fmt: skip
    dfs = decomposed_kernels.decomposed_fieldset(case, rank, world, halo=a.halo, time_window=a.time_window or None, device=dev)
    if p2p:
        D.connect_p2p(dfs, dist, a.inbox or n)
    try:
        out, stats = D.execute_decomposed(dfs, D.shard_particles(case["full"], rank, world), case["kernels"], case["dt"],
                                          case["endtime"], dist, seed=case["seed"])  # fmt: skip
    except RuntimeError as e:  # (every rank raises a halo violation in the same round)
        print(f"rank {rank}: RuntimeError: {e}")
        dist.destroy_process_group()
        sys.exit(3)
    tot = D.allreduce_sum(stats["migrated"], dist, device="cpu" if a.same_gpu else f"cuda:{dev}")
    merged = D.gather_particles(out, dist, dst=0)
    ok = True
    if rank == 0:
        ref = decomposed_kernels.reference(case, device=dev)
        ok, msgs = decomposed_kernels.compare(merged, ref, a.kernel)
        print("\n".join(msgs))
        print(f"decomposed {a.kernel} ({a.interp}, {world} ranks, backend={dist.get_backend()}, {a.mesh}{', backward' if a.backward else ''}): "
              f"{len(ref['x'])} of {n} left, {int(tot)} migrations, rounds={stats['rounds']}, transport={stats['transport']}"
              + (f", time window {a.time_window} of {a.nt} levels" if a.time_window else "") + f" -> {'PASS bit-exact' if ok else 'FAIL'}")  # fmt: skip
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)
full = create_particle_data(nparticles=n, ngrids=1, initial=dict(x=x, y=y, z=z, t=np.zeros(n), particle_id=np.arange(n)))
dfs = D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                           mesh="spherical", rank=rank, world=world, halo_cells=a.halo, device=dev, time_window=a.time_window or None)
if p2p:
    D.connect_p2p(dfs, dist, a.inbox or n)
mine = D.shard_particles(full, rank, world)  # arbitrary shard: routed to the owners by the first migration round
out, stats = D.execute_decomposed(dfs, mine, [pb.AdvectionRK4_3D, pb.DeleteParticle], dt, runtime, dist)
tot = D.allreduce_sum(stats["migrated"], dist, device="cpu" if a.same_gpu else f"cuda:{dev}")
merged = D.gather_particles(out, dist, dst=0)
ok = True
if rank == 0:
    order = np.argsort(merged["particle_id"], kind="stable")
    merged = {k: v[order] for k, v in merged.items()}
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                                 mesh="spherical")
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=np.zeros(n), device=dev)
    ps.execute([pb.AdvectionRK4_3D, pb.DeleteParticle], dt=dt, runtime=runtime)
    ref = ps._data
    for k in ("particle_id", "state", "t", "ei", "x", "y", "z"):
        same = merged[k].shape == ref[k].shape and np.array_equal(merged[k], ref[k])
        ok &= same
        if not same:
            print(f"MISMATCH {k}: {merged[k].shape} vs {ref[k].shape}")
            if merged[k].shape == ref[k].shape:
                bad = np.where((merged[k] != ref[k]).reshape(len(ref[k]), -1).any(axis=1))[0]
                print("   count", len(bad), "first:", [(int(merged["particle_id"][b]), merged[k][b].tolist(), ref[k][b].tolist(),
                                                        float(merged["x"][b]), float(ref["x"][b])) for b in bad[:6]])
    print(f"decomposed({world} ranks, backend={dist.get_backend()}): {len(ref['x'])} survivors, {int(tot)} migrations, "
          f"rounds={stats['rounds']}, transport={stats['transport']}"
          + (f", time window {a.time_window} of {a.nt} levels" if a.time_window else "") + f" -> {'PASS bit-exact' if ok else 'FAIL'}")
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
