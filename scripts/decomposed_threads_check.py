"""Mode D with IN-KERNEL migration driven by the product's own round loop (distributed.run_decomposed_p2p /
execute_decomposed) on the host simulation: CUDA IPC needs real devices, so the ranks are THREADS of one process -- each with its
own engine, inboxes linked by address (pb_migrate_p2p_connect's local bases) -- and ``torch.distributed`` is replaced by a
thread-barrier stand-in with the same calls.  Engine calls of different ranks are serialised by a lock (the simulated device
runs a kernel as a loop over global thread / block indices and its atomics are plain host operations).  Checks the merged result
bit for bit against the undecomposed run; with --time-window the slabs stream their time levels and slide in lock-step while the
comparison run keeps every level resident.
Run:  PB_LIB=oracle/_build/hostsim/libparcels_b200_hostsim.so PB_HOSTSIM_TEST=1 python scripts/decomposed_threads_check.py"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import numpy as np

import bench
import decomposed_kernels
import parcels_b200 as pb
import thread_ranks
from parcels_b200 import distributed as D
from parcels_b200.particle import create_particle_data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=3)
    ap.add_argument("--particles", type=int, default=3000)
    ap.add_argument("--inbox", type=int, default=0)
    ap.add_argument("--time-window", type=int, default=0)
    ap.add_argument("--nt", type=int, default=3)
    ap.add_argument("--runtime", type=float, default=86400.0)
    ap.add_argument("--backward", action="store_true")
    ap.add_argument("--kernel", default="rk4_3d", choices=list(decomposed_kernels.KERNELS),
                    help="[AdvectionRK4 | RK4_3D | RK45 | AdvectionDiffusionM1 | EM, DeleteParticle]; anything but the default "
                    "XLinear_Velocity RK4_3D run on a spherical mesh takes its case from scripts/decomposed_kernels.py")
    ap.add_argument("--interp", default="linear", choices=list(decomposed_kernels.INTERP),
                    help="vector interpolator of the slabs: XLinear_Velocity, CGrid_Velocity, XFreeslip, XPartialslip, nearest node")
    ap.add_argument("--dt", type=float, default=600.0, help="time step in seconds (RK45: the initial one)")
    ap.add_argument("--f32-coords", action="store_true", help="float32 lon / lat / depth")
    ap.add_argument("--ordered-releases", action="store_true", help="delayed releases in the order of the particle ids")
    ap.add_argument("--mesh", default="spherical", choices=["spherical", "flat"])
    ap.add_argument("--delayed", action="store_true", help="releases at three different times")
    ap.add_argument("--halo", type=int, default=3)
    ap.add_argument("--max-dt", type=float, default=3600.0, help="RK45_max_dt")
    a = ap.parse_args()
    world, n = a.world, a.particles
    if a.kernel != "rk4_3d" or a.interp != "linear" or a.mesh != "spherical" or a.delayed or a.f32_coords or a.ordered_releases:
        return kernel_case(a)
    f = bench.c2_field(nx=120, ny=60, nz=12, nt=a.nt)
    f["U"] *= np.float32(40.0)
    f["V"] *= np.float32(40.0)
    rng = np.random.default_rng(7)
    x, y, z = rng.uniform(-175, 175, n), rng.uniform(-70, 70, n), rng.uniform(5, 5000, n)
    dt = -a.dt if a.backward else a.dt
    t_start = float(f["times"][-1]) if a.backward else 0.0
    # staggered releases: particles wait at different times, the lock-step slide has to serve the earliest first
    t = t_start + np.sign(dt) * rng.choice([0.0, 7200.0, 100800.0], n) if a.time_window else np.full(n, t_start)
    endtime = t_start + np.sign(dt) * a.runtime
    kernels = [pb.AdvectionRK4_3D, pb.DeleteParticle]
    full = create_particle_data(nparticles=n, ngrids=1, initial=dict(x=x, y=y, z=z, t=t, particle_id=np.arange(n)))
    slabs = [D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"],
                                  mesh="spherical", rank=r, world=world, halo_cells=a.halo, device=0,
                                  time_window=a.time_window or None)
             for r in range(world)]  # fmt: skip
    bases = [s.engine.migrate_p2p_init(a.inbox or n)[1] for s in slabs]
    for s in slabs:
        s.engine.migrate_p2p_connect(local_bases=bases)
        s.p2p = True
    thread_ranks.serialise_engine_calls()
    res = thread_ranks.run_ranks(world, lambda r, dist: D.execute_decomposed(slabs[r], D.shard_particles(full, r, world), kernels, dt,
                                                                             endtime, dist))  # fmt: skip
    outs, stats = [o for o, _ in res], [s for _, s in res]
    merged = {k: np.concatenate([o[k] for o in outs], axis=0) for k in outs[0]}
    order = np.argsort(merged["particle_id"], kind="stable")
    merged = {k: v[order] for k, v in merged.items()}
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"], W=f["W"], mesh="spherical")
    ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=t, device=0)
    ps.execute(kernels, dt=dt, endtime=endtime)
    ref = ps._data
    ok = True
    for k in ("particle_id", "state", "t", "ei", "x", "y", "z"):
        same = merged[k].shape == ref[k].shape and np.array_equal(merged[k], ref[k])
        ok &= same
        if not same:
            print(f"MISMATCH {k}: {merged[k].shape} vs {ref[k].shape}")
    migrated = sum(s["migrated"] for s in stats)
    print(f"decomposed({world} thread ranks): {len(ref['x'])} survivors, {migrated} migrations, rounds={stats[0]['rounds']}, "
          f"transport={stats[0]['transport']}" + (f", time window {a.time_window} of {a.nt} levels" if a.time_window else "")
          + f" -> {'PASS bit-exact' if ok else 'FAIL'}")  # fmt: skip
    return 0 if ok else 1


def kernel_case(a):
    case = decomposed_kernels.make_case(a.kernel, mesh=a.mesh, n=a.particles, nt=a.nt, runtime=a.runtime, backward=a.backward,
                                        delayed=a.delayed or bool(a.time_window), max_dt=a.max_dt, interp=a.interp,
                                        f32_coords=a.f32_coords, dt=a.dt, ordered=a.ordered_releases)  # fmt: skip
    world, n = a.world, a.particles
    slabs = [decomposed_kernels.decomposed_fieldset(case, r, world, halo=a.halo, time_window=a.time_window or None) for r in range(world)]
    bases = [s.engine.migrate_p2p_init(a.inbox or n)[1] for s in slabs]
    for s in slabs:
        s.engine.migrate_p2p_connect(local_bases=bases)
        s.p2p = True
    thread_ranks.serialise_engine_calls()
    full = case["full"]
    res = thread_ranks.run_ranks(world, lambda r, dist: D.execute_decomposed(slabs[r], D.shard_particles(full, r, world), case["kernels"],
                                                                             case["dt"], case["endtime"], dist, seed=case["seed"]))  # fmt: skip
    outs, stats = [o for o, _ in res], [s for _, s in res]
    merged = {k: np.concatenate([o[k] for o in outs], axis=0) for k in outs[0]}
    ref = decomposed_kernels.reference(case)
    ok, msgs = decomposed_kernels.compare(merged, ref, a.kernel)
    print("\n".join(msgs))
    migrated = sum(s["migrated"] for s in stats)
    print(f"decomposed {a.kernel} ({a.interp}, {world} thread ranks, {a.mesh}{', backward' if a.backward else ''}): {len(ref['x'])} of {n} left, "
          f"{migrated} migrations, rounds={stats[0]['rounds']}, transport={stats[0]['transport']}"
          + (f", time window {a.time_window} of {a.nt} levels" if a.time_window else "") + f" -> {'PASS bit-exact' if ok else 'FAIL'}")  # fmt: skip
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
