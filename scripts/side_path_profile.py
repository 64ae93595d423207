"""Where the headline A-grid RK4 kernel (afast.cu) spends its time: the cell-change side path versus the straight-line path.
   python scripts/side_path_profile.py [--workload ns] [--steps 3] [--warmup 1]
Builds the -DPB_SIDE_PROFILE variant of the library (clock64 counters per warp-evaluation; the default build has none), runs the
device-resident arm of one bench.py workload with it and prints one JSON line of per-launch figures.  The counters cost time of
their own: the shares are the thing to read, the profiled kernel time is printed beside the default build's for scale."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = "sideprof"
LIB = os.path.join(ROOT, "parcels_b200", "lib", f"libparcels_b200_{TAG}.so")
NAMES = ["warp_evals", "miss_evals", "eval_cycles", "miss_eval_cycles", "side_cycles", "side_lane_entries"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ns")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--particles", type=int, default=None)
    ap.add_argument("--rebuild", action="store_true")
    a = ap.parse_args()
    if a.rebuild or not os.path.exists(LIB):
        subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "build_variant.py"), TAG, "afast.cu:-DPB_SIDE_PROFILE"], check=True)
    os.environ["PB_LIB"] = LIB
    sys.path.insert(0, ROOT)
    import bench
    from parcels_b200 import _lib

    lib = _lib.load()
    buf = (ctypes.c_ulonglong * len(NAMES))()
    args = types.SimpleNamespace(particles=a.particles, sorted=False, pipeline=-1)
    out = bench.run_gpu_workload(args, a.workload, rank=0, local_rank=0, world=1, dist=None, steps=a.steps, warmup=a.warmup,
                                 with_e2e=False, with_cpu=False)  # fmt: skip
    _lib.check(lib.pb_side_profile_read(buf))
    launches = a.steps + a.warmup  # every launch restores the same snapshot: the counters are the same launch after launch
    c = {k: buf[i] / launches for i, k in enumerate(NAMES)}
    hit_evals = c["warp_evals"] - c["miss_evals"]
    hit_avg = (c["eval_cycles"] - c["miss_eval_cycles"]) / max(hit_evals, 1)
    miss_avg = c["miss_eval_cycles"] / max(c["miss_evals"], 1)
    res = {
        "workload": a.workload, "per_launch": c,
        "refills": out["measured"]["corner_cache_refills_per_launch"],
        "profiled_kernel_ms": out["measured"]["kernel_ms_per_launch"],
        "miss_eval_fraction": c["miss_evals"] / max(c["warp_evals"], 1),
        "cycles_per_hit_eval": hit_avg, "cycles_per_miss_eval": miss_avg,
        # warp time inside side_path / warp time inside evaluations
        "side_path_share": c["side_cycles"] / max(c["eval_cycles"], 1),
        # what the misses add over a hit evaluation / warp time inside evaluations
        "miss_excess_share": (c["miss_eval_cycles"] - c["miss_evals"] * hit_avg) / max(c["eval_cycles"], 1),
    }  # fmt: skip
    print(json.dumps(res))


if __name__ == "__main__":
    main()
