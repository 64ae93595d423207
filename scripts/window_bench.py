#!/usr/bin/env python
"""Time-slab streaming (``FieldSet.from_arrays(..., time_window=W)``) against the fully resident field, per kernel list.

The field is config 2's shape (1/4 deg x 50 levels, float32, spherical) with ``--levels`` daily time levels; the windowed
FieldSet keeps ``--window`` of them in HBM and streams the others in as the particles' clock crosses them.  Three lists:
  rk45   [AdvectionRK45]                                     one launch per window slide (pb_advect_rk45)
  m1     [AdvectionDiffusionM1, DeleteParticle]             one launch per window slide (pb_advect_diffusion)
  user   [AdvectionRK4_3D, <user kernel sampling UV and P>, DeleteParticle]  step by step: the host drives the loop
  tracer [AdvectionRK4_3D, <user kernel sampling a time-varying float32 T>, DeleteParticle]  step by step; the windowed run
         streams T through the velocity window too (``add_field(..., time_window=W)``), the resident one uploads it whole
Every list runs resident and windowed alternately, ``--repeats`` times each, from the same particles; the time of one
``ParticleSet.execute`` is measured on the wall clock around the call (it returns after the result is back on the host, so
the GPU work is done), after the engine's first use has uploaded the resident field.  ``kernel_ms`` is the CUDA-event time
of the device launches of the last Kernel.execute (RK45, M1).  ``field_hbm_bytes`` is what the engine allocates for the field
buffers, from the shapes: whole fields, or a ring of ``--window`` + 1 levels per windowed field.  The windowed and resident
results are compared bit for bit.  Prints one JSON line per list, the card's name and power limit first.

  python scripts/window_bench.py [--particles 1000000] [--user-particles 100000] [--days 5] [--repeats 2]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the config-2 field generator)
import parcels_b200 as pb  # noqa: E402
from parcels_b200.fieldset import Field  # noqa: E402

DAY = 86400.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()  # fmt: skip
        name, power = (s.strip() for s in out.split(",", 1))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 -- the numbers are still numbers; say that the card is unknown
        return {"gpu": None, "power_limit": None, "error": f"{type(e).__name__}: {e}"}


def sample(particles, fieldset):
    """A user kernel as the reference's users write them: the velocity at the end of the step and a scalar field."""
    _, v1 = fieldset.UV[particles.t + particles.dt, particles.z, particles.y, particles.x]
    particles.v1 = v1
    particles.p = fieldset.P[particles]


def sample_temperature(particles, fieldset):
    particles.temp = fieldset.T[particles]


def make_fieldset(f, kind, window):
    fs = pb.FieldSet.from_arrays(lon=f["lon"], lat=f["lat"], depth=f["depth"], time=f["times"], U=f["U"], V=f["V"],
                                 W=f["W"] if kind in ("user", "tracer") else None, mesh="spherical", time_window=window)  # fmt: skip
    nz, ny, nx = f["U"].shape[1:]
    if kind == "rk45":
        fs.add_context("RK45_tol", 10.0)
        fs.add_context("RK45_min_dt", 60.0)
        fs.add_context("RK45_max_dt", 3600.0)
    elif kind == "m1":
        x = np.linspace(0.0, 1.0, nx, dtype=np.float32)[None, None, None, :]
        y = np.linspace(0.0, 1.0, ny, dtype=np.float32)[None, None, :, None]
        fs.add_field("Kh_zonal", np.broadcast_to(np.float32(20.0) + np.float32(10.0) * x * y, (1, nz, ny, nx)).copy())
        fs.add_field("Kh_meridional", np.broadcast_to(np.float32(15.0) + np.float32(5.0) * y, (1, nz, ny, nx)).copy())
        fs.add_context("dres", float(f["lon"][1] - f["lon"][0]) / 10)
    elif kind == "tracer":
        fs.add_field("T", f["T"], time_window=window)
    else:
        fs.add_field("P", np.ascontiguousarray(f["U"][:1]) + np.float32(1.0))
    return fs


def field_hbm_bytes(fs):
    """HBM the engine allocates for the field buffers, from the shapes: a whole field, or a ring of time_window + 1 levels."""
    total = 0
    for fld in fs.fields.values():
        if isinstance(fld, Field) and fld.interp_method != "constant":
            level = int(np.prod(fld.data.shape[1:])) * np.dtype(fld.data.dtype).itemsize
            total += level * (fs.time_window + 1 if fld._windowed else fld.data.shape[0])
    return total


PCLASS = {
    "rk45": pb.Particle.add_variable(pb.Variable("next_dt", dtype=np.float32, initial=0)),
    "m1": pb.Particle,
    "user": pb.Particle.add_variable([pb.Variable("v1", dtype=np.float64), pb.Variable("p", dtype=np.float64)]),
    "tracer": pb.Particle.add_variable(pb.Variable("temp", dtype=np.float64)),
}
KERNELS = {"rk45": [pb.AdvectionRK45], "m1": [pb.AdvectionDiffusionM1, pb.DeleteParticle],
           "user": [pb.AdvectionRK4_3D, sample, pb.DeleteParticle], "tracer": [pb.AdvectionRK4_3D, sample_temperature, pb.DeleteParticle]}
DT = {"rk45": 600.0, "m1": 600.0, "user": 1800.0, "tracer": 1800.0}
VARS = {"rk45": (), "m1": (), "user": ("p",), "tracer": ("temp",)}


def run(f, kind, window, x, y, z, days):
    fs = make_fieldset(f, kind, window)
    fs.engine(0)  # resident: the field upload, not timed
    ps = pb.ParticleSet(fs, pclass=PCLASS[kind], x=x, y=y, z=z, t=np.zeros(len(x)), seed=11)
    t0 = time.perf_counter()
    ps.execute(KERNELS[kind], dt=DT[kind], runtime=days * DAY)
    sec = time.perf_counter() - t0
    rep = ps.last_report or {}
    out = {k: np.array(ps._data[k]) for k in ("x", "y", "z", "t", *VARS[kind])}
    hbm = field_hbm_bytes(fs)
    fs.release()
    return sec, float(rep.get("kernel_ms", float("nan"))), out, hbm


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--particles", type=int, default=1_000_000)
    ap.add_argument("--user-particles", type=int, default=100_000)
    ap.add_argument("--levels", type=int, default=8)
    ap.add_argument("--window", type=int, default=3)
    ap.add_argument("--days", type=float, default=5.0)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--lists", default="rk45,m1,user,tracer")
    ap.add_argument("--small", action="store_true", help="a 1/4-size field (a quick check of the script, not a measurement)")
    a = ap.parse_args()
    print(json.dumps({"card": card(), "levels": a.levels, "time_window": a.window, "days": a.days}), flush=True)
    f = bench.c2_field(nx=360, ny=180, nz=10, nt=a.levels) if a.small else bench.c2_field(nt=a.levels)
    f["times"] = np.arange(a.levels) * DAY
    # a temperature-like tracer that changes from day to day
    f["T"] = (np.float32(0.5) * f["U"] + np.float32(10.0) + np.arange(a.levels, dtype=np.float32)[:, None, None, None]).astype(np.float32)
    rng = np.random.default_rng(3)
    for kind in a.lists.split(","):
        n = a.user_particles if kind in ("user", "tracer") else a.particles
        x, y, z = rng.uniform(-170, 170, n), rng.uniform(-70, 70, n), rng.uniform(5, 5000, n)
        times = {"resident": [], "windowed": []}
        kms = {"resident": [], "windowed": []}
        hbm = {}
        same = True
        for _ in range(a.repeats):
            res = {}
            for label, window in (("resident", None), ("windowed", a.window)):
                sec, ms, res[label], hbm[label] = run(f, kind, window, x, y, z, a.days)
                times[label].append(sec)
                kms[label].append(ms)
            same = same and all(np.array_equal(res["resident"][k], res["windowed"][k]) for k in res["resident"])
        r, w = min(times["resident"]), min(times["windowed"])
        print(json.dumps({"list": kind, "particles": n, "dt": DT[kind], "resident_s": times["resident"], "windowed_s": times["windowed"],
                          "resident_kernel_ms": kms["resident"], "windowed_kernel_ms": kms["windowed"],
                          "windowed_over_resident": round(w / r, 3), "field_hbm_bytes": hbm, "bit_identical": bool(same)}),
              flush=True)  # fmt: skip


if __name__ == "__main__":
    main()
