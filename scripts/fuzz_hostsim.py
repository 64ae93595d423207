"""Differential fuzzing of the kernel SOURCES (compiled for the host, oracle/hostsim) against the oracle on random
configurations: dtypes, meshes, dimensionality, schemes, release patterns, time direction, error handling.
Run:  PB_LIB=oracle/_build/hostsim/libparcels_b200_hostsim.so PB_HOSTSIM_TEST=1 python scripts/fuzz_hostsim.py [n_cases] [seed] [--curv]

Rectilinear cases (A-grid linear / slip / nearest, rectilinear C-grid) must agree exactly (flat) or to 4 float32 ulp (spherical).
--curv adds random curvilinear meshes: informational only -- on arbitrary meshes the reference's closed-form bilinear inverse
depends on its BLAS (FMA, summation order, batch size; DESIGN.md waiver 6), so a few-ulp scatter and the odd edge-grazing
cell flip are expected there; the parity tests use meshes on which the reference itself is reproducible."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import cases
from engine_run import run_engine, ulp_diff_f32
from oracle_run import run_oracle

ERR_NAME = {60: "FieldOutOfBoundError", 61: "FieldOutOfBoundSurfaceError", 70: "OutsideTimeInterval", 51: "FieldInterpolationError",
            52: "GridSearchingError", 50: "GeneralError"}


CURV = "--curv" in sys.argv


def random_curv_spec(rng):
    """curvilinear C-grid cases (tests/cases.py kind="curv"): hint + neighbour + spatial-hash search, CGrid_Velocity"""
    three = rng.random() < 0.4
    mesh = str(rng.choice(["flat", "spherical"]))
    nt = int(rng.choice([2, 3]))
    dt = float(rng.choice([60.0, 300.0, 900.0])) * (1 if rng.random() < 0.8 else -1)
    nsteps = int(rng.integers(1, 10))
    tstep = abs(dt) * nsteps / (nt - 1) * float(rng.choice([1.0, 1.5]))
    spec = dict(seed=int(rng.integers(1, 10**6)), kind="curv", cdtype=str(rng.choice(["f4", "f8"])), mesh=mesh, nx=int(rng.integers(8, 40)),
                ny=int(rng.integers(8, 30)), nz=int(rng.integers(3, 7)) if three else 1, nt=nt, tstep=tstep, n=int(rng.integers(1, 150)),
                kernels=["AdvectionRK4_3D" if three else str(rng.choice(["AdvectionRK4", "AdvectionRK2", "AdvectionEE"]))], dt=dt,
                segments=[dict(runtime=abs(dt) * nsteps)], delete=True,
                umax=float(rng.choice([0.5, 1.5])) if mesh == "flat" else float(rng.choice([5.0, 20.0])))  # fmt: skip
    return spec


def random_spec(rng):
    if CURV and rng.random() < 0.25:
        return random_curv_spec(rng)
    three = rng.random() < 0.5
    scheme = rng.choice(["AdvectionRK4_3D", "AdvectionRK2_3D"]) if three else rng.choice(["AdvectionRK4", "AdvectionRK2", "AdvectionEE"])
    mesh = rng.choice(["flat", "spherical"])
    nt = int(rng.choice([1, 2, 3, 5]))
    interp = rng.choice(["linear", "linear", "freeslip", "partialslip", "nearest", "cgrid_velocity"])
    if interp == "nearest" and not three:  # the reference's XNearest_Velocity wrapper samples U, V AND W
        interp = "linear"
    nz = int(rng.integers(2, 8))
    no_depth = (not three) and rng.random() < 0.3
    tstep = float(rng.choice([200.0, 1000.0, 3600.0]))
    dt = float(rng.choice([10.0, 50.0, 300.0, 600.0])) * (1 if rng.random() < 0.75 else -1)
    nsteps = int(rng.integers(1, 12))
    runtime = abs(dt) * nsteps * float(rng.choice([1.0, 1.0, 0.83]))  # sometimes a clamped last step
    tmax = tstep * (nt - 1)
    spec = dict(seed=int(rng.integers(1, 10**6)), kind="smooth", cdtype=str(rng.choice(["f4", "f8"])), ddtype=str(rng.choice(["f4", "f8"])),
                mesh=str(mesh), nx=int(rng.integers(5, 30)), ny=int(rng.integers(5, 25)), nz=1 if no_depth else nz, nt=nt, tstep=tstep,
                n=int(rng.integers(1, 200)), kernels=[str(scheme)], dt=dt, segments=[dict(runtime=runtime)],
                delete=bool(rng.random() < 0.7), margin=float(rng.choice([-0.03, 0.0, 0.05, 0.2])),
                umax=float(rng.choice([0.5, 3.0, 10.0 if mesh == "spherical" else 4.0])), wmax=float(rng.choice([1e-3, 0.05])))  # fmt: skip
    if interp != "linear":
        spec["interp"] = str(interp)
    if interp in ("freeslip", "partialslip"):
        spec["land"] = True
    if no_depth:
        spec["no_depth"] = True
    if nt > 1:
        runtime = min(runtime, 0.9 * tmax)
        spec["segments"] = [dict(runtime=runtime)]
        if dt > 0:
            lo, hi = 0.0, max(tmax - runtime - abs(dt), 0.0)
        else:
            lo, hi = min(runtime + abs(dt), tmax), tmax
        spec["release"] = ("const", float(rng.choice([lo, hi, 0.5 * (lo + hi)]))) if (rng.random() < 0.6 or hi - lo < 2) else ("uniform", lo, hi)
    if rng.random() < 0.25:
        spec["segments"] = [dict(runtime=runtime * 0.5), dict(runtime=runtime * 0.5)]
    return spec


def inject_boundary_cases(rng, spec, c):
    """Releases on nodes / domain edges / depth levels, non-finite coordinates, releases just outside the time interval, repeated
    releases on the first time level (in place, on the case dict ``c``)."""
    n = len(c["x"])
    if spec["kind"] == "smooth" and rng.random() < 0.4 and n >= 4:
        # boundary cases: releases exactly on nodes, on the domain edges, on depth levels; a few non-finite coordinates
        lon, lat = np.asarray(c["lon"], dtype=np.float64), np.asarray(c["lat"], dtype=np.float64)
        pick = rng.integers(0, n, 4)
        c["x"][pick[0]], c["y"][pick[0]] = lon[rng.integers(0, len(lon))], lat[rng.integers(0, len(lat))]
        c["x"][pick[1]] = lon[[0, -1][rng.integers(0, 2)]]
        c["y"][pick[2]] = lat[[0, -1][rng.integers(0, 2)]]
        if c["depth"] is not None:
            c["z"][pick[3]] = np.asarray(c["depth"], dtype=np.float64)[rng.integers(0, len(c["depth"]))]
        if rng.random() < 0.3:
            c[str(rng.choice(list("xyz")))][rng.integers(0, n)] = rng.choice([np.nan, np.inf, -np.inf])
    if spec["kind"] == "smooth" and spec["nt"] > 1 and rng.random() < 0.3:
        # a few releases just outside the fields' time interval: their first sample raises OutsideTimeInterval, which flags
        # (with DeleteParticle: deletes) the reference's WHOLE evaluated view of that iteration (field.py:31-44)
        runtime0 = spec["segments"][0]["runtime"]
        delta = float(rng.uniform(0.05, 0.95)) * min(runtime0, 2 * abs(spec["dt"]))
        pick = rng.integers(0, n, int(rng.integers(1, 3)))
        c["t"] = np.asarray(c["t"], dtype=np.float64).copy()
        c["t"][pick] = -delta if spec["dt"] > 0 else spec["tstep"] * (spec["nt"] - 1) + delta
    elif spec["kind"] == "smooth" and spec["nt"] > 1 and spec["dt"] > 0 and rng.random() < 0.3:
        # repeated release: some particles exactly on the first time level (tau == 0), the others later -- the reference's
        # batch-level lenT then promotes the first-level particles' first sample (float32 grids)
        later = float(rng.choice([0.5, 1.0, 2.0])) * spec["dt"]
        c["t"] = np.where(rng.random(n) < 0.5, 0.0, later)


def compare_with_reference(spec, c, da, ea, db, eb):
    """Differences of the engine's particle data ``db`` (raised ``eb``) from the reference's ``da`` (raised ``ea``) after the same
    trajectory case: ids / states / times / cells / dt identical, positions bit-exact on flat meshes and within a few float32 ulp
    on spherical ones; curvilinear meshes as stated below."""
    msg = []
    if ea != eb:
        msg.append(f"raised {eb!r} vs the reference's {ea!r}")
    if len(da["x"]) != len(db["x"]):
        msg.append(f"survivors {len(db['x'])} vs {len(da['x'])}")
    else:
        skip_xyz = ea.endswith("OutsideTimeInterval")  # DESIGN.md waiver 2: dx / ei of the aborted step
        if spec["kind"] == "curv" and spec["mesh"] == "flat":
            # the reference's flat-mesh bilinear inverse is ill-conditioned on random near-parallelogram cells and changes with
            # its own batch size (DESIGN.md waiver 6): only who is left, in which state and at what time is compared
            for key in ("particle_id", "state", "t"):
                if not np.array_equal(da[key], db[key]):
                    msg.append(key)
            return msg
        if ea.endswith("IndexError"):
            return []  # the reference's own failure (3-D slip, no particle below the first level: DESIGN.md waiver 1)
        for key in ("particle_id", "state", "t") + (() if skip_xyz else ("ei", "dt")):
            if not np.array_equal(da[key], db[key]):
                msg.append(key)
        if not skip_xyz:
            for key in "xyz":
                floor = 0.01 * float(np.abs(np.asarray(c[key])).max()) or None
                u = ulp_diff_f32(db[key], da[key], floor=floor)
                tol = 0 if spec["mesh"] == "flat" else 4
                if spec["kind"] == "curv":
                    # curvilinear C-grids (hint + neighbour + spatial-hash search) on SPHERICAL random meshes: cells, states and
                    # times identical; positions within 1e-4 of a cell -- the set is fresh, so the reference computes its first
                    # evaluation with float32-TYPED barycentric coordinates (DESIGN.md waiver 4: 1e-7 relative) and the C-grid's
                    # face discontinuities grow that seed (measured over 300 random meshes: <= 2 float32 ulp with float64
                    # nodes, <= 11 with float32 nodes, rarely more).  FLAT random meshes: see below.
                    cell = float(np.abs(np.diff(np.asarray(c["lon"], dtype=np.float64), axis=1)).mean())
                    if len(da[key]) and float(np.abs(db[key].astype(np.float64) - da[key].astype(np.float64)).max()) > 1e-4 * cell:
                        msg.append(f"{key}: {float(np.abs(db[key].astype(np.float64) - da[key].astype(np.float64)).max()) / cell:.2e} cells")
                    continue
                if spec["mesh"] == "flat" and spec.get("interp") == "cgrid_velocity":
                    tol = 0.5  # (a batch of exactly one evaluated particle: DESIGN.md waiver 8)
                if spec["mesh"] == "spherical" and spec.get("interp") == "cgrid_velocity" and spec["cdtype"] == "f4":
                    tol = 64  # (float32 edge lengths with a float32 cos, main() below)
                if u.size and u.max() > tol:
                    msg.append(f"{key}: {u.max():.1f} ulp (tol {tol})")
    return msg


def main():
    argv = [a for a in sys.argv[1:] if not a.startswith("--")]
    n_cases = int(argv[0]) if argv else 100
    rng = np.random.default_rng(int(argv[1]) if len(argv) > 1 else 0)
    bad = 0
    for k in range(n_cases):
        spec = random_spec(rng)
        try:
            c = cases.build(spec)
            inject_boundary_cases(rng, spec, c)
            ps, err = run_engine(c)
            pd, oerr = run_oracle(c)
        except Exception as e:  # noqa: BLE001
            if isinstance(e, IndexError) and spec.get("interp") in ("freeslip", "partialslip") and spec["kernels"][0].endswith("_3D"):
                # the reference's own failure (DESIGN.md waiver 1, last paragraph): a 3-D slip evaluation of a batch with no particle
                # below the first depth level indexes a depth level that was not gathered (_xinterpolators.py:460-470) -- the oracle
                # restates it, the engine returns the value
                print(f"[{k}] known: the reference raises IndexError here (3-D slip, lenZ == 1)")
                continue
            print(f"[{k}] EXC {type(e).__name__}: {e}\n    spec={spec}")
            bad += 1
            continue
        d = ps._data
        msg = []
        if err != (ERR_NAME.get(oerr, str(oerr)) if oerr else ""):
            msg.append(f"error {err!r} vs oracle {oerr}")
        if len(d["x"]) != len(pd["x"]):
            msg.append(f"survivors {len(d['x'])} vs {len(pd['x'])}")
        else:
            skip_xyz = err == "OutsideTimeInterval"  # waiver 2: dx / ei of the aborted step
            for key in ("particle_id", "state", "t") + (() if skip_xyz else ("ei", "dt")):
                if not np.array_equal(d[key], pd[key]):
                    msg.append(f"{key} differs at {np.flatnonzero((d[key] != pd[key]).reshape(len(d['x']), -1).any(axis=1))[:5]}")
            if not skip_xyz:
                for key in "xyz":
                    floor = 0.01 * float(np.abs(np.asarray(c[key])).max()) or None
                    u = ulp_diff_f32(d[key], pd[key], floor=floor)
                    tol = 8 if spec["kind"] == "curv" else (0 if spec["mesh"] == "flat" else 4)
                    if spec["mesh"] == "spherical" and spec.get("interp") == "cgrid_velocity" and spec["cdtype"] == "f4":
                        tol = 64  # float32 edge lengths with a float32 cos: one ulp of cosf (libm vs NumPy's SIMD cos) is 6e-8 of every flux
                    if u.size and u.max() > tol:
                        msg.append(f"{key}: {u.max():.1f} ulp (tol {tol})")
        if msg:
            bad += 1
            print(f"[{k}] MISMATCH {'; '.join(msg)}\n    spec={spec}")
    print(f"{n_cases} cases, {bad} with differences")


if __name__ == "__main__":
    main()
