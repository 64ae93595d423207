"""Differential fuzzing of the HOST LAYER's bookkeeping (which copy of the particle set is current -- host arrays, device arrays,
a lazily resident set -- across execute() calls, edits, removals and additions): random SEQUENCES of public-API operations on one
ParticleSet, mirrored on the oracle's particle dict, compared after every execute().  Rectilinear flat A-grids, where the kernels are
bit-exact, so any difference is the bookkeeping's.
  ops: execute (random kernel list, runtime, with or without an output file between the intervals; also WITHOUT the DeleteParticle
       handler: same exception, same states, the set usable afterwards; and with a user Python kernel + error handler in the list:
       loop control on the host), in-place edits through the
       arrays the attributes return, `pset[i].x = ...` / `pset[mask].y = ...` views, `pset.z = ...`, remove_indices, add(),
       plain reads (len, attribute access), a second ParticleSet on the same FieldSet executing in between.
Run:  PB_LIB=oracle/_build/hostsim/libparcels_b200_hostsim.so PB_HOSTSIM_TEST=1 python scripts/fuzz_hostsim_api.py [n] [seed]
      [--windowed-lists]: on time-windowed fieldsets also run the lists without the handler and the lists with user kernels"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import warnings
import numpy as np
import cases
import parcels_b200 as pb
from engine_run import make_fieldset
from oracle import parcels_oracle as po
from oracle_run import oracle_fieldset

warnings.simplefilter("ignore")
ERR_NAME = {60: "FieldOutOfBoundError", 61: "FieldOutOfBoundSurfaceError", 70: "OutsideTimeInterval", 51: "FieldInterpolationError",
            52: "GridSearchingError", 50: "GeneralError"}
VERBOSE = os.environ.get("FUZZ_VERBOSE") == "1"
WINDOWED_LISTS = "--windowed-lists" in sys.argv
KEYS = ("particle_id", "state", "t", "ei", "x", "y", "z", "dx", "dy", "dz", "dt")


class Recorder:
    """In-memory output file: the rows the product hands to ParticleFile.write at every output time (same column source)."""

    def __init__(self, outputdt):
        self.outputdt, self.rows = outputdt, []

    def write(self, pset, t):
        cols, _ = pset._output_columns(float(t), ["t", "z", "y", "x", "particle_id"])
        self.rows.append((float(t), {k: np.array(v) for k, v in cols.items()}))


def oracle_rows(rows):
    def on_output(pdata, t):
        sel = po.to_write_particles(pdata, t)
        rows.append((float(t), {k: pdata[k][sel].copy() for k in ("t", "z", "y", "x", "particle_id")}))

    return on_output


def same_rows(a, b):
    return len(a) == len(b) and all(ta == tb and all(np.array_equal(ca[k], cb[k]) for k in ca) for (ta, ca), (tb, cb) in zip(a, b))


def compare(ps, pd, tag):
    d = ps._data
    if len(d["x"]) != len(pd["x"]):
        return [f"{tag}: {len(d['x'])} particles vs oracle {len(pd['x'])}"]
    return [f"{tag}: {k}" for k in KEYS if not np.array_equal(d[k], pd[k], equal_nan=True)]


def one_case(rng):
    three = bool(rng.random() < 0.5)
    nt = int(rng.choice([1, 3, 4]))
    tstep = 3600.0
    dt = float(rng.choice([300.0, 600.0]))
    spec = dict(seed=int(rng.integers(1, 10**6)), kind="smooth", cdtype=str(rng.choice(["f4", "f8"])), ddtype=str(rng.choice(["f4", "f8"])),
                mesh="flat", nx=int(rng.integers(6, 24)), ny=int(rng.integers(6, 20)), nz=int(rng.integers(2, 6)), nt=nt, tstep=tstep,
                n=int(rng.integers(2, 120)), kernels=["AdvectionRK4_3D" if three else "AdvectionRK4"], dt=dt, segments=[dict(runtime=dt)],
                delete=True, margin=float(rng.choice([0.0, 0.1, 0.25])), umax=float(rng.choice([0.5, 3.0])), wmax=1e-3)  # fmt: skip
    if nt > 1:
        spec["release"] = ("const", 0.0)
    c = cases.build(spec)
    # time-slab streaming in a quarter of the cases with a time axis: 2 or 3 of the levels resident, slid as the set's clock advances
    # across the calls of the sequence (without --windowed-lists only the lists with the DeleteParticle handler run there)
    window = int(rng.choice([2, 3])) if (nt == 4 and rng.random() < 0.4) else None
    if window:
        fs = pb.FieldSet.from_arrays(lon=c["lon"], lat=c["lat"], depth=c["depth"], time=c["times"], U=c["U"], V=c["V"], W=c["W"],
                                     mesh=c["mesh"], time_window=window)  # fmt: skip
    else:
        fs = make_fieldset(c)
    ofs = oracle_fieldset(c)
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    # the paths large sets take -- chunked host-array pipeline (pb_advect_host), deferred `particles.dt` fill, compacted download
    # after deletions -- at these sizes: lower the set's threshold in half of the cases
    knobs = f"[time_window {window}] " if window else ""
    if rng.random() < 0.5:
        ps.PIPELINE_MIN_PARTICLES = int(rng.choice([1, 4, 16]))
        ps.pipeline_chunks = int(rng.choice([2, 3, 8]))
        knobs = f"[pipeline >= {ps.PIPELINE_MIN_PARTICLES} x{ps.pipeline_chunks}] "
    if rng.random() < 0.3:
        ps.eager_host = True
        knobs += "[eager_host] "
    pd = po.create_particle_data(c["x"], c["y"], c["z"], c["t"], ngrids=ofs.ngrids)
    other = None  # a second set on the same FieldSet (the engine keeps ONE resident set per device: ownership hand-over)
    t_end = tstep * (nt - 1) if nt > 1 else np.inf
    names2 = ["AdvectionRK4", "AdvectionRK2", "AdvectionEE"]
    names3 = ["AdvectionRK4_3D", "AdvectionRK2_3D"] + names2
    log, msg = [], []
    for step in range(int(rng.integers(3, 9))):
        op = str(rng.choice(["exec", "exec", "exec", "exec_raise", "exec_mixed", "edit", "view", "setattr", "remove", "add", "read", "other"]))
        n = len(pd["x"])
        if n == 0:
            break
        if window and op in ("exec_raise", "exec_mixed") and not WINDOWED_LISTS:
            continue
        if op == "exec":
            name = str(rng.choice(names3 if three else names2))
            nsteps = int(rng.integers(1, 6))
            t_now = float(np.nanmax(pd["t"])) if n else 0.0
            if t_now + nsteps * dt > t_end:
                continue
            kw = {}
            if rng.random() < 0.4:
                rec = Recorder(float(rng.choice([dt, 2 * dt])))
                kw["output_file"] = rec
            log.append(f"exec {name} x{nsteps}{' +output' if kw else ''}")
            ps.execute([getattr(pb, name), pb.DeleteParticle], dt=dt, runtime=nsteps * dt, **kw)
            okw, orows = {}, []
            if kw:
                okw = dict(outputdt=rec.outputdt, on_output=oracle_rows(orows))
            po.pset_execute(pd, ofs, [getattr(po, name), po.DeleteOnError], dt, runtime=nsteps * dt, **okw)
            if kw and not same_rows(rec.rows, orows):
                msg.append(f"step {step}: output rows differ ({[(t, len(c_['x'])) for t, c_ in rec.rows]} vs {[(t, len(c_['x'])) for t, c_ in orows]})")
            if rng.random() < 0.5:  # sometimes look right away, sometimes leave the set where it is (lazy residency)
                msg += compare(ps, pd, f"step {step} ({log[-1]})")
        elif op == "exec_mixed":
            # a user Python kernel and a user error handler in the list: loop control on the host, the built-in on the device
            name = str(rng.choice(names3 if three else names2))
            nsteps = int(rng.integers(1, 5))
            if float(np.nanmax(pd["t"])) + nsteps * dt > t_end:
                continue
            drift = float(rng.choice([0.0, 0.01, 0.25])) * float(spec["umax"])

            def Drift(particles, fieldset):
                particles.dy += drift * particles.dt

            def DeleteErr(particles, fieldset):
                particles[particles.state >= 50].state = 30

            def ODrift(p, fs_):
                p.dy = p.dy + drift * p.dt

            log.append(f"exec [{name}, Drift({drift}), DeleteErr] x{nsteps}")
            ps.execute([getattr(pb, name), Drift, DeleteErr], dt=dt, runtime=nsteps * dt)
            po.pset_execute(pd, ofs, [getattr(po, name), ODrift, po.DeleteOnError], dt, runtime=nsteps * dt)
            if rng.random() < 0.5:
                msg += compare(ps, pd, f"step {step} ({log[-1]})")
        elif op == "exec_raise":
            # no DeleteParticle handler: a particle that leaves the domain stops the whole set at the end of that iteration with the
            # reference's exception (kernel.py:239-245) -- the engine replays up to that iteration; the set must be usable afterwards
            name = str(rng.choice(names3 if three else names2))
            nsteps = int(rng.integers(1, 6))
            if float(np.nanmax(pd["t"])) + nsteps * dt > t_end:
                continue
            err, oerr = "", None
            try:
                ps.execute([getattr(pb, name)], dt=dt, runtime=nsteps * dt)
            except RuntimeError as e:
                if type(e).__module__.startswith("parcels_b200._lib"):
                    raise
                err = type(e).__name__
            try:
                po.pset_execute(pd, ofs, [getattr(po, name)], dt, runtime=nsteps * dt)
            except po.OracleParticleError as e:
                oerr = e.code
            log.append(f"exec {name} x{nsteps} without handler -> {err or 'no error'}")
            if err != (ERR_NAME.get(oerr, str(oerr)) if oerr else ""):
                msg.append(f"step {step}: raised {err!r} vs oracle {oerr}")
            msg += compare(ps, pd, f"step {step} ({log[-1]})")
            if err:  # what a user does next: drop the particles in an error state, carry on
                bad_rows = np.where(pd["state"] >= 50)[0]
                if len(bad_rows) == 0 or len(bad_rows) >= len(pd["x"]):
                    break
                if not np.array_equal(np.where(ps.state >= 50)[0], bad_rows):
                    msg.append(f"step {step}: error rows")
                ps.remove_indices(bad_rows)
                for k in pd:
                    pd[k] = np.delete(pd[k], bad_rows, axis=0)
        elif op == "edit":
            idx = rng.integers(0, n, int(rng.integers(1, 4)))
            key = str(rng.choice(["x", "y", "z"] if three else ["x", "y"]))
            delta = np.float32(rng.uniform(-0.02, 0.02) * float(np.abs(np.asarray(c["lon" if key == "x" else "lat"])).max()) if key != "z" else rng.uniform(0, 1.0))
            log.append(f"edit {key}[{idx.tolist()}] += {delta}")
            getattr(ps, key)[idx] += delta
            pd[key][idx] += delta
        elif op == "view":
            i = int(rng.integers(0, n))
            if rng.random() < 0.5:
                v = np.float32(pd["y"][i] * np.float32(0.999))
                log.append(f"pset[{i}].y = {v}")
                ps[i].y = v
                pd["y"][i] = v
            else:
                mask = rng.random(n) < 0.3
                log.append(f"pset[mask {int(mask.sum())}].x *= 0.999")
                view = ps[mask]
                view.x = view.x * np.float32(0.999)
                pd["x"][mask] = pd["x"][mask] * np.float32(0.999)
        elif op == "setattr":
            log.append("pset.dz = 0")
            ps.dz = 0.0
            pd["dz"][:] = 0.0
        elif op == "remove":
            idx = np.unique(rng.integers(0, n, int(rng.integers(1, 3))))
            if len(idx) >= n:
                continue
            log.append(f"remove {idx.tolist()}")
            ps.remove_indices(idx)
            for k in pd:
                pd[k] = np.delete(pd[k], idx, axis=0)
        elif op == "add":
            m = int(rng.integers(1, 5))
            j = rng.integers(0, len(c["x"]), m)
            t_new = np.full(m, float(np.nanmax(pd["t"])))
            log.append(f"add {m} at t={t_new[0]}")
            ps.add(pb.ParticleSet(fs, x=c["x"][j], y=c["y"][j], z=c["z"][j], t=t_new))
            new = po.create_particle_data(c["x"][j], c["y"][j], c["z"][j], t_new, ngrids=ofs.ngrids)
            new["particle_id"] = new["particle_id"] + (pd["particle_id"].max() + 1)  # particleset.py:188-224
            for k in pd:
                pd[k] = np.concatenate((pd[k], new[k]))
        elif op == "read":
            log.append("read")
            if len(ps) != n or not np.array_equal(ps.t, pd["t"], equal_nan=True):
                msg.append(f"step {step}: read len / t")
        elif op == "other":
            if other is None:
                m = min(3, len(c["x"]))
                other = (pb.ParticleSet(fs, x=c["x"][:m], y=c["y"][:m], z=c["z"][:m], t=np.zeros(m)),
                         po.create_particle_data(c["x"][:m], c["y"][:m], c["z"][:m], np.zeros(m), ngrids=ofs.ngrids))  # fmt: skip
            ops_, opd = other
            if len(opd["x"]) and float(np.nanmax(opd["t"])) + dt <= t_end:
                log.append("other set executes")
                name = "AdvectionRK4_3D" if three else "AdvectionRK4"
                ops_.execute([getattr(pb, name), pb.DeleteParticle], dt=dt, runtime=dt)
                po.pset_execute(opd, ofs, [getattr(po, name), po.DeleteOnError], dt, runtime=dt)
                msg += compare(ops_, opd, f"step {step} (other set)")
        if msg:
            break
    if not msg:
        msg += compare(ps, pd, "end")
    fs.release()
    return knobs + " | ".join(log), spec, msg


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(args[0]) if len(args) > 0 else 50
    rng = np.random.default_rng(int(args[1]) if len(args) > 1 else 0)
    bad = 0
    for k in range(n):
        try:
            what, spec, msg = one_case(rng)
        except Exception as e:  # noqa: BLE001
            import traceback

            print(f"[{k}] EXC {type(e).__name__}: {e}")
            traceback.print_exc()
            bad += 1
            continue
        if msg:
            bad += 1
            print(f"[{k}] {what}\n    {msg}\n    spec={spec}")
        elif VERBOSE:
            print(f"[{k}] ok: {what}")
    print(f"{n} cases, {bad} with differences")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
