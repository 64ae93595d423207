"""The engine against the REFERENCE ITSELF (not the oracle): random rectilinear configurations run twice through the reference's own
``ParticleSet.execute`` under the stub harness (oracle/ref_harness.py) -- untouched, and with ``parcels_b200.install()`` patching
``Kernel.execute`` so that the inner loop runs on the engine (here: the host simulation of the kernel sources) -- and the two
``pset._data`` compared: ids / states / times / cells / dt identical, positions bit-exact on flat meshes and within 4 float32 ulp on
spherical ones (the tolerances of scripts/fuzz_hostsim.py), the same exception class when there is no error handler.  Every fifth
case is AdvectionRK45 (per-particle dt / next_dt and the Repeat loop; alone or followed by a user kernel), every fifth a batch of
single evaluations: the reference's `Field.eval` (four scalar interpolators) and `VectorField.eval` against the device sampling; every
seventh a random CURVILINEAR C-grid mesh (cells / states / times identical, positions asserted on spherical meshes), every fifth a
random SEQUENCE of operations on the reference's own ParticleSet (executes, edits, views, remove_indices, add) with and without the patch.
Needs /root/reference (the build container).
Run:  PB_LIB=oracle/_build/hostsim/libparcels_b200_hostsim.so PB_HOSTSIM_TEST=1 python scripts/fuzz_install_vs_reference.py [n] [seed]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "scripts"))
import warnings
import numpy as np
from oracle import ref_harness as rh

if not rh.reference_available():
    print("reference not present: nothing to compare with")
    sys.exit(0)
rh.install()
import parcels._core.statuscodes as rcodes  # noqa: E402
import cases  # noqa: E402
import parcels_b200 as pb  # noqa: E402
from engine_run import ulp_diff_f32  # noqa: E402
from fuzz_hostsim import compare_with_reference, inject_boundary_cases, random_curv_spec, random_spec  # noqa: E402

warnings.simplefilter("ignore")
K = rh.kernels()


def user_delete(particles, fieldset):  # the reference's own idiom (tests/common_kernels.py:12-13)
    particles[particles.state >= 50].state = rcodes.StatusCode.Delete


def run(c, spec, patched, token):
    (pb.install if patched else pb.uninstall)()
    fs = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"], mesh=c["mesh"],
                           constants=c.get("constants"), interp=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")))  # fmt: skip
    ps = rh.make_pset(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    kern = [getattr(K, k) for k in c["kernels"]]
    if c["delete_on_error"]:
        kern.append(pb.DeleteParticle if (patched and token) else user_delete)
    err = ""
    try:
        for seg in c["segments"]:
            ps.execute(kern, dt=np.timedelta64(int(round(c["dt"] * 1e9)), "ns"), verbose_progress=False,
                       **{k: np.timedelta64(int(round(v * 1e9)), "ns") for k, v in seg.items()})  # fmt: skip
    except Exception as e:  # noqa: BLE001
        err = f"{type(e).__module__}.{type(e).__name__}"
    finally:
        pb.uninstall()
    return ps, err


def rk45_case(rng):
    """AdvectionRK45 (per-particle dt / next_dt, Repeat loop), alone or followed by a user kernel, through both sides."""
    from fuzz_hostsim_more import base_case

    spec, c = base_case(rng, two_d=True, interps=("linear", "cgrid_velocity", "freeslip", "partialslip"))
    tmax = None if c["times"] is None else float(c["times"][-1])
    dt = float(rng.choice([50.0, 200.0])) * (1 if rng.random() < 0.8 else -1)
    runtime = abs(dt) * int(rng.integers(2, 10))
    if tmax is not None:
        runtime = min(runtime, 0.45 * tmax)  # RK45 waiver (DESIGN.md): stay inside the time axis
        c["t"] = np.full(len(c["x"]), (0.0 if dt > 0 else tmax) + (0.05 * tmax if dt > 0 else -0.05 * tmax))
    runtime = float(int(runtime))
    tol = float(rng.choice([1e-4, 1e-2, 1.0]))
    min_dt, max_dt = float(rng.choice([0.5, 5.0])), abs(dt) * float(rng.choice([2, 4]))
    mixed = bool(rng.random() < 0.4)

    def Drift(particles, fieldset):
        particles.dy += 0.25 * particles.dt

    out = []
    for patched in (False, True):
        (pb.install if patched else pb.uninstall)()
        fs = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"], mesh=c["mesh"],
                               interp=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")))  # fmt: skip
        fs.add_context("RK45_tol", tol)
        fs.add_context("RK45_min_dt", min_dt)
        fs.add_context("RK45_max_dt", max_dt)
        ps = rh.make_pset(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"], extra_variables=[("next_dt", np.float32, 0)])
        err = ""
        try:
            ps.execute([K.AdvectionRK45, Drift] if mixed else [K.AdvectionRK45], dt=np.timedelta64(int(dt), "s"),
                       runtime=np.timedelta64(int(runtime), "s"), verbose_progress=False)  # fmt: skip
        except Exception as e:  # noqa: BLE001
            err = f"{type(e).__module__}.{type(e).__name__}"
        finally:
            pb.uninstall()
        out.append((ps, err))
    (a, ea), (b, eb) = out
    msg = [] if ea == eb else [f"raised {eb!r} vs the reference's {ea!r}"]
    da, db = a._data, b._data
    if len(da["x"]) != len(db["x"]):
        return spec, msg + [f"survivors {len(db['x'])} vs {len(da['x'])}"], b
    msg += [k for k in ("particle_id", "state", "t", "dt", "next_dt", "ei") if not np.array_equal(da[k], db[k])]
    for key in "xy":
        floor = 0.01 * float(np.abs(np.asarray(c[key])).max()) or None
        u = ulp_diff_f32(db[key], da[key], floor=floor)
        # C-grids: the reference's np.einsum takes another summation path for a batch of exactly ONE evaluated particle (a lone
        # straggler at min_dt here) -- last-bit differences inside the reference itself, DESIGN.md waiver 8: half an ulp of the
        # coordinate scale instead of bit-exactness
        tol = (0.5 if c.get("interp") == "cgrid_velocity" else 0) if c["mesh"] == "flat" else 4
        if u.size and u.max() > tol:
            msg.append(f"{key}: {u.max():.3f} ulp (tol {tol})")
    spec = dict(spec, rk45=dict(tol=tol, min_dt=min_dt, max_dt=max_dt, dt=dt, runtime=runtime, mixed=mixed))
    return spec, msg, b


def eval_case(rng):
    """Single evaluations: `fieldset.P.eval(t, z, y, x, particles)` (XLinear / XNearest / CGrid_Tracer / XLinearInvdistLandTracer) and
    `fieldset.UVW.eval(...)` of the reference against the engine's device sampling: values, dtypes, `ei`, states."""
    from engine_run import make_fieldset
    from fuzz_hostsim_more import base_case

    spec, c = base_case(rng, two_d=False, interps=("linear", "cgrid_velocity", "freeslip", "partialslip"))
    T = c["U"].shape[0] if rng.random() < 0.6 else 1
    P = (1.0 + rng.uniform(0, 1, (T,) + c["U"].shape[1:])).astype(rng.choice([np.float32, np.float64]))
    P[rng.uniform(size=P.shape) < 0.15] = 0  # land
    how = str(rng.choice(["linear", "nearest", "cgrid_tracer", "linear_invdist_land"]))
    n = len(c["x"])
    if n == 1 and how == "linear_invdist_land":
        how = "linear"  # (a batch of ONE sample: DESIGN.md waiver 1)
    tmax = 0.0 if c["times"] is None else float(c["times"][-1])
    tq = rng.uniform(0, tmax, n) if tmax else np.zeros(n)
    f32 = bool(rng.random() < 0.5)
    dt_ = np.float32 if f32 else np.float64
    x, y, z = (np.asarray(c[k]).astype(dt_) for k in "xyz")
    # reference
    rfs = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"], mesh=c["mesh"],
                            interp=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")), scalars={"P": (P, how)})  # fmt: skip
    rps = rh.make_pset(rfs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    rval = np.asarray(rfs.P.eval(tq, z, y, x, rps))
    r_ei, r_state = rps._data["ei"].copy(), rps._data["state"].copy()
    rps2 = rh.make_pset(rfs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    ruvw = [np.asarray(a) for a in rfs.UVW.eval(tq, z, y, x, rps2)]
    # engine
    fs = make_fieldset(c)
    fs.add_field("P", P, interp_method=how)
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    val = np.asarray(fs.P.eval(tq, z, y, x, ps))
    ps2 = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    uvw = [np.asarray(a) for a in fs.UVW.eval(tq, z, y, x, ps2)]
    msg = []
    if val.dtype != rval.dtype and not (T > 1):
        msg.append(f"P dtype {val.dtype} vs {rval.dtype}")
    if not np.array_equal(ps._data["ei"], r_ei):
        msg.append("P ei")
    if not np.array_equal(ps._data["state"], r_state):
        msg.append("P state")
    same = (val.astype(np.float64) == rval.astype(np.float64)) | (np.isnan(val) & np.isnan(rval))
    if not same.all():
        bad = np.flatnonzero(~same)
        msg.append(f"P at {bad[:4]}: {val[bad[:4]]} vs {rval[bad[:4]]}")
    if not np.array_equal(ps2._data["ei"], rps2._data["ei"]) or not np.array_equal(ps2._data["state"], rps2._data["state"]):
        msg.append("UVW ei / state")
    for name, g, w in zip("uvw", uvw, ruvw):
        scale = float(np.abs(w[np.isfinite(w)]).max()) if np.isfinite(w).any() else 0.0
        if c["mesh"] == "spherical":  # (the tolerances of tests/test_gpu_eval.py)
            tol = 4 * np.finfo(np.float32).eps if (f32 or w.dtype == np.float32) else 64 * np.finfo(np.float64).eps
            if c.get("interp") == "cgrid_velocity" and spec["cdtype"] == "f4":
                tol = 64 * np.finfo(np.float32).eps  # float32 edge lengths with a float32 cos (the trajectory rule above)
            elif c.get("interp") == "cgrid_velocity" and tol < 1e-10:
                tol = 1024 * np.finfo(np.float64).eps  # Jacobian cancellation on top of the einsum / cos last bits (waivers 8, 9)
        elif c.get("interp") == "cgrid_velocity":
            tol = 32 * np.finfo(np.float64).eps if w.dtype == np.float64 and not f32 else 4 * np.finfo(np.float32).eps
        else:
            tol = 0.0
        err = np.abs(g.astype(np.float64) - w.astype(np.float64))
        err = np.where(np.isnan(w) & np.isnan(g), 0.0, err)
        if err.size and float(np.nanmax(err)) > tol * scale:
            msg.append(f"{name}: {float(np.nanmax(err)) / max(scale, 1e-300):.2e} x scale (tol {tol:.1e})")
    # ParticleSet.populate_indices (reference _core/particleset.py:252-262): the hintless search of every particle, also on a random
    # curvilinear mesh (spatial hash)
    rps3 = rh.make_pset(rfs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    rps3.populate_indices()
    ps3 = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    ps3.populate_indices()
    if not np.array_equal(ps3._data["ei"], rps3._data["ei"]):
        msg.append("populate_indices")
    cspec = random_curv_spec(rng)
    cc = cases.build(cspec)
    cfs = rh.build_fieldset(lon=cc["lon"], lat=cc["lat"], depth=cc["depth"], times=cc["times"], U=cc["U"], V=cc["V"], W=cc["W"],
                            mesh=cc["mesh"], interp="cgrid_velocity", padding=cc.get("padding", ("low", "low", "high")))  # fmt: skip
    rps4 = rh.make_pset(cfs, x=cc["x"], y=cc["y"], z=cc["z"], t=cc["t"])
    rps4.populate_indices()
    efs = make_fieldset(cc)
    ps4 = pb.ParticleSet(efs, x=cc["x"], y=cc["y"], z=cc["z"], t=cc["t"])
    ps4.populate_indices()
    if not np.array_equal(ps4._data["ei"], rps4._data["ei"]):
        bad_ = np.flatnonzero((ps4._data["ei"] != rps4._data["ei"]).any(axis=1))
        msg.append(f"populate_indices (curvilinear {cspec['mesh']} {cspec['cdtype']}): {len(bad_)} of {len(cc['x'])} cells differ")
    efs.release()
    fs.release()
    spec = dict(spec, eval=dict(how=how, T=T, f32=f32, P=str(P.dtype)))
    return spec, msg


def sequence_case(rng):
    """A random SEQUENCE of operations on the reference's own ParticleSet -- executes (built-ins with the user error handler or the
    engine's token, several kernels), in-place edits of `pset._data`, `pset[i]` / `pset[mask]` view assignments, `remove_indices`,
    `add` -- applied to an untouched set and to one whose Kernel.execute is patched: the adapter shares the reference's arrays, so
    every mutation between the calls (np.delete and np.concatenate REPLACE the columns) has to be picked up."""
    from fuzz_hostsim_more import base_case

    three = bool(rng.random() < 0.5)
    spec, c = base_case(rng, two_d=not three, interps=("linear", "freeslip", "cgrid_velocity"))
    if spec["mesh"] != "flat":  # bit-exact comparison: flat meshes
        spec["mesh"] = "flat"
        c = cases.build(spec)
        if not three:
            c["W"] = None
            c["z"] = np.abs(np.asarray(c["z"]))
    dt = float(rng.choice([50.0, 100.0]))
    tmax = np.inf if c["times"] is None else float(c["times"][-1])
    names = ["AdvectionRK4_3D", "AdvectionRK2_3D"] if three else ["AdvectionRK4", "AdvectionRK2", "AdvectionEE"]
    sets = []
    for patched in (False, True):
        fs = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"], mesh=c["mesh"],
                               interp=c.get("interp", "linear"), padding=c.get("padding", ("low", "low", "high")))  # fmt: skip
        sets.append((fs, rh.make_pset(fs, x=c["x"], y=c["y"], z=c["z"], t=np.zeros(len(c["x"])))))
    log, msg = [], []
    t_now = 0.0
    for step in range(int(rng.integers(3, 8))):
        n = len(sets[0][1]._data["x"])
        if n == 0:
            break
        op = str(rng.choice(["exec", "exec", "exec", "edit", "view", "remove", "add"]))
        if op == "exec":
            name = str(rng.choice(names))
            nsteps = int(rng.integers(1, 5))
            if t_now + nsteps * dt > tmax:
                continue
            token = bool(rng.random() < 0.5)
            errs = []
            for patched, (fs, ps) in zip((False, True), sets):
                (pb.install if patched else pb.uninstall)()
                try:
                    ps.execute([getattr(K, name), pb.DeleteParticle if (patched and token) else user_delete], dt=np.timedelta64(int(dt), "s"),
                               runtime=np.timedelta64(int(nsteps * dt), "s"), verbose_progress=False)  # fmt: skip
                    errs.append("")
                except Exception as e:  # noqa: BLE001
                    errs.append(type(e).__name__)
                finally:
                    pb.uninstall()
            t_now += nsteps * dt
            log.append(f"exec {name} x{nsteps} token={token}")
            if errs[0] != errs[1]:
                msg.append(f"step {step}: raised {errs}")
            da, db = sets[0][1]._data, sets[1][1]._data
            if set(da) != set(db) or len(da["x"]) != len(db["x"]):
                msg.append(f"step {step}: {len(db['x'])} particles vs {len(da['x'])}")
            else:
                msg += [f"step {step} ({log[-1]}): {k}" for k in da if not np.array_equal(da[k], db[k], equal_nan=True)]
        elif op == "edit":
            idx = rng.integers(0, n, int(rng.integers(1, 4)))
            delta = np.float32(rng.uniform(-0.01, 0.01) * float(np.abs(np.asarray(c["lon"])).max()))
            log.append(f"edit x[{idx.tolist()}]")
            for _, ps in sets:
                ps._data["x"][idx] += delta
        elif op == "view":
            i = int(rng.integers(0, n))
            mask = rng.random(n) < 0.3
            log.append(f"views [{i}], mask {int(mask.sum())}")
            for _, ps in sets:
                ps[i].y = ps[i].y * np.float32(0.999)
                v = ps[mask]
                v.x = v.x * np.float32(0.9995)
        elif op == "remove":
            idx = np.unique(rng.integers(0, n, int(rng.integers(1, 3))))
            if len(idx) >= n:
                continue
            log.append(f"remove {idx.tolist()}")
            for _, ps in sets:
                ps.remove_indices(idx)
        elif op == "add":
            m = int(rng.integers(1, 4))
            j = rng.integers(0, len(c["x"]), m)
            log.append(f"add {m}")
            for fs, ps in sets:
                ps.add(rh.make_pset(fs, x=np.asarray(c["x"])[j], y=np.asarray(c["y"])[j], z=np.asarray(c["z"])[j], t=np.full(m, t_now)))
        if msg:
            break
    return dict(spec, sequence=" | ".join(log)), msg


def main():
    n_cases = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
    bad = on_engine = 0
    for k in range(n_cases):
        if k % 5 == 4:
            try:
                spec, msg, b = rk45_case(rng)
            except Exception as e:  # noqa: BLE001
                import traceback

                print(f"[{k}] EXC {type(e).__name__}: {e}")
                traceback.print_exc()
                bad += 1
                continue
            on_engine += b.__dict__.get("_b200_pset") is not None
            if msg:
                bad += 1
                print(f"[{k}] MISMATCH (AdvectionRK45) {'; '.join(msg)}\n    spec={spec}")
            continue
        if k % 5 in (0, 2):
            try:
                spec, msg = eval_case(rng) if k % 5 == 2 else sequence_case(rng)
            except Exception as e:  # noqa: BLE001
                import traceback

                print(f"[{k}] EXC {type(e).__name__}: {e}")
                traceback.print_exc()
                bad += 1
                continue
            on_engine += 1
            if msg:
                bad += 1
                print(f"[{k}] MISMATCH ({'eval' if k % 5 == 2 else 'sequence'}) {'; '.join(msg)}\n    spec={spec}")
            continue
        spec = random_curv_spec(rng) if k % 7 == 3 else random_spec(rng)
        if spec["kind"] == "curv" and rng.random() < 0.4:
            spec["interp"] = "linear"  # XLinear_Velocity behind the curvilinear search (A-grid data on a curvilinear mesh)
        token = bool(rng.random() < 0.6)
        try:
            c = cases.build(spec)
            inject_boundary_cases(rng, spec, c)
            a, ea = run(c, spec, False, token)
            b, eb = run(c, spec, True, token)
        except Exception as e:  # noqa: BLE001
            import traceback

            print(f"[{k}] EXC {type(e).__name__}: {e}\n    spec={spec}")
            traceback.print_exc()
            bad += 1
            continue
        on_engine += b.__dict__.get("_b200_pset") is not None
        msg = compare_with_reference(spec, c, a._data, ea, b._data, eb)
        if msg:
            bad += 1
            print(f"[{k}] MISMATCH {'; '.join(msg)}  (token={token})\n    spec={spec}")
    print(f"{n_cases} cases ({on_engine} through the engine), {bad} with differences")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
