"""The engine against the REFERENCE'S OWN outputs on 140 random trajectory configurations (tests/golden/reference_fuzz.npz, made by
``python -m oracle.make_golden reference_fuzz`` where the reference is importable): every case is rebuilt from its stored spec and
release arrays, run through the public API (``parcels_b200.ParticleSet.execute``, built-in kernels + ``DeleteParticle`` where the
case deletes on error) and compared with the reference's particle data by the rules of scripts/fuzz_hostsim.compare_with_reference.
Run:  PB_LIB=oracle/_build/hostsim/libparcels_b200_hostsim.so PB_HOSTSIM_TEST=1 python scripts/replay_reference_fuzz.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import numpy as np  # noqa: E402

import cases  # noqa: E402
import parcels_b200 as pb  # noqa: E402
from engine_run import make_fieldset  # noqa: E402
from fuzz_hostsim import compare_with_reference  # noqa: E402
from oracle.make_golden import REFERENCE_FUZZ_COLUMNS  # noqa: E402
from parcels_b200._lib import EngineError  # noqa: E402


def run_engine(c):
    fs = make_fieldset(c)
    t = (np.asarray(c["t"], dtype=np.float64) * 1e9).astype("timedelta64[ns]")  # release times as the reference was given them
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=t)
    kern = [getattr(pb, k) for k in c["kernels"]] + ([pb.DeleteParticle] if c["delete_on_error"] else [])
    err = ""
    try:
        for seg in c["segments"]:  # the times the reference was given: nanosecond timedelta64 (oracle/make_golden.py)
            ps.execute(kern, dt=np.timedelta64(int(round(c["dt"] * 1e9)), "ns"),
                       **{k: np.timedelta64(int(round(v * 1e9)), "ns") for k, v in seg.items()})  # fmt: skip
    except EngineError:
        raise
    except Exception as e:  # noqa: BLE001 -- compared with what the reference raised
        err = type(e).__name__
    return ps._data, err


def main():
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference_fuzz.npz"))
    n_cases = len([k for k in g.files if k.endswith("/spec")])
    bad = 0
    for k in range(n_cases):
        spec = json.loads(str(g[f"{k}/spec"]))
        c = cases.build(spec)
        c.update({key: g[f"{k}/in_{key}"] for key in "xyzt"})
        ref = {key: g[f"{k}/{key}"] for key in REFERENCE_FUZZ_COLUMNS}
        d, err = run_engine(c)
        msg = compare_with_reference(spec, c, ref, str(g[f"{k}/error"]), d, err)
        if msg:
            bad += 1
            print(f"[{k}] MISMATCH {'; '.join(msg)}\n    spec={spec}")
    print(f"{n_cases} cases against the reference's stored outputs, {bad} with differences")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
