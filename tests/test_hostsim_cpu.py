"""CPU (no GPU needed): the GPU parity tests run against the product's kernel SOURCES compiled for the host
(oracle/hostsim: g++ build of parcels_b200/csrc behind the same C-ABI, one simulated thread at a time).

This checks the LOGIC of the CUDA sources -- state machine, searches, interpolation arithmetic, error / delete / replay
handling, output selection, hash build, host bindings -- against the oracle and the reference's golden outputs on machines
without a GPU.  It is test infrastructure: the product never loads the simulation (it needs PB_LIB pointing at it AND
PB_HOSTSIM_TEST=1), and the real parity statement is `pytest -m gpu` on the H100."""

import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no C++ compiler for the host simulation")

# the 2-rank domain-decomposed check runs separately below (fewer particles); the NCCL variant needs two real GPUs
DESELECT = ["tests/test_gpu_decomposed.py"]


def _env(lib):
    env = dict(os.environ, PB_LIB=lib, PB_HOSTSIM_TEST="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return env


def test_gpu_suite_passes_on_the_host_compiled_kernel_sources():
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "pytest", "tests", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"]
    for d in DESELECT:
        cmd += ["--deselect", d]
    res = subprocess.run(cmd, cwd=ROOT, env=_env(lib), capture_output=True, text=True, timeout=1500)
    tail = "\n".join(res.stdout.splitlines()[-25:])
    assert res.returncode == 0, tail + "\n" + res.stderr[-2000:]
    assert " passed" in tail and "failed" not in tail, tail


def test_simulation_is_inert_without_the_test_switch():
    """The simulated device only exists for the harness: without PB_HOSTSIM_TEST=1 the library reports no device at all."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    code = ("import ctypes, sys; l = ctypes.CDLL(sys.argv[1]); l.pb_device_count.restype = ctypes.c_int32; "
            "h = ctypes.c_void_p(); print(l.pb_device_count(), l.pb_engine_create(0, ctypes.byref(h)))")  # fmt: skip
    env = {k: v for k, v in os.environ.items() if k != "PB_HOSTSIM_TEST"}
    out = subprocess.run([sys.executable, "-c", code, lib], env=env, capture_output=True, text=True, timeout=120).stdout.split()
    assert out[0] == "0" and int(out[1]) < 0, out


def test_differential_fuzz_of_the_kernel_sources_against_the_oracle():
    """120 random rectilinear configurations (dtypes, meshes, 2-D / 3-D, schemes, interpolators, release patterns, time direction,
    error handling; scripts/fuzz_hostsim.py): the host-compiled kernels and the oracle must agree on every one."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    res = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "fuzz_hostsim.py"), "120", "2026"], cwd=ROOT, env=_env(lib),
                         capture_output=True, text=True, timeout=900)  # fmt: skip
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().endswith("120 cases, 0 with differences"), res.stdout[-3000:]


def test_differential_fuzz_of_sampling_rk45_and_advection_diffusion():
    """70 random cases of scalar Field.eval (four interpolators), AdvectionRK45, AdvectionDiffusionM1 / EM, fused
    DiffusionUniformKh over several execute() calls, time-slab streaming vs the resident field, the rows handed to the output
    file at every output time, and mixed lists with user kernels (scripts/fuzz_hostsim_more.py): host-compiled kernels == oracle."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    res = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "fuzz_hostsim_more.py"), "70", "2026"], cwd=ROOT, env=_env(lib),
                         capture_output=True, text=True, timeout=900)  # fmt: skip
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().endswith("70 cases, 0 with differences"), res.stdout[-3000:]


def test_differential_fuzz_of_the_round_two_paths():
    """80 random cases of what round 2 added (scripts/fuzz_hostsim_r2.py): RK4 / Euler behind the curvilinear search (A-grid bilinear
    and C-grid), scalar Field.eval on curvilinear meshes (XLinear and the C-grid tracer rules), AdvectionDiffusionM1 / EM on a C-grid
    velocity, fields on a second grid inside one kernel list, the in-kernel migration records of the peer-memory transport, and
    time-slab streaming under mode D through distributed.execute_decomposed on thread ranks."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    res = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "fuzz_hostsim_r2.py"), "80", "2026"], cwd=ROOT, env=_env(lib),
                         capture_output=True, text=True, timeout=900)  # fmt: skip
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().endswith("80 cases, 0 with differences"), res.stdout[-3000:]


def test_differential_fuzz_of_the_host_layers_bookkeeping():
    """400 random SEQUENCES of public-API operations on one ParticleSet (execute with random kernel lists and output files, in-place
    edits, views, removals, additions, a second set on the same FieldSet, the chunked host-array pipeline forced on small sets),
    mirrored on the oracle and compared after every execute (scripts/fuzz_hostsim_api.py): which copy of the set is current --
    host arrays, device arrays, a lazily resident set -- never goes wrong."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    res = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "fuzz_hostsim_api.py"), "400", "2026"], cwd=ROOT, env=_env(lib),
                         capture_output=True, text=True, timeout=900)  # fmt: skip
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().endswith("400 cases, 0 with differences"), res.stdout[-3000:]


def test_domain_decomposed_migration_on_the_host_compiled_kernels():
    """Mode D (X-slab decomposition, classify / pack / compact / unpack kernels, gloo all-to-all of the 48-byte records): 2 ranks,
    each with its own simulated engine, reproduce the single-engine trajectories bit for bit (scripts/decomposed_check.py)."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29641", os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--particles", "3000"]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


def test_domain_decomposed_diffusion_statistics_on_the_host_compiled_kernels():
    """Fused DiffusionUniformKh under mode D: every migration round is a new launch with its own RNG call index, so particles that
    hop between the ranks keep drawing fresh Wiener increments (Var = 2 K t, every particle accounted for once)."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29642", os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--particles", "3000", "--diffusion"]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0 and "PASS statistics" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_in_kernel_migration_logic_on_the_host_compiled_kernels():
    """Mode D over peer memory: the advection kernel delivers leavers into the new owner's inbox itself.  CUDA IPC needs real devices,
    so the kernel / inbox / finish LOGIC runs here with three slab engines of one process linked by address (incl. a 50-record inbox
    that overflows); the cross-process mapping is covered on the GPU box (tests/test_gpu_decomposed.py, bench.py's bitexact_check)."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "pytest", "tests/test_gpu_decomposed.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "-k",
           "three_slabs_one_process"]  # fmt: skip
    res = subprocess.run(cmd, cwd=ROOT, env=_env(lib), capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "2 passed" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_peer_memory_transport_falls_back_to_the_collectives_on_every_rank():
    """A rank that cannot map a peer's inbox (here: no CUDA IPC in the host simulation) must not leave the others waiting: all ranks
    agree -- one all-gather -- to stay on the collective transport, and the run is still bit-exact (distributed.connect_p2p)."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29643", os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--particles", "3000",
           "--transport", "p2p"]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "transport=collectives" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_time_slab_streaming_under_domain_decomposition():
    """Mode D on time-windowed slabs (2 of 6 levels resident per rank, windows slid in lock-step, distributed._slide_in_lockstep):
    bit-exact against the undecomposed run that keeps every level resident.  (a) 2 gloo ranks on the collective transport;
    (b) the product's own peer-memory round loop (execute_decomposed -> run_decomposed_p2p) with 3 thread ranks whose inboxes are
    linked by address, staggered releases and a 50-record inbox that overflows; (c) backward in time, 4 ranks, 3 levels."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29644", os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--particles", "2000",
           "--nt", "6", "--runtime", "345600", "--time-window", "2", "--transport", "collective"]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "time window 2 of 6" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    threads = [sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--nt", "6", "--runtime", "345600"]
    for extra in (["--inbox", "50", "--time-window", "2"], ["--backward", "--time-window", "3", "--world", "4"]):
        r = subprocess.run(threads + extra, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
        assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "peer memory" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
        assert " 0 migrations" not in r.stdout


def test_peer_memory_round_loop_on_thread_ranks():
    """distributed.run_decomposed_p2p itself (not a hand-driven copy of its rounds): 3 and 8 thread ranks, resident fields."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py")], capture_output=True, text=True,
                       timeout=900, cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "peer memory" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    # the slab count of the driver's largest run (8), with an inbox that overflows: leavers wait for later rounds, some cross several slabs
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--world", "8", "--particles", "6000",
                        "--inbox", "64"], capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout and "8 thread ranks" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_nan_node_on_the_device_side_hash_build_and_query():
    """reference tests/test_spatialhash.py:125-181 through the device code (hash build from the per-face boxes + hintless query),
    flat and spherical: scripts/hash_nan_check.py."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "hash_nan_check.py")], capture_output=True, text=True,
                       timeout=600, cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0 and "PASS nan node" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_random_configurations_against_the_references_stored_outputs():
    """140 random trajectory configurations (scripts/fuzz_hostsim.py's generators: dtypes, meshes, 2-D / 3-D, five schemes, five
    interpolators, random curvilinear C-grids, boundary releases, non-finite coordinates, releases outside the time interval) through
    the public API, against what the reference's own ParticleSet.execute produced on them (tests/golden/reference_fuzz.npz)."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "replay_reference_fuzz.py")], capture_output=True, text=True,
                       timeout=900, cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.strip().endswith("140 cases against the reference's stored outputs, 0 with differences"), r.stdout[-3000:]


def _bench_line(stdout):
    import json

    lines = [ln for ln in stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, stdout[-2000:]  # ONE JSON line
    return json.loads(lines[0])


def test_bench_control_flow_single_rank(tmp_path):
    """bench.py's N = 1 flow on the simulated device (scripts/bench_hostsim.py: torch.cuda entry points stubbed, numbers
    meaningless): the arms run, the line carries every key of the contract, the parity sample agrees with the oracle, and
    --dump-outputs writes the particle set of the last timed step."""
    import numpy as np

    from oracle.hostsim import build as hb

    lib = hb.build()
    dump = tmp_path / "dump"
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "bench_hostsim.py"), "--workload", "c2_small", "--particles", "1500", "--steps", "3",
           "--warmup", "3", "--extras", "c3_small", "--dump-outputs", str(dump)]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]
    d = _bench_line(r.stdout)
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "parity_sample", "clocks", "extra"):  # fmt: skip
        assert k in d, k
    assert d["n_gpus"] == 1 and d["steps"] == 3 and d["gpu_launches"] > 0 and d["value"] > 0 and d["e2e"]["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 1500 * 48 and d["e2e"]["d2h_bytes_per_step"] == 1500 * 40
    assert set(d["roofline"]) >= {"bound", "achieved", "peak", "unit", "frac", "traffic"}
    assert d["parity_sample"]["ok"] and d["extra"]["c3_small"]["parity_sample"]["ok"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] == 1
    for name in ("c3_small", "c2_small"):
        cols = {k: np.load(dump / f"{name}_{k}.npy") for k in ("x", "y", "z", "t", "state", "ei", "particle_id", "row")}
        assert all(v.shape == (1500,) and v.dtype in (np.float32, np.float64) for v in cols.values())
        assert np.array_equal(cols["particle_id"], np.arange(1500))
    # what was dumped is what the pass computed: the oracle advects the same 1500 particles of c2_small (bench seeds rank 0 with 1)
    import bench
    from engine_run import ulp_diff_f32

    w = bench.WORKLOADS["c2_small"]
    field = w["field"](**w["fkw"])
    pd, _, _ = bench._oracle_pass("c2_small", w, field, w["particles"](field, 1500, 1))
    live = pd["particle_id"]
    assert len(live) > 0 and np.all(cols["state"][np.setdiff1d(np.arange(1500), live)] != 0)  # the rest were deleted
    assert np.array_equal(cols["t"][live], pd["t"]) and np.array_equal(cols["ei"][live], pd["ei"][:, -1])
    for k in "xyz":
        assert ulp_diff_f32(cols[k][live], pd[k], floor=0.05).max() <= w["ulp"], k


def test_bench_control_flow_two_ranks_and_the_mode_d_watchdog():
    """bench.py under torchrun (2 ranks, gloo instead of NCCL, both on the simulated device): mode R line + `mode_d` block -- the
    peer-memory transport is refused by the simulation, every rank agrees on the collectives, the bit-exactness check passes -- and
    with a 1-second limit the watchdog prints the mode R line with the reason and every rank exits 0."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    base = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1"]
    args = [os.path.join(ROOT, "scripts", "bench_hostsim.py"), "--gpus", "2", "--workload", "c2_small", "--particles", "1500",
            "--particles-d", "3000", "--steps", "3", "--warmup", "3", "--extras", "", "--no-cpu-baseline"]  # fmt: skip
    r = subprocess.run(base + ["--master-port", "29646"] + args, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env(lib))
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]
    d = _bench_line(r.stdout)
    md = d["mode_d"]
    assert d["n_gpus"] == 2 and "error" not in md, md
    assert md["transport"].startswith("collectives") and "p2p_unavailable" in md  # the agreed fallback
    assert md["bitexact_check"]["bit_exact_vs_one_gpu"] is True and md["bitexact_check"]["migrations"] > 0
    r = subprocess.run(base + ["--master-port", "29647"] + args + ["--mode-d-timeout", "1"], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]
    d = _bench_line(r.stdout)
    assert d["value"] > 0 and "did not finish within 1 s" in d["mode_d"]["error"]


def test_graft_entry_smoke_on_the_simulated_device():
    """__graft_entry__.smoke() (what the driver runs on cuda:0 before the bench) end to end on the simulated device."""
    from oracle.hostsim import build as hb

    lib = hb.build()
    r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=_env(lib))  # fmt: skip
    assert r.returncode == 0 and "smoke ok" in r.stdout, r.stdout[-1500:] + r.stderr[-2000:]
