"""CPU (host simulation of the kernel sources, oracle/hostsim): mode D on CURVILINEAR grids -- column slabs of the fields, the whole
horizontal grid and its spatial hash on every rank (DecomposedFieldSet.from_curvilinear) -- reproduces the undecomposed run bit for
bit: the peer-memory round loop on thread ranks (scripts/decomposed_threads_check.py) and the gloo collective transport of two
ranks (scripts/decomposed_check.py), with CGrid_Velocity and curvilinear XLinear_Velocity.  A halo too small for the step raises on
every rank; every rank's hash table is the single engine's."""

import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

needs_cxx = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no C++ compiler for the host simulation")


def _env():
    from oracle.hostsim import build as hb

    return dict(os.environ, PB_LIB=hb.build(), PB_HOSTSIM_TEST="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))


def _gloo(port, *extra):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", "decomposed_check.py"), "--same-gpu", "--transport", "collective",
           "--particles", "200", "--halo", "1", *extra]  # fmt: skip
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())


def _passed(r):
    assert r.returncode == 0 and "PASS bit-exact" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert " 0 migrations" not in r.stdout


# (kernel, interp, extra): 2-D and 3-D, both interpolators, both meshes and directions, delayed releases ordered by id with the
# hints of the first shards all zero, RK45, an inbox that overflows, a time window of 3 levels against the resident run
THREADS = [("rk4", "curv_cgrid", []), ("rk4_3d", "curv_cgrid", ["--ordered-releases"]), ("ee", "curv_linear", ["--backward"]),
           ("rk4", "curv_cgrid", ["--mesh", "flat", "--inbox", "16"]), ("rk45", "curv_cgrid", ["--delayed"]),
           ("rk45", "curv_cgrid", ["--ordered-releases", "--backward"]),
           ("rk4", "curv_linear", ["--time-window", "3", "--nt", "4"])]  # fmt: skip


@needs_cxx
@pytest.mark.parametrize("kernel,interp,extra", THREADS)
def test_thread_ranks_in_kernel_migration(kernel, interp, extra):
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "decomposed_threads_check.py"), "--kernel", kernel, "--interp", interp,
           "--particles", "200", "--halo", "1", *extra]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    _passed(r)
    assert "grid " in r.stdout and "fields " in r.stdout  # the per-rank device bytes are reported


@needs_cxx
@pytest.mark.parametrize("kernel,extra,port", [("rk4_3d", ["--ordered-releases"], 29691), ("rk45", ["--delayed"], 29692)])
def test_gloo_collective_transport(kernel, extra, port):
    _passed(_gloo(port, "--kernel", kernel, "--interp", "curv_cgrid", *extra))


@needs_cxx
def test_halo_violation_raises_on_every_rank():
    """Day-long RK4 steps leave a halo of one cell column: every rank raises, no particle is silently deleted."""
    r = _gloo(29693, "--kernel", "rk4", "--interp", "curv_cgrid", "--dt", "86400")
    assert r.returncode != 0
    assert r.stdout.count("RuntimeError: halo violation") == 2, r.stdout[-2000:] + r.stderr[-2000:]


def test_column_slab_plan():
    from parcels_b200 import distributed as D

    plans = D.column_slab_plan(72, 3, 2)
    assert [p["col_edges"].tolist() for p in plans] == [[0, 24, 47, 71]] * 3
    assert [(p["lo"], p["hi"], p["xi_offset"]) for p in plans] == [(0, 26, 0), (22, 49, 22), (45, 71, 45)]
    assert [(p["left_global"], p["right_global"]) for p in plans] == [(True, False), (False, False), (False, True)]
    with pytest.raises(ValueError):
        D.column_slab_plan(3, 3, 1)


@needs_cxx
def test_every_rank_holds_the_single_engine_hash_table():
    r = subprocess.run([sys.executable, "-c", _HASH_CHECK], capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "SAME" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


_HASH_CHECK = """
import sys, numpy as np
sys.path[:0] = ['scripts', 'tests']
import decomposed_kernels as K, parcels_b200 as pb
from parcels_b200 import distributed as D
case = K.make_case('rk4', n=10, interp='curv_cgrid')
f = case['f']
one = pb.FieldSet.from_arrays(lon=f['lon'], lat=f['lat'], time=f['times'], U=f['U'], V=f['V'], mesh='spherical', **case['fs_kw'])
ref = one.engine(0).hash_table()
for r in range(3):
    h = K.decomposed_fieldset(case, r, 3).engine.hash_table()
    assert all(np.array_equal(h[k], ref[k]) for k in ref), r
print('SAME')
"""


@needs_cxx
def test_first_evaluation_hint_rule_is_the_whole_sets():
    """The launches' ``hint_all_zero`` is the whole set's, not a shard's, and the set is routed to the owners of its cells before
    the first launch (with the first evaluation's hint rule).  Checked on the launch arguments: the float32 rounding of the hash
    path's barycentric coordinates moves a float32 position by far less than its ulp, so the trajectories rarely show the rule."""
    r = subprocess.run([sys.executable, "-c", _HINT_CHECK], capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "HINTS OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


_HINT_CHECK = """
import sys, numpy as np
sys.path[:0] = ['scripts', 'tests']
import decomposed_kernels as K, thread_ranks
from parcels_b200 import distributed as D
from parcels_b200.engine import Engine
from parcels_b200.plan import batch_facts
log = []
def spy(name, f, key):
    def call(self, *a, **kw):
        out = f(self, *a, **kw)
        log.append((id(self), name, key(a, out)))
        return out
    setattr(Engine, name, call)
spy('advect', Engine.advect, lambda a, out: (int(a[0].hint_all_zero), int(a[0].resume)))
spy('advect_async', Engine.advect_async, lambda a, out: (int(a[0].hint_all_zero), int(a[0].resume)))
spy('migrate_classify_columns', Engine.migrate_classify_columns, lambda a, out: (int(a[0]), int(out.sum())))
thread_ranks.serialise_engine_calls()
for ordered, p2p in ((False, True), (True, True), (False, False), (True, False)):
    case = K.make_case('rk4', n=150, interp='curv_cgrid', ordered=ordered)
    slabs = [K.decomposed_fieldset(case, r, 3) for r in range(3)]
    if p2p:
        bases = [s.engine.migrate_p2p_init(150)[1] for s in slabs]
        for s in slabs:
            s.engine.migrate_p2p_connect(local_bases=bases)
            s.p2p = True
    shards = [D.shard_particles(case['full'], r, 3) for r in range(3)]
    local = [batch_facts(slabs[r].fs, shards[r], shards[r]['ei'][:, -1], case['dt'], case['endtime'])[0] for r in range(3)]
    assert local[0] and (all(local) != ordered), local  # ordered: rank 0's shard alone would skip the hint, the whole set does not
    log.clear()
    thread_ranks.run_ranks(3, lambda r, dist: D.execute_decomposed(slabs[r], shards[r], case['kernels'], case['dt'], case['endtime'], dist))
    for s in slabs:
        mine = [(n, k) for e, n, k in log if e == id(s.engine)]
        launches = [k for n, k in mine if n.startswith('advect')]
        assert launches[0] == (int(not ordered), 0) and all(h == 0 for h, _ in launches[1:]), (ordered, p2p, launches)
        first = mine[0]
        assert first[0] == 'migrate_classify_columns' and first[1][0] == int(not ordered), (ordered, p2p, mine[:3])
    moved = sum(k[1] for e, n, k in log if n == 'migrate_classify_columns' and k[0] == int(not ordered))
    assert moved > 0  # particles started on other ranks than the owners of their cells
print('HINTS OK')
"""


def test_sampling_is_refused_on_column_slabs():
    """The sampling kernels index the fields by global column: on a column slab they would read past it, so the engine refuses."""
    r = subprocess.run([sys.executable, "-c", _SAMPLE_CHECK], capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "REFUSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


_SAMPLE_CHECK = """
import sys, numpy as np
sys.path[:0] = ['scripts', 'tests']
import decomposed_kernels as K
from parcels_b200._lib import EngineError
case = K.make_case('rk4', n=10, interp='curv_cgrid')
dfs = K.decomposed_fieldset(case, 0, 2)
x, y = case['x'][:4], case['y'][:4]
for call in (lambda: dfs.fs.UV.eval(np.zeros(4), np.zeros(4), y, x), lambda: dfs.engine.sample_velocity(np.zeros(4), np.zeros(4), y, x, three_d=False)):
    try:
        call()
    except EngineError as e:
        assert 'column slab' in str(e), e
    else:
        raise AssertionError('sampling a column slab was not refused')
print('REFUSED')
"""


def test_refusals():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")]
    import decomposed_kernels

    from parcels_b200 import distributed as D

    f = decomposed_kernels.curvilinear_field("rk4", "spherical", 3, False)
    with pytest.raises(NotImplementedError, match="curvilinear"):
        D.DecomposedFieldSet(lon=f["lon"], lat=f["lat"], time=f["times"], U=f["U"], V=f["V"], interp_method="cgrid_velocity", rank=0, world=2)
    with pytest.raises(ValueError, match="node coordinates"):
        D.DecomposedFieldSet.from_curvilinear(lon=f["lon"][0], lat=f["lat"][:, 0], time=f["times"], U=f["U"], V=f["V"], rank=0, world=2)


@needs_cxx
def test_kernel_refusals_are_the_single_gpu_ones():
    """AdvectionRK45 with curvilinear XLinear_Velocity and AdvectionDiffusionM1 / EM (their Kh fields cannot be added to a column
    slab) are refused on column slabs, as on one GPU; a set of one particle is refused (its hint rule is a whole-set rule)."""
    r = subprocess.run([sys.executable, "-c", _REFUSAL_CHECK], capture_output=True, text=True, timeout=900, cwd=ROOT, env=_env())
    assert r.returncode == 0 and "REFUSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


_REFUSAL_CHECK = """
import sys, numpy as np, pytest
sys.path[:0] = ['scripts', 'tests']
import decomposed_kernels as K, thread_ranks, parcels_b200 as pb
from parcels_b200 import distributed as D
case = K.make_case('rk45', n=10, interp='curv_linear')
with pytest.raises(NotImplementedError, match='AdvectionRK45 is implemented for'):
    D.decomposed_plan(K.decomposed_fieldset(case, 0, 2), case['kernels'], case['full'])
case = K.make_case('rk4', n=10, interp='curv_cgrid')
dfs = K.decomposed_fieldset(case, 0, 2)
with pytest.raises(NotImplementedError, match='U, V and W only'):
    dfs.add_field('Kh_zonal', case['f']['U'])
with pytest.raises(AttributeError, match='Kh_zonal'):
    D.decomposed_plan(dfs, [pb.AdvectionDiffusionM1, pb.DeleteParticle], case['full'])
one = {k: v[:1].copy() for k, v in case['full'].items()}
slabs = [dfs, K.decomposed_fieldset(case, 1, 2)]
with pytest.raises(NotImplementedError, match='ONE particle'):
    thread_ranks.run_ranks(2, lambda r, dist: D.execute_decomposed(slabs[r], D.shard_particles(one, r, 2), case['kernels'], case['dt'],
                                                                   case['endtime'], dist))
print('REFUSED')
"""
