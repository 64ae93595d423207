"""The per-axis cell tables of float64 rectilinear grids (AxisCellRec, csrc/common.cuh) and the cell change of the specialised RK4
kernel (csrc/afast.cu) that reads them.

* The tables, read back from the device, hold {a[i], a[i+1], 1 / (a[i+1] - a[i])} with the reciprocal the same bits as the host's
  division: irregular lon / lat, a non-uniform depth axis, a time axis that does not start at 0, and two-node axes.
* Forward and backward trajectories on the ns_small and c2_small workloads of bench.py, with particles released exactly on cell
  faces of every axis and on the first time node, equal the generic kernel's bit for bit (both schedules of the fast kernel)."""

import os

import numpy as np
import pytest

import bench
import parcels_b200 as pb

pytestmark = pytest.mark.gpu

KEYS = ("particle_id", "state", "t", "ei", "x", "y", "z", "dx", "dy", "dz", "dt")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("shape", [(23, 17, 9, 4), (2, 2, 2, 2), (5, 3, 0, 2)], ids=["irregular", "two_nodes", "no_depth"])
def test_cell_tables_equal_the_host_division(shape):
    nx, ny, nz, nt = shape
    rng = np.random.default_rng(20261016)
    lon = np.sort(rng.uniform(-180.0, 180.0, nx))
    lat = np.linspace(-60.0, 70.0, ny) + rng.uniform(-0.3, 0.3, ny) * (130.0 / ny)
    depth = None if nz == 0 else 5500.0 * np.linspace(0.0, 1.0, nz) ** 1.8
    times = 1234.5 + np.cumsum(rng.uniform(1800.0, 7200.0, nt))
    sh = (nt, max(nz, 1), ny, nx)
    U = rng.uniform(-1, 1, sh).astype(np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, depth=depth, time=times, U=U, V=U, W=U if nz else None, mesh="spherical")
    try:
        eng = fs.engine(0)
        axes = {"lon": lon, "lat": lat, "time": times - times[0]}
        if nz:
            axes["depth"] = depth
        for name, a in axes.items():
            got = eng.debug_axis_cells(name, len(a))
            lo, hi = a[:-1], a[1:]
            np.testing.assert_array_equal(_bits(got[:, 0]), _bits(lo), err_msg=f"{name} lo")
            np.testing.assert_array_equal(_bits(got[:, 1]), _bits(hi), err_msg=f"{name} hi")
            np.testing.assert_array_equal(_bits(got[:, 2]), _bits(1.0 / (hi - lo)), err_msg=f"{name} 1 / (hi - lo)")
        if not nz:
            with pytest.raises(RuntimeError):
                eng.debug_axis_cells("depth", 2)
    finally:
        fs.release()


@pytest.fixture(scope="module", params=["ns_small", "c2_small"])
def workload(request):
    name = request.param
    w = bench.WORKLOADS[name]
    yield name, w, bench.build_field(name, w, host=True)


def _on_faces(field, n, seed):
    """particles exactly on nodes of lon / lat / depth (cell faces), mixed with interior positions"""
    rng = np.random.default_rng(seed)
    lon, lat, depth = (np.asarray(field[k], dtype=np.float64) for k in ("lon", "lat", "depth"))
    x, y = rng.uniform(-170, 170, n), rng.uniform(-70, 70, n)
    z = rng.uniform(5, 5000, n)
    ix = rng.integers(1, len(lon) - 1, n)
    iy = rng.integers(1, len(lat) - 1, n)
    iz = rng.integers(0, len(depth) - 1, n)
    sel = rng.random((3, n)) < 0.5
    x[sel[0]] = lon[ix[sel[0]]]
    y[sel[1]] = lat[iy[sel[1]]]
    z[sel[2]] = depth[iz[sel[2]]]
    return x, y, z


def _run(field, x, y, z, t, dt, runtime, fast):
    os.environ["PB_DISABLE_FAST_KERNEL"] = "0" if fast else "1"
    os.environ["PB_FAST_KERNEL"] = str(fast or 1)
    try:
        fs = pb.FieldSet.from_arrays(lon=field["lon"], lat=field["lat"], depth=field["depth"], time=field["times"], U=field["U"],
                                     V=field["V"], W=field["W"], mesh=field["mesh"])  # fmt: skip
        try:
            ps = pb.ParticleSet(fs, x=x, y=y, z=z, t=t, seed=5)
            ps.execute([pb.AdvectionRK4_3D, pb.DeleteParticle], dt=dt, runtime=runtime)
            rep = dict(ps.last_report)
            return {k: np.array(ps._data[k]) for k in KEYS}, rep
        finally:
            fs.release()
    finally:
        os.environ.pop("PB_DISABLE_FAST_KERNEL", None)
        os.environ.pop("PB_FAST_KERNEL", None)


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_trajectories_from_cell_faces_equal_the_generic_kernel(workload, direction):
    name, w, field = workload
    n = 4000
    x, y, z = _on_faces(field, n, 7 if direction == "forward" else 8)
    times = np.asarray(field["times"], dtype=np.float64)
    dt = w["dt"]
    if direction == "forward":
        t = np.zeros(n)  # the first time node
    else:
        dt = -dt
        t = np.full(n, times[-1] - times[0])
        t[: n // 8] = 0.0  # on the first time node, stepping out of the time interval
    runtime = 24 * abs(dt)
    ref, rref = _run(field, x, y, z, t, dt, runtime, fast=0)
    assert rref["kernel_variant"] == 0
    for version in (1, 2):
        got, rep = _run(field, x, y, z, t, dt, runtime, fast=version)
        assert rep["kernel_variant"] == version and rep["cache_refills"] > 0
        for k in KEYS:
            np.testing.assert_array_equal(got[k].view(np.uint8), ref[k].view(np.uint8), err_msg=f"{name} {direction} {k} (schedule {version})")
        for k in ("particle_steps", "n_error", "n_deleted", "first_error_iter", "n_out_of_time", "max_state"):
            assert rep[k] == rref[k], (k, rep[k], rref[k])
