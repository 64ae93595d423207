"""Device-side spatial-hash build (csrc/hashbuild.cu: count -> scan -> expand -> radix sort -> CSR) against the host
restatement of the reference's table (parcels_b200/spatialhash.py, itself pinned to the reference's own SpatialHash by
tests/test_oracle_vs_reference.py): keys, starts, counts and faces bit-identical, and curvilinear runs give the same
trajectories with either table."""

import numpy as np
import pytest

import cases
from engine_run import make_fieldset, run_engine
from oracle_run import load_case
from parcels_b200.spatialhash import build_spatial_hash

pytestmark = pytest.mark.gpu


def _meshes():
    for ny, nx, sph, cd in ((23, 31, False, "f8"), (33, 41, True, "f8"), (23, 31, True, "f4"), (120, 170, True, "f4")):
        yield (ny, nx, sph, cd), cases.curv_mesh(ny, nx, sph, np.dtype(cd))


@pytest.mark.parametrize("spec", [m[0] for m in _meshes()])
def test_device_table_equals_host_table(spec):
    import parcels_b200 as pb

    ny, nx, sph, cd = spec
    lon, lat = cases.curv_mesh(ny, nx, sph, np.dtype(cd))
    U = np.zeros((1, 1, ny, nx), dtype=np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, U=U, V=U, mesh="spherical" if sph else "flat", interp_method="cgrid_velocity")
    assert "keys" not in fs.grid.get_spatial_hash()  # the product path hands over the boxes only
    dev = fs.engine(0).hash_table()
    host = build_spatial_hash(lon, lat, sph, table=True)
    assert len(dev["faces"]) == host["n_entries"]
    for k in ("keys", "starts", "counts", "faces"):
        np.testing.assert_array_equal(dev[k], host[k], err_msg=k)


def test_host_table_route_gives_identical_trajectories():
    c = load_case("curv_sph_2d")
    ps_dev, err = run_engine(c)
    assert err == ""
    import parcels_b200 as pb

    fs = make_fieldset(c)
    fs.grid.get_spatial_hash(table=True)  # upload the NumPy-built table instead
    ps = pb.ParticleSet(fs, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    ps.execute([pb.AdvectionRK4, pb.DeleteParticle], dt=c["dt"], **c["segments"][0])
    for k in ("particle_id", "state", "t", "ei", "x", "y"):
        np.testing.assert_array_equal(ps._data[k], ps_dev._data[k], err_msg=k)


def test_device_table_equals_host_table_at_tens_of_millions_of_entries():
    """The device build's cub scan and radix sort at a size no other case reaches: a 3000 x 4000-node spherical mesh (about
    1.2e7 faces, 2.7e7 table entries, well above ORCA025's 1.27e7).  Under the host simulation a 300 x 400 mesh (logic only)."""
    import os

    import parcels_b200 as pb

    ny, nx = (300, 400) if os.environ.get("PB_HOSTSIM_TEST") == "1" else (3000, 4000)
    lon, lat = cases.curv_mesh(ny, nx, True, np.dtype("f8"))
    U = np.zeros((1, 1, ny, nx), dtype=np.float32)
    fs = pb.FieldSet.from_arrays(lon=lon, lat=lat, U=U, V=U, mesh="spherical", interp_method="cgrid_velocity")
    dev = fs.engine(0).hash_table()
    host = build_spatial_hash(lon, lat, True, table=True)
    if ny == 3000:
        assert host["n_entries"] > 2.5e7
    assert len(dev["faces"]) == host["n_entries"]
    for k in ("keys", "starts", "counts", "faces"):
        np.testing.assert_array_equal(dev[k], host[k], err_msg=k)
