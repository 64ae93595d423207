"""CPU test (needs the reference's own Python package, oracle/ref_harness.py): the adapter reads a live reference FieldSet correctly."""

import numpy as np
import pytest

from oracle import ref_harness as rh
from oracle_run import load_case

pytestmark = pytest.mark.skipif(not rh.reference_available(), reason="the reference's own Python package is not importable (PARCELS_REFERENCE_SRC)")


def test_from_parcels_reads_reference_fieldset():
    from parcels_b200 import adapter

    c = load_case("diffusion")
    ref = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"],
                            mesh=c["mesh"], constants=c["constants"])  # fmt: skip
    fs = adapter.from_parcels(ref)
    np.testing.assert_array_equal(fs.grid.lon, c["lon"])
    np.testing.assert_array_equal(fs.grid.depth, c["depth"])
    assert fs.grid.is_spherical() and fs.grid.deg2m == ref.U.grid.deg2m
    assert (fs.grid.xdim, fs.grid.ydim, fs.grid.zdim) == (ref.U.grid.xdim, ref.U.grid.ydim, ref.U.grid.zdim)
    np.testing.assert_array_equal(fs._time_s, c["times"])
    np.testing.assert_array_equal(fs.W.data, c["W"])
    assert fs.constants == {"Kh_zonal": 100.0, "Kh_meridional": 50.0}
    assert len(fs.gridset) == len(ref.gridset) == 2
    rp = rh.make_pset(ref, x=c["x"], y=c["y"], z=c["z"], t=c["t"])
    ps = adapter.pset_from_parcels(rp, fs)
    assert ps._data is rp._data and ps._data["ei"].shape == (len(c["x"]), 2)


def test_from_parcels_curvilinear_cgrid_scalars_and_context():
    from parcels_b200 import adapter
    from parcels_b200.particleset import KernelPlan
    import parcels_b200 as pb

    c = load_case("curv_sph_2d")
    ref = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=c["W"],
                            mesh=c["mesh"], interp="cgrid_velocity", padding=c["padding"])  # fmt: skip
    fs = adapter.from_parcels(ref)
    assert fs.grid.curvilinear and fs.interp_method == "cgrid_velocity" and fs.offsets == (1, 1, 0)
    assert (fs.grid.xdim, fs.grid.ydim) == (ref.U.grid.xdim, ref.U.grid.ydim)
    np.testing.assert_array_equal(fs.grid.lon, c["lon"])

    c = load_case("flat_f32c_f64d")
    kz = np.abs(c["U"]) + 1
    ref = rh.build_fieldset(lon=c["lon"], lat=c["lat"], depth=c["depth"], times=c["times"], U=c["U"], V=c["V"], W=None,
                            mesh=c["mesh"], scalars={"Kh_zonal": (kz, "linear"), "Kh_meridional": (kz[:1], "linear")})  # fmt: skip
    ref.add_context("dres", 12.5)
    fs = adapter.from_parcels(ref)
    assert fs.context == {"dres": 12.5} and fs.Kh_zonal._slot == 3 and fs.Kh_meridional.data.shape[0] == 1
    k = rh.kernels()
    with pytest.raises(NotImplementedError, match="share dtype and time dimension"):
        KernelPlan([k.AdvectionDiffusionM1], fs)  # the reference's own kernel function is recognised as the built-in
    assert KernelPlan([k.AdvectionRK4, pb.DeleteParticle], fs).scheme == 4
