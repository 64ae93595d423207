"""TEST INFRASTRUCTURE ONLY -- the oracle's trigonometry, one method per call site.

The oracle restates the reference's IEEE operations in the reference's order and dtypes; the only operations whose last bit
depends on the library are the sin / cos below.  ``NumpyTrig`` (the default) returns exactly the NumPy expressions of the
reference, so the oracle stays bit-identical to the reference (tests/test_oracle_golden.py, tests/test_oracle_vs_reference.py).
A test may install another provider with ``use(...)`` -- e.g. one that evaluates the engine's own device functions
(tests/device_trig.py) -- to pin the kernels' remaining arithmetic bit for bit.  Arguments are radians, in the dtype the
reference evaluates them in; every method returns that dtype.

The two hooks at the end are not trigonometry: they are the two places where the reference is not reproducible to the last
bit by itself (DESIGN.md waivers 4 and 8).  The default keeps the reference's behaviour.
"""

from __future__ import annotations

import contextlib

import numpy as np


class NumpyTrig:
    """The reference's own expressions."""

    # A-grid unit conversion, XLinear and the slip interpolators (_xinterpolators.py:182-184, _Spatialslip): cos(deg2rad(y))
    def agrid_conv(self, lat):
        return np.cos(lat)

    # DiffusionUniformKh's metric (_advectiondiffusion.py:11-13): cos(y * pi / 180)
    def kh_metric(self, lat):
        return np.cos(lat)

    # AdvectionDiffusionM1 / EM's metric (the same meters_to_degrees_zonal)
    def m1em_metric(self, lat):
        return np.cos(lat)

    # curvilinear point-in-cell: the four corners of a cell on the unit sphere (index_search.py:180-239)
    def curv_corners(self, lat, lon):
        return np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)

    # curvilinear point-in-cell: the query point on the unit sphere (index_search.py:180-239)
    def curv_query(self, lat, lon):
        return np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)

    # spatial-hash query: the sampled point on the unit sphere, in the position's dtype (spatialhash.py:417-421)
    def hash_query(self, lat, lon):
        return np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)

    # CGrid_Velocity edge length (_geodetic_distance, utils/interpolation.py:178-185): cos of the mid-edge latitude
    def edge_length(self, lat):
        return np.cos(lat)

    # CGrid_Velocity unit conversion (_xinterpolators.py:193-332): cos(deg2rad(y))
    def cgrid_conv(self, lat):
        return np.cos(lat)

    # -- not trigonometry: the reference's own irreproducible last bits --
    # waiver 8: np.einsum("ij,ji->i", phi, p) (mid-edge latitudes, Jacobian)
    def einsum_rows(self, phi, p):
        return np.einsum("ij,ji->i", phi, p)

    # waiver 4: (xsi, eta) of a first, un-hinted curvilinear search -- float32-typed in the reference
    def unhinted_coords(self, coords):
        return coords


_CURRENT = [NumpyTrig()]


def current():
    return _CURRENT[-1]


@contextlib.contextmanager
def use(provider):
    """Evaluate the oracle with `provider` inside the block."""
    _CURRENT.append(provider)
    try:
        yield provider
    finally:
        _CURRENT.pop()
