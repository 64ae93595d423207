"""The oracle in "engine arithmetic" mode: every sin / cos of the oracle (oracle/trig.py) evaluated by the very device function
the kernels call at the matching site (pb_debug_math), and the engine's documented resolution of the reference's two
irreproducible last bits (DESIGN.md waivers 4 and 8).  With it the oracle computes what the kernels compute, bit for bit, on
spherical and curvilinear meshes too -- as `philox_ref.device_normals` does for the Wiener increments.

Which device function each site uses (parcels_b200/csrc):
  * A-grid unit conversion (agrid.cuh XLinear / slip, afast.cu `spherical`, cgrid.cuh curvilinear XLinear): cos_np in the
    dtype of the sampled latitude -- CUDA's cosf for float32, common.cuh's polynomial for float64;
  * DiffusionUniformKh (common.cuh fused block) and M1 / EM (advdiff.cu): cosf of the float32 latitude;
  * curvilinear cell corners (cgrid.cuh project_cell, the per-cell table): CUDA's float64 cos / sin;
  * curvilinear query vector (cgrid.cuh eval_rt / sample_scalar_curv_kernel): cos_np(lat), sincos_lon(lon), sin_lat(lat);
  * spatial-hash query (cgrid.cuh hash_coords): cosf / sinf of a float32 position; a float64 position reuses the query vector
    in the advection / velocity kernels (hash_coords_xyz) and takes cosx / sinx -- cos_np, CUDA's sin -- in the scalar
    sampler (`scalar_sampler=True`);
  * C-grid edge length and unit conversion (cgrid.cuh edge_length, cgrid_finish callers): cosx in the value's dtype -- cosf
    for float32, cos_np for float64.
"""

from __future__ import annotations

import numpy as np

from oracle import trig

_ENGINE = {}


def _engine(device=0):
    from parcels_b200.engine import Engine

    if device not in _ENGINE:
        _ENGINE[device] = Engine(device)
    return _ENGINE[device]


def dev(op, x, out=0):
    """Device op `op` of pb_debug_math on x, element by element; float32 ops take and return float32."""
    x = np.asarray(x)
    f32 = op in ("cosf", "sinf")
    if f32 and x.dtype != np.float32:
        raise TypeError(f"{op} of a {x.dtype} argument")
    r = _engine().debug_math(op, x.astype(np.float64))[:, out].reshape(x.shape)
    return r.astype(np.float32) if f32 else r


def _cos_in_dtype(x):
    """cosx / cos_np of the kernels: CUDA's cosf for float32, the cos_np polynomial for float64."""
    x = np.asarray(x)
    if x.dtype == np.float32:
        return dev("cosf", x)
    if x.dtype == np.float64:
        return dev("cos_np", x)
    raise TypeError(f"cos of a {x.dtype} argument")


def _query_vector(lat, lon):
    lat, lon = np.asarray(lat, dtype=np.float64), np.asarray(lon, dtype=np.float64)
    cl = dev("cos_np", lat)
    sl, cl2 = dev("sincos_lon", lon, 0), dev("sincos_lon", lon, 1)
    return cl2 * cl, sl * cl, dev("sin_lat", lat)


class DeviceTrig(trig.NumpyTrig):
    """Engine arithmetic for the oracle: use with `oracle.trig.use(DeviceTrig())`."""

    def __init__(self, scalar_sampler=False):
        self.scalar_sampler = scalar_sampler

    def agrid_conv(self, lat):
        return _cos_in_dtype(lat)

    def kh_metric(self, lat):
        return dev("cosf", lat)

    def m1em_metric(self, lat):
        return dev("cosf", lat)

    def curv_corners(self, lat, lon):
        cl = dev("cos", lat)
        return dev("cos", lon) * cl, dev("sin", lon) * cl, dev("sin", lat)

    def curv_query(self, lat, lon):
        return _query_vector(lat, lon)

    def hash_query(self, lat, lon):
        lat, lon = np.asarray(lat), np.asarray(lon)
        if lat.dtype == np.float32 and lon.dtype == np.float32:
            cl = dev("cosf", lat)
            return dev("cosf", lon) * cl, dev("sinf", lon) * cl, dev("sinf", lat)
        if lat.dtype != np.float64 or lon.dtype != np.float64:
            raise TypeError(f"hash query of {lat.dtype} / {lon.dtype} positions")
        if not self.scalar_sampler:
            return _query_vector(lat, lon)
        cl = dev("cos_np", lat)
        return dev("cos_np", lon) * cl, dev("sin", lon) * cl, dev("sin", lat)

    def edge_length(self, lat):
        return _cos_in_dtype(lat)

    def cgrid_conv(self, lat):
        return _cos_in_dtype(lat)

    def einsum_rows(self, phi, p):
        # waiver 8: the engine sums the four products left to right (cgrid.cuh cgrid_finish), which is what np.einsum does when
        # its operands share a dtype; with mixed dtypes, or a batch of one row, NumPy's own last bits change with the batch
        acc = phi[:, 0] * p[0]
        for k in range(1, 4):
            acc = acc + phi[:, k] * p[k]
        return acc

    def unhinted_coords(self, coords):
        # waiver 4: the engine carries the float32-rounded (xsi, eta) of an un-hinted search in float64 arithmetic
        return coords.astype(np.float64)
