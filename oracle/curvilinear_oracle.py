"""TEST INFRASTRUCTURE ONLY -- oracle for the curvilinear / C-grid rows of the hot path
(SURVEY.md 8a rows a12-a14): curvilinear cell search with hint + spatial-hash fallback, and the
``CGrid_Velocity`` interpolator.  NumPy restatement of the reference with the same operations,
order and dtypes; every function cites the reference file:line (relative to
``/root/reference/src/parcels``).  Pinned bit-exact against the reference's own code by
``tests/test_oracle_vs_reference.py`` / ``tests/golden/ref_cases.npz`` and against the v3-JIT
``cgrid_velocity`` goldens.  See ``parcels_oracle.py`` for who may import this.
"""

from __future__ import annotations

import numpy as np

from . import trig

GRID_SEARCH_ERROR = -3

# ----------------------------------------------------------------------------------------------
# point-in-cell: closed-form bilinear inverse, in a per-cell tangent plane on spherical meshes
# ----------------------------------------------------------------------------------------------
_INV_A = np.array([[1, 0, 0, 0], [-1, 1, 0, 0], [-1, 0, 0, 1], [1, -1, 1, -1]])  # index_search.py:122-129


def latlon_rad_to_xyz(lat, lon):
    """_core/index_search.py:439-450."""
    return np.cos(lon) * np.cos(lat), np.sin(lon) * np.cos(lat), np.sin(lat)


def bilinear_inverse(px, py, xq, yq):
    """_core/index_search.py:132-149: (xsi, eta) with bilinear blend of the corners == query."""
    minus_one = -1.0 * np.ones(len(xq), dtype=float)
    a, b = np.dot(_INV_A, px), np.dot(_INV_A, py)
    aa = a[3] * b[2] - a[2] * b[3]
    bb = a[3] * b[0] - a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + xq * b[3] - yq * a[3]
    cc = a[1] * b[0] - a[0] * b[1] + xq * b[1] - yq * a[1]
    det2 = bb * bb - 4 * aa * cc
    with np.errstate(divide="ignore", invalid="ignore"):
        det = np.where(det2 > 0, np.sqrt(det2), minus_one)
        eta = np.where(abs(aa) < 1e-12, -cc / bb, np.where(det2 > 0, (-bb + det) / (2 * aa), minus_one))
        xsi = np.where(
            abs(a[1] + a[3] * eta) < 1e-12,
            ((yq - py[0]) / (py[1] - py[0]) + (yq - py[3]) / (py[2] - py[3])) * 0.5,
            (xq - a[0] - a[2] * eta) / (a[1] + a[3] * eta),
        )
    return xsi, eta


def project_cell_and_query(clon, clat, x, y):
    """_core/index_search.py:180-239: corners and query on the cell's own tangent plane."""
    cX, cY, cZ = trig.current().curv_corners(np.deg2rad(clat), np.deg2rad(clon))
    qX, qY, qZ = trig.current().curv_query(np.deg2rad(np.asarray(y, dtype=float)), np.deg2rad(np.asarray(x, dtype=float)))
    ux = (cX[1] + cX[2]) - (cX[0] + cX[3])
    uy = (cY[1] + cY[2]) - (cY[0] + cY[3])
    uz = (cZ[1] + cZ[2]) - (cZ[0] + cZ[3])
    un = np.sqrt(ux * ux + uy * uy + uz * uz)
    un = np.where(un == 0.0, 1.0, un)
    eux, euy, euz = ux / un, uy / un, uz / un
    vx = (cX[2] + cX[3]) - (cX[0] + cX[1])
    vy = (cY[2] + cY[3]) - (cY[0] + cY[1])
    vz = (cZ[2] + cZ[3]) - (cZ[0] + cZ[1])
    d = vx * eux + vy * euy + vz * euz  # Gram-Schmidt
    vx = vx - d * eux
    vy = vy - d * euy
    vz = vz - d * euz
    vn = np.sqrt(vx * vx + vy * vy + vz * vz)
    vn = np.where(vn == 0.0, 1.0, vn)
    evx, evy, evz = vx / vn, vy / vn, vz / vn

    def proj(ax, ay, az):
        return ax * eux + ay * euy + az * euz, ax * evx + ay * evy + az * evz

    pu, pv = proj(cX, cY, cZ)
    qu, qv = proj(qX, qY, qZ)
    return pu, pv, qu, qv


def point_in_cell(grid, y, x, yi, xi):
    """_core/index_search.py:94-119 (``curvilinear_point_in_cell``): corners CCW from (yi, xi)."""
    lon, lat = grid.lon, grid.lat
    clon = np.asarray([lon[yi, xi], lon[yi, xi + 1], lon[yi + 1, xi + 1], lon[yi + 1, xi]], dtype=float)
    clat = np.asarray([lat[yi, xi], lat[yi, xi + 1], lat[yi + 1, xi + 1], lat[yi + 1, xi]], dtype=float)
    if grid.spherical:
        px, py, xq, yq = project_cell_and_query(clon, clat, x, y)
        xsi, eta = bilinear_inverse(px, py, xq, yq)
    else:  # raw lon/lat, no antimeridian shift (index_search.py:115-116,152-168)
        xsi, eta = bilinear_inverse(clon.copy(), clat, np.asarray(x, dtype=float).copy(), np.asarray(y, dtype=float))
    inside = np.where((xsi >= 0) & (xsi <= 1) & (eta >= 0) & (eta <= 1), 1, 0)
    return inside, np.column_stack((xsi, eta))


# ----------------------------------------------------------------------------------------------
# spatial hash (Morton-keyed CSR table over the faces' bounding boxes)
# ----------------------------------------------------------------------------------------------
_ENTRIES_PER_FACE = 16  # spatialhash.py:24-26
_ENTRY_BUDGET_MIN = 2**22
_MAX_BITWIDTH = 1023


def quantize(x, y, z, box, bitwidth):
    """_core/spatialhash.py:647-695 (``quantize_coordinates``)."""
    xmin, xmax, ymin, ymax, zmin, zmax = box
    x, y, z = np.asarray(x), np.asarray(y), np.asarray(z)
    dx, dy, dz = xmax - xmin, ymax - ymin, zmax - zmin
    with np.errstate(invalid="ignore"):
        xn = np.where(dx != 0, (x - xmin) / dx, 0.0)
        yn = np.where(dy != 0, (y - ymin) / dy, 0.0)
        zn = np.where(dz != 0, (z - zmin) / dz, 0.0)
        xq = np.clip(xn * bitwidth, 0, bitwidth).astype(np.uint32)
        yq = np.clip(yn * bitwidth, 0, bitwidth).astype(np.uint32)
        zq = np.clip(zn * bitwidth, 0, bitwidth).astype(np.uint32)
    return xq, yq, zq


def dilate10(n):
    """_core/spatialhash.py:554-597 (``_dilate_bits``)."""
    n = np.asarray(n, dtype=np.uint32)
    n &= np.uint32(0x000003FF)
    n = (n | (n << np.uint32(16))) & np.uint32(0xFF0000FF)
    n = (n | (n << np.uint32(8))) & np.uint32(0x0300F00F)
    n = (n | (n << np.uint32(4))) & np.uint32(0x030C30C3)
    n = (n | (n << np.uint32(2))) & np.uint32(0x09249249)
    return n


def morton3(xq, yq, zq):
    """_core/spatialhash.py:698-716: x0,y0,z0,x1,y1,z1,... from the LSB upward."""
    return ((dilate10(zq) << 2) | (dilate10(yq) << 1) | dilate10(xq)).astype(np.uint32)


class OHash:
    """_core/spatialhash.py:29-535 for an XGrid with 2-D lon/lat."""

    def __init__(self, grid):
        self.grid = grid
        lon2, lat2 = grid.lon, grid.lat
        if grid.spherical:  # :59-107
            x, y, z = latlon_rad_to_xyz(np.deg2rad(lat2), np.deg2rad(lon2))
            self.box = (np.nanmin(x), np.nanmax(x), np.nanmin(y), np.nanmax(y), np.nanmin(z), np.nanmax(z))
        else:  # :127-163
            x, y, z = lon2, lat2, None
            self.box = (np.nanmin(x), np.nanmax(x), np.nanmin(y), np.nanmax(y), 0.0, 0.0)

        def lowhigh(a):
            st = np.stack((a[:-1, :-1], a[:-1, 1:], a[1:, 1:], a[1:, :-1]), axis=-1)
            return np.min(st, axis=-1), np.max(st, axis=-1)

        self.xlow, self.xhigh = lowhigh(x)
        self.ylow, self.yhigh = lowhigh(y)
        if z is not None:
            self.zlow, self.zhigh = lowhigh(z)
        else:
            self.zlow, self.zhigh = np.zeros_like(self.xlow), np.zeros_like(self.xlow)
        self.shape = self.xlow.shape
        self.valid = ~(np.isnan(self.xlow) | np.isnan(self.xhigh) | np.isnan(self.ylow) | np.isnan(self.yhigh)
                       | np.isnan(self.zlow) | np.isnan(self.zhigh))  # fmt: skip
        self.bitwidth = _MAX_BITWIDTH
        budget = max(_ENTRIES_PER_FACE * np.size(self.xlow), _ENTRY_BUDGET_MIN)  # :212-228
        if self._total_entries(self.bitwidth) > budget:
            lo, hi = 1, self.bitwidth
            while lo < hi:
                mid = (lo + hi + 1) // 2
                if self._total_entries(mid) <= budget:
                    lo = mid
                else:
                    hi = mid - 1
            self.bitwidth = lo
        self._build()

    def _qboxes(self, bitwidth):
        lo = quantize(self.xlow, self.ylow, self.zlow, self.box, bitwidth)
        hi = quantize(self.xhigh, self.yhigh, self.zhigh, self.box, bitwidth)
        return lo, hi

    def _total_entries(self, bitwidth):  # :232-267
        (xl, yl, zl), (xh, yh, zh) = self._qboxes(bitwidth)
        nx = xh.astype(np.int64) - xl + 1
        ny = yh.astype(np.int64) - yl + 1
        nz = zh.astype(np.int64) - zl + 1
        return int(np.where(self.valid, nx * ny * nz, 0).sum())

    def _build(self):  # :269-387
        (xl, yl, zl), (xh, yh, zh) = self._qboxes(self.bitwidth)
        xl, yl, zl, xh, yh, zh = (a.ravel().astype(np.int32) for a in (xl, yl, zl, xh, yh, zh))
        nx, ny, nz = xh - xl + 1, yh - yl + 1, zh - zl + 1
        per_face = np.where(self.valid.ravel(), nx * ny * nz, 0).astype(np.int32)
        total = int(per_face.sum(dtype=np.int64))
        nface = np.size(self.xlow)
        face_ids = np.repeat(np.arange(nface, dtype=np.uint32), per_face)
        face_starts = np.concatenate(([0], np.cumsum(per_face, dtype=np.int64)))[:-1]
        intra = np.arange(total, dtype=np.int64) - np.repeat(face_starts, per_face)
        ny_nz = np.repeat(ny * nz, per_face)
        nz_rep = np.repeat(nz, per_face)
        xi = intra // ny_nz
        rem = intra % ny_nz
        yi = rem // nz_rep
        zi = rem % nz_rep
        codes = morton3(np.repeat(xl, per_face) + xi, np.repeat(yl, per_face) + yi, np.repeat(zl, per_face) + zi)
        packed = (codes.astype(np.uint64) << np.uint64(32)) | face_ids
        packed.sort()
        self.faces = packed.astype(np.uint32)
        sorted_codes = (packed >> np.uint64(32)).astype(np.uint32)
        self.starts = np.concatenate(([0], np.flatnonzero(sorted_codes[1:] != sorted_codes[:-1]) + 1))
        self.keys = sorted_codes[self.starts]
        self.counts = np.diff(np.concatenate((self.starts, [sorted_codes.size])))

    def query(self, y, x):  # :389-535
        y, x = np.asarray(y), np.asarray(x)
        if self.grid.spherical:
            qx, qy, qz = trig.current().hash_query(np.deg2rad(y), np.deg2rad(x))
        else:
            qx, qy, qz = x, y, np.zeros_like(x)
        codes = morton3(*quantize(qx, qy, qz, self.box, self.bitwidth)).ravel()
        nq = codes.size
        pos = np.searchsorted(self.keys, codes)
        valid = (pos < len(self.keys)) & np.isfinite(x) & np.isfinite(y)
        pos = np.clip(pos, 0, len(self.keys) - 1)
        valid[valid] &= codes[valid] == self.keys[pos[valid]]
        j_best = np.full(nq, GRID_SEARCH_ERROR, dtype=np.int32)
        i_best = np.full(nq, GRID_SEARCH_ERROR, dtype=np.int32)
        hits = np.where(valid, self.counts[pos], 0).astype(np.int32)
        if hits.sum() == 0:
            return j_best, i_best, np.full((nq, 2), -1.0, dtype=np.float32)
        owner = np.repeat(np.arange(nq, dtype=np.int32), hits)
        offsets = np.concatenate(([0], np.cumsum(hits))).astype(np.int32)
        total = int(offsets[-1])
        intra = np.arange(total, dtype=np.int32) - np.repeat(offsets[:-1], hits)
        src = self.starts[pos[owner]].astype(np.int32) + intra
        j_all, i_all = np.unravel_index(self.faces[src], self.shape)
        inside, coords = point_in_cell(self.grid, np.repeat(y, hits), np.repeat(x, hits), j_all, i_all)
        best = np.full((nq, 2), -1.0, dtype=np.float32)
        f_idx = np.flatnonzero(inside)
        q = np.searchsorted(offsets[1:], f_idx, side="right")
        uq, first = np.unique(q, return_index=True)
        keep = (hits > 0)[uq]
        if keep.any():
            uq = uq[keep]
            p = f_idx[first[keep]]
            j_best[uq] = j_all[p]
            i_best[uq] = i_all[p]
            best[uq] = coords[p]  # float64 -> float32 store (spatialhash.py:511,529)
        return j_best, i_best, best


def get_hash(grid):
    if grid.hash is None:
        grid.hash = OHash(grid)
    return grid.hash


def search_indices_curvilinear_2d(grid, y, x, yi=None, xi=None):
    """_core/index_search.py:242-295."""
    hinted = bool(np.any(xi))
    if hinted:
        inside, coords = point_in_cell(grid, y, x, yi, xi)
        y_check, x_check = y[inside == 0], x[inside == 0]
        miss = np.where(inside == 0)[0]
    else:
        yi = np.full(len(y), GRID_SEARCH_ERROR, dtype=np.int32)
        xi = np.full(len(x), GRID_SEARCH_ERROR, dtype=np.int32)
        y_check, x_check = y, x
        coords = -1.0 * np.ones((len(y), 2), dtype=np.float32)
        miss = np.arange(len(y))
    if len(miss) > 0:
        yq, xq, cq = get_hash(grid).query(y_check, x_check)
        coords[miss, :] = cq
        yi[miss] = yq
        xi[miss] = xq
    if not hinted:
        coords = trig.current().unhinted_coords(coords)
    return yi, coords[:, 1], xi, coords[:, 0]


# ----------------------------------------------------------------------------------------------
# CGrid_Velocity
# ----------------------------------------------------------------------------------------------
def _phi2d(eta, xsi):
    """_core/utils/interpolation.py:25-31 (``phi2D_lin``)."""
    return np.column_stack([(1 - xsi) * (1 - eta), xsi * (1 - eta), xsi * eta, (1 - xsi) * eta])


def _edge_length(lat1, lat2, lon1, lon2, spherical, lat, deg2m):
    """_core/utils/interpolation.py:178-185 (``_geodetic_distance``)."""
    if spherical:
        rad = np.pi / 180.0
        return np.sqrt(((lon2 - lon1) * deg2m * trig.current().edge_length(rad * lat)) ** 2 + ((lat2 - lat1) * deg2m) ** 2)
    return np.sqrt((lon2 - lon1) ** 2 + (lat2 - lat1) ** 2)


def _jacobian(py, px, eta, xsi):
    """_core/utils/interpolation.py:188-198."""
    dphidxsi = np.column_stack([eta - 1, 1 - eta, eta, -eta])
    dphideta = np.column_stack([xsi - 1, -xsi, xsi, 1 - xsi])
    rows = trig.current().einsum_rows
    dxdxsi = rows(dphidxsi, px)
    dxdeta = rows(dphideta, px)
    dydxsi = rows(dphidxsi, py)
    dydeta = rows(dphideta, py)
    return dxdxsi * dydeta - dxdeta * dydxsi


def _take(data, ti, zi, yi, xi):
    T, Z, Y, X = data.shape
    ti = ti if T > 1 else np.zeros_like(ti)
    zi = zi if Z > 1 else np.zeros_like(zi)
    yi = yi if Y > 1 else np.zeros_like(yi)
    xi = xi if X > 1 else np.zeros_like(xi)
    return data[ti, zi, yi, xi]


def cgrid_velocity(fs, pos, gp):
    """interpolators/_xinterpolators.py:193-332 (``CGrid_Velocity.interp``)."""
    (ti, tau), (zi, zeta), (yi, eta), (xi, xsi) = gp
    grid = fs.grid
    U, V = fs.U, fs.V
    off = grid.offsets
    tdim, zdim, ydim, xdim = U.shape
    two_t = bool(np.any(tau > 0))
    lon, lat = grid.lon, grid.lat
    if lon.ndim == 1:
        px = np.array([lon[xi], lon[xi + 1], lon[xi + 1], lon[xi]])
        py = np.array([lat[yi], lat[yi], lat[yi + 1], lat[yi + 1]])
    else:
        px = np.array([lon[yi, xi], lon[yi, xi + 1], lon[yi + 1, xi + 1], lon[yi + 1, xi]])
        py = np.array([lat[yi, xi], lat[yi, xi + 1], lat[yi + 1, xi + 1], lat[yi + 1, xi]])
    if grid.spherical:
        px = ((px + 180.0) % 360.0) - 180.0
        px[1:] = np.where(px[1:] - px[0] > 180, px[1:] - 360, px[1:])
        px[1:] = np.where(-px[1:] + px[0] > 180, px[1:] + 360, px[1:])
    sph, d2m = grid.spherical, grid.deg2m
    rows = trig.current().einsum_rows
    c1 = _edge_length(py[0], py[1], px[0], px[1], sph, rows(_phi2d(0.0, xsi), py), d2m)
    c2 = _edge_length(py[1], py[2], px[1], px[2], sph, rows(_phi2d(eta, 1.0), py), d2m)
    c3 = _edge_length(py[2], py[3], px[2], px[3], sph, rows(_phi2d(1.0, xsi), py), d2m)
    c4 = _edge_length(py[3], py[0], px[3], px[0], sph, rows(_phi2d(eta, 0.0), py), d2m)
    t_lv = (ti, np.clip(ti + 1, 0, tdim - 1)) if two_t else (ti,)

    def two_faces(data, zs, ys, xs):
        """the two bracketing face values, reduced over time (:256-275)."""
        c = np.array([[_take(data, t, z, y, x) for (z, y, x) in zip(zs, ys, xs, strict=True)] for t in t_lv])
        if two_t:
            w = tau[np.newaxis, :]
            return c[0, :] * (1 - w) + c[1, :] * w
        return c[0, :]

    yi_o = np.clip(yi + off["Y"], 0, ydim - 1)
    xi_1 = np.clip(xi + 1, 0, xdim - 1)
    cu = two_faces(U, (zi, zi), (yi_o, yi_o), (xi, xi_1))
    U0 = cu[0, :] * c4
    U1 = cu[1, :] * c2
    Uvel = (1 - xsi) * U0 + xsi * U1
    yi_1 = np.clip(yi + 1, 0, ydim - 1)
    xi_o = np.clip(xi + off["X"], 0, xdim - 1)
    cv = two_faces(V, (zi, zi), (yi, yi_1), (xi_o, xi_o))
    V0 = cv[0, :] * c1
    V1 = cv[1, :] * c3
    Vvel = (1 - eta) * V0 + eta * V1
    jac = _jacobian(py, px, eta, xsi) * d2m if sph else _jacobian(py, px, eta, xsi)
    u = (
        (-(1 - eta) * Uvel - (1 - xsi) * Vvel) * px[0]
        + ((1 - eta) * Uvel - xsi * Vvel) * px[1]
        + (eta * Uvel + xsi * Vvel) * px[2]
        + (-eta * Uvel + (1 - xsi) * Vvel) * px[3]
    ) / jac
    v = (
        (-(1 - eta) * Uvel - (1 - xsi) * Vvel) * py[0]
        + ((1 - eta) * Uvel - xsi * Vvel) * py[1]
        + (eta * Uvel + xsi * Vvel) * py[2]
        + (-eta * Uvel + (1 - xsi) * Vvel) * py[3]
    ) / jac
    if sph:
        conv = d2m * trig.current().cgrid_conv(np.deg2rad(pos["y"]))
        u /= conv
        v /= conv
    if fs.W is not None:
        zi_0 = np.clip(zi + off["Z"], 0, zdim - 1)
        zi_1 = np.clip(zi + off["Z"] + 1, 0, zdim - 1)
        cw = two_faces(fs.W, (zi_0, zi_1), (yi_o, yi_o), (xi_o, xi_o))
        w = cw[0, :] * (1 - zeta) + cw[1, :] * zeta
    else:
        w = np.zeros_like(u)
    return u, v, w
