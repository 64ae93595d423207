"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the hot path ``ParticleSet.execute(AdvectionRK4 | ...)``.

A NumPy restatement of the reference's (Parcels v4-alpha, ``/root/reference``) algorithm for the
path named in BASELINE.json's ``north_star``.  It deliberately uses the same NumPy operations in
the same order and with the same dtype promotion as the reference, so that it is bit-identical to
the reference's own code (pinned by ``tests/test_oracle_vs_reference.py`` through
``oracle/ref_harness.py`` and by the committed fixtures under ``tests/golden/``, which hold
outputs of the reference itself plus the reference's own known-answer tests).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import this module, and only as the checker / CPU baseline.  The product
(``parcels_b200``) never imports it and has no CPU fallback.

Every function cites the reference file:line it follows (paths relative to
``/root/reference/src/parcels``).
"""

from __future__ import annotations

import numpy as np

from . import trig

# --- status codes: _core/statuscodes.py:19-34 -------------------------------------------------
SUCCESS, END_OF_LOOP, EVALUATE, REPEAT, DELETE = 0, 1, 10, 20, 30
STOP_EXECUTION, STOP_ALL_EXECUTION = 40, 41
ERROR, ERROR_INTERPOLATION, ERROR_GRID_SEARCHING = 50, 51, 52
ERROR_OUT_OF_BOUNDS, ERROR_THROUGH_SURFACE, ERROR_OUTSIDE_TIME_INTERVAL = 60, 61, 70

# --- search sentinels: _core/index_search.py:15-17 --------------------------------------------
GRID_SEARCH_ERROR, LEFT_OUT_OF_BOUNDS, RIGHT_OUT_OF_BOUNDS = -3, -2, -1

EARTH_RADIUS = 6366707.019493707  # _core/mesh.py:6
DEG2M_EARTH = EARTH_RADIUS * np.pi / 180.0  # _core/mesh.py:37-40


class OutsideTimeInterval(RuntimeError):
    pass


class OracleParticleError(RuntimeError):
    """Raised where the reference raises a mapped exception (_core/kernel.py:239-245)."""

    def __init__(self, code, msg=""):
        super().__init__(f"particle error state {code} {msg}")
        self.code = code


# ----------------------------------------------------------------------------------------------
# Grid / fields (host-side description; equivalent of XGrid + ModelData for this path)
# ----------------------------------------------------------------------------------------------
class OGrid:
    """Structured grid: 1-D (rectilinear) or 2-D (curvilinear) lon/lat, 1-D depth.

    An axis that the grid does not have is ``None`` (``XGrid.axes``, _core/xgrid.py:145-147).
    ``xdim/ydim/zdim`` are *cell counts* (_core/xgrid.py:21-24,208-231): for LOW/HIGH padding
    with no face dimension in the dataset this is ``n_nodes - 1``; pass explicitly otherwise.
    """

    def __init__(self, lon=None, lat=None, depth=None, mesh="flat", radius=None, xdim=None, ydim=None, zdim=None,
                 offsets=(1, 1, 0)):
        self.lon = None if lon is None else np.asarray(lon)
        self.lat = None if lat is None else np.asarray(lat)
        self.depth = None if depth is None else np.asarray(depth)
        self.spherical = mesh == "spherical" or radius is not None
        # XGrid.deg2m (_core/xgrid.py:201-206): 1.0 on flat meshes
        self.deg2m = ((EARTH_RADIUS if radius is None else radius) * np.pi / 180.0) if self.spherical else 1.0
        self.curvilinear = self.lon is not None and self.lon.ndim == 2
        if self.lon is not None:
            nxn = self.lon.shape[-1]
            self.xdim = (nxn - 1) if xdim is None else xdim
        else:
            self.xdim = None
        if self.lat is not None:
            nyn = self.lat.shape[0]
            self.ydim = (nyn - 1) if ydim is None else ydim
        else:
            self.ydim = None
        if self.depth is not None:
            self.zdim = (len(self.depth) - 1) if zdim is None else zdim
        else:
            self.zdim = None
        # C-grid staggering offsets X, Y, Z (_xinterpolators.py:99-109): 1 for LOW padding else 0
        self.offsets = {"X": offsets[0], "Y": offsets[1], "Z": offsets[2]}
        self.hash = None

    @property
    def axes(self):
        out = []
        if self.depth is not None:
            out.append("Z")
        if self.lat is not None:
            out.append("Y")
        if self.lon is not None:
            out.append("X")
        return out


class OFieldSet:
    """U, V (, W) arrays laid out (T, Z, Y, X) on one grid, plus constant fields.

    ``time``: float64 seconds since the start of the time interval, or None for a field
    without a time dimension (``Field.time_interval`` is None, _core/field.py:112-117).
    ``interp``: "linear" (XLinear_Velocity) or "cgrid_velocity" (CGrid_Velocity).
    ``constants``: name -> value (``FieldSet.add_constant_field``, _core/fieldset.py:175-205);
    constant fields live on their own 1-node grid (_core/model.py:292-318), so ``ngrids`` is 2.
    """

    def __init__(self, grid: OGrid, U, V, W=None, time=None, interp="linear", constants=None, const_mesh=None):
        self.grid = grid
        self.U = np.asarray(U)
        self.V = np.asarray(V)
        self.W = None if W is None else np.asarray(W)
        self.time = None if time is None else np.asarray(time, dtype=np.float64)
        if self.time is not None and len(self.time) < 2:
            self.time = None  # model.py:511-515: a single time level => no time interval
        self.interp = interp
        self.context = {}  # FieldSet.add_context (_core/fieldset.py:207-222), e.g. RK45_tol / RK45_min_dt / RK45_max_dt
        self.constants = dict(constants or {})
        self.scalars = {}  # scalar fields on the same grid: name -> (array (T, Z, Y, X), "linear" | "nearest" | "cgrid_tracer")
        self.const_spherical = grid.spherical if const_mesh is None else (const_mesh == "spherical")
        self.const_deg2m = DEG2M_EARTH if self.const_spherical else 1.0

    @property
    def ngrids(self):
        return 2 if self.constants else 1


def create_particle_data(x, y, z, t, ngrids=1, dt=1.0, particle_ids=None):
    """SoA dict of the default Particle (_core/particle.py:123-222)."""
    x = np.asarray(x).flatten()
    n = x.size
    t = np.asarray(t, dtype=np.float64).flatten()
    if t.size == 1:
        t = np.repeat(t, n)
    return {
        "ei": np.zeros((n, ngrids), dtype=np.int32),
        "t": t.astype(np.float64),
        "z": np.asarray(z).flatten().astype(np.float32),
        "y": np.asarray(y).flatten().astype(np.float32),
        "x": x.astype(np.float32),
        "particle_id": (np.arange(n) if particle_ids is None else np.asarray(particle_ids)).astype(np.int64),
        "dz": np.zeros(n, dtype=np.float32),
        "dy": np.zeros(n, dtype=np.float32),
        "dx": np.zeros(n, dtype=np.float32),
        "dt": np.full(n, dt, dtype=np.float64),
        "state": np.full(n, EVALUATE, dtype=np.int32),
    }


class View:
    """Boolean-mask window on the SoA (_core/particlesetview.py): reads copy, writes go through."""

    def __init__(self, data, mask):
        object.__setattr__(self, "_d", data)
        object.__setattr__(self, "_m", mask)

    def __getattr__(self, name):
        return self._d[name][self._m]

    def __setattr__(self, name, value):
        self._d[name][self._m] = value

    def n(self):
        return int(np.count_nonzero(self._m))


# ----------------------------------------------------------------------------------------------
# Index search
# ----------------------------------------------------------------------------------------------
def search_1d(arr, x):
    """_core/index_search.py:20-62 (``_search_1d_array``)."""
    if len(arr) < 2:
        return np.zeros(shape=x.shape, dtype=np.int32), np.zeros_like(x)
    n = len(arr)
    idx = np.clip(np.searchsorted(arr, x, side="left") - 1, 0, n - 2)
    lo = arr[idx]
    hi = arr[np.clip(idx + 1, 1, n - 1)]
    b = (x - lo) / (hi - lo)
    idx = np.where(x < arr[0], LEFT_OUT_OF_BOUNDS, idx)
    idx = np.where(x > arr[-1], RIGHT_OUT_OF_BOUNDS, idx)
    return np.atleast_1d(idx), np.atleast_1d(b)


def search_time(time_flt, t):
    """_core/index_search.py:65-91 (``_search_time_index``) + TimeInterval check (utils/time.py:62-64)."""
    t = np.atleast_1d(t)
    if time_flt is None:
        return np.zeros(t.shape, dtype=np.int32), np.zeros(t.shape, dtype=np.float32)
    length = time_flt[-1] - time_flt[0]
    if not ((0 <= t).all() and (t <= length).all()):
        raise OutsideTimeInterval(str(t))
    return search_1d(time_flt - time_flt[0], t)


def ravel_index(grid: OGrid, zi, yi, xi):
    """_core/basegrid.py:83-118,259-278: ei = zi*ydim*xdim + yi*xdim + xi over the axes present."""
    dims, idx = [], []
    for ax, d, i in (("Z", grid.zdim, zi), ("Y", grid.ydim, yi), ("X", grid.xdim, xi)):
        if ax in grid.axes:
            dims.append(d)
            idx.append(np.asarray(i).astype(int))
    dims = np.array(dims, dtype=int)
    strides = np.cumprod(dims[::-1])[::-1]
    ei = 0
    for k in range(len(dims) - 1):
        ei = ei + idx[k] * strides[k + 1]
    return ei + idx[-1]


def unravel_index(grid: OGrid, ei):
    """_core/basegrid.py:120-152,219-256."""
    axes = grid.axes
    dims = np.array([{"Z": grid.zdim, "Y": grid.ydim, "X": grid.xdim}[a] for a in axes], dtype=int)
    strides = np.cumprod(dims[::-1])[::-1]
    out = {}
    ei = np.asarray(ei)
    for k in range(len(dims) - 1):
        out[axes[k]] = ei // strides[k + 1]
        ei = ei % strides[k + 1]
    out[axes[-1]] = ei
    return out


def grid_search(grid: OGrid, z, y, x, ei=None):
    """_core/xgrid.py:316-356 (``XGrid.search``)."""
    if grid.depth is not None:
        zi, zeta = search_1d(grid.depth, z)
    else:
        zi, zeta = np.zeros(z.shape, dtype=int), np.zeros(z.shape, dtype=float)
    if grid.curvilinear:
        from . import curvilinear_oracle as co

        yi0 = xi0 = None
        if ei is not None:
            hint = unravel_index(grid, ei)
            xi0, yi0 = hint.get("X"), hint.get("Y")
        yi, eta, xi, xsi = co.search_indices_curvilinear_2d(grid, y, x, yi0, xi0)
        return (zi, zeta), (yi, eta), (xi, xsi)
    if grid.lat is not None:
        yi, eta = search_1d(grid.lat, y)
    else:
        yi, eta = np.zeros(y.shape, dtype=int), np.zeros(y.shape, dtype=float)
    if grid.lon is not None:
        xi, xsi = search_1d(grid.lon, x)
    else:
        xi, xsi = np.zeros(x.shape, dtype=int), np.zeros(x.shape, dtype=float)
    return (zi, zeta), (yi, eta), (xi, xsi)


# ----------------------------------------------------------------------------------------------
# Interpolation
# ----------------------------------------------------------------------------------------------
def _take(data, ti, zi, yi, xi):
    """Pointwise gather ``data[ti, zi, yi, xi]``; size-1 (mock) dims are not indexed
    (_xinterpolators.py:61-75: an axis the field has no dimension for repeats its corner)."""
    T, Z, Y, X = data.shape
    ti = ti if T > 1 else np.zeros_like(ti)
    zi = zi if Z > 1 else np.zeros_like(zi)
    yi = yi if Y > 1 else np.zeros_like(yi)
    xi = xi if X > 1 else np.zeros_like(xi)
    return data[ti, zi, yi, xi]


def xlinear(data, ti, tau, zi, zeta, yi, eta, xi, xsi):
    """_xinterpolators.py:78-96,112-153 (``XLinear.interp`` on A-grid corner data).

    Negative sentinel indices wrap like NumPy fancy indexing does in the reference; the caller
    zeroes those values afterwards (_core/field.py:359-370).
    """
    T, Z, Y, X = data.shape
    two_t = bool(np.any(tau > 0))
    two_z = bool(np.any(zeta > 0))
    t_lv = (ti, np.clip(ti + 1, 0, T - 1)) if two_t else (ti,)
    z_lv = (zi, np.clip(zi + 1, 0, Z - 1)) if two_z else (zi,)
    y_lv = (yi, np.clip(yi + 1, 0, Y - 1))
    x_lv = (xi, np.clip(xi + 1, 0, X - 1))
    c = np.array([[[[_take(data, a, b, cc, d) for d in x_lv] for cc in y_lv] for b in z_lv] for a in t_lv])
    if two_t:
        w = tau[np.newaxis, :]
        c = c[0, :] * (1 - w) + c[1, :] * w
    else:
        c = c[0, :]
    if two_z:
        w = zeta[np.newaxis, :]
        c = c[0, :] * (1 - w) + c[1, :] * w
    else:
        c = c[0, :]
    return (
        (1 - xsi) * (1 - eta) * c[0, 0, :]
        + xsi * (1 - eta) * c[0, 1, :]
        + (1 - xsi) * eta * c[1, 0, :]
        + xsi * eta * c[1, 1, :]
    )


def xlinear_velocity(fs: OFieldSet, pos, gp):
    """_xinterpolators.py:169-190 (``XLinear_Velocity.interp``)."""
    (ti, tau), (zi, zeta), (yi, eta), (xi, xsi) = gp
    u = xlinear(fs.U, ti, tau, zi, zeta, yi, eta, xi, xsi)
    v = xlinear(fs.V, ti, tau, zi, zeta, yi, eta, xi, xsi)
    if fs.grid.spherical:
        u /= fs.grid.deg2m * trig.current().agrid_conv(np.deg2rad(pos["y"]))
        v /= fs.grid.deg2m
    if fs.W is not None:
        w = xlinear(fs.W, ti, tau, zi, zeta, yi, eta, xi, xsi)
    else:
        w = np.zeros_like(u)
    return u, v, w


def _corner_block(data, ti, tau, zi, zeta, yi, xi):
    """_xinterpolators.py:78-96 (``_get_corner_data_Agrid``): (lenT, lenZ, 2, 2, N)"""
    T, Z, Y, X = data.shape
    two_t = bool(np.any(tau > 0))
    two_z = bool(np.any(zeta > 0))
    t_lv = (ti, np.clip(ti + 1, 0, T - 1)) if two_t else (ti,)
    z_lv = (zi, np.clip(zi + 1, 0, Z - 1)) if two_z else (zi,)
    y_lv = (yi, np.clip(yi + 1, 0, Y - 1))
    x_lv = (xi, np.clip(xi + 1, 0, X - 1))
    return np.array([[[[_take(data, a, b, cc, d) for d in x_lv] for cc in y_lv] for b in z_lv] for a in t_lv]), two_z


def spatialslip_velocity(fs: OFieldSet, pos, gp, a, b):
    """_xinterpolators.py:385-480 (``_Spatialslip``; XFreeslip a=1, b=0; XPartialslip a=b=0.5): XLinear damped near
    land (cells whose corner velocities are all ~0 at the lower time level)."""
    (ti, tau), (zi, zeta), (yi, eta), (xi, xsi) = gp
    u = xlinear(fs.U, ti, tau, zi, zeta, yi, eta, xi, xsi)
    v = xlinear(fs.V, ti, tau, zi, zeta, yi, eta, xi, xsi)
    w = xlinear(fs.W, ti, tau, zi, zeta, yi, eta, xi, xsi) if fs.W is not None else None
    cU, two_z = _corner_block(fs.U, ti, tau, zi, zeta, yi, xi)
    cV, _ = _corner_block(fs.V, ti, tau, zi, zeta, yi, xi)

    def land(z_, y_, x_):
        return np.where(np.isclose(cU[0, z_, y_, x_, :], 0.0) & np.isclose(cV[0, z_, y_, x_, :], 0.0), True, False)

    def all_land(pairs):
        m = np.ones(len(xsi), dtype=bool)
        for y_, x_ in pairs:
            m &= land(0, y_, x_)
        if two_z:
            for y_, x_ in pairs:
                m &= land(1, y_, x_)
        return m

    def all_land_zz(pairs):  # the W factors always look at both Z levels (:460-470)
        m = np.ones(len(xsi), dtype=bool)
        for y_, x_ in pairs:
            m &= land(0, y_, x_) & land(1, y_, x_)
        return m

    f_u = np.ones_like(xsi)
    m = all_land([(0, 0), (0, 1)]) & (eta > 0)
    f_u[m] = f_u[m] * (a + b * eta[m]) / eta[m]
    m = all_land([(1, 0), (1, 1)]) & (eta < 1)
    f_u[m] = f_u[m] * (1 - b * eta[m]) / (1 - eta[m])
    u = u * f_u
    if fs.grid.spherical:
        u /= 1852 * 60 * trig.current().agrid_conv(np.deg2rad(pos["y"]))
    f_v = np.ones_like(eta)
    m = all_land([(0, 0), (1, 0)]) & (xsi > 0)
    f_v[m] = f_v[m] * (a + b * xsi[m]) / xsi[m]
    m = all_land([(0, 1), (1, 1)]) & (xsi < 1)
    f_v[m] = f_v[m] * (1 - b * xsi[m]) / (1 - xsi[m])
    v = v * f_v
    if fs.grid.spherical:
        v /= 1852 * 60
    if w is not None:
        f_w = np.ones_like(zeta)
        m = all_land_zz([(0, 0), (0, 1)]) & (eta > 0)
        f_w[m] = f_w[m] * (a + b * eta[m]) / eta[m]
        m = all_land_zz([(1, 0), (1, 1)]) & (eta < 1)
        f_w[m] = f_w[m] * (1 - b * eta[m]) / (1 - eta[m])
        m = all_land_zz([(0, 0), (1, 0)]) & (xsi > 0)
        f_w[m] = f_w[m] * (a + b * xsi[m]) / xsi[m]
        m = all_land_zz([(0, 1), (1, 1)]) & (xsi < 1)
        f_w[m] = f_w[m] * (1 - b * xsi[m]) / (1 - xsi[m])
        w = w * f_w
    else:
        w = np.zeros_like(u)
    return u, v, w


def xnearest(data, ti, tau, zi, zeta, yi, eta, xi, xsi):
    """_xinterpolators.py:515-560 (``XNearest.interp``): nearest node in space, linear in time."""
    T, Z, Y, X = data.shape
    two_t = bool(np.any(tau > 0))
    zf = np.where(zeta <= 0.5, zi, np.clip(zi + 1, 0, Z - 1))
    yf = np.where(eta <= 0.5, yi, np.clip(yi + 1, 0, Y - 1))
    xf = np.where(xsi <= 0.5, xi, np.clip(xi + 1, 0, X - 1))
    c0 = _take(data, ti, zf, yf, xf)
    if two_t:
        return c0 * (1 - tau) + _take(data, np.clip(ti + 1, 0, T - 1), zf, yf, xf) * tau
    return c0


def xnearest_velocity(fs: OFieldSet, pos, gp):
    """``XNearest_Velocity`` of the reference's regression test (tests/test_interpolation.py:279-294): no unit conversion."""
    (ti, tau), (zi, zeta), (yi, eta), (xi, xsi) = gp
    return tuple(xnearest(f, ti, tau, zi, zeta, yi, eta, xi, xsi) for f in (fs.U, fs.V, fs.W))


# ----------------------------------------------------------------------------------------------
# VectorField.eval
# ----------------------------------------------------------------------------------------------
def _flag_positions(view: View | None, zi, yi, xi):
    """_core/field.py:327-356 (``_update_particle_states_position``).  NB: X/Y index -2 (left
    out of bounds) is NOT flagged by the reference; only -1 and -3 are."""
    if view is None or view.n() == 0:  # `if particles:` is False for an empty view
        return
    for idx in (xi, yi):
        view.state = np.maximum(np.where(idx == -1, ERROR_OUT_OF_BOUNDS, view.state), view.state)
        view.state = np.maximum(np.where(idx == GRID_SEARCH_ERROR, ERROR_GRID_SEARCHING, view.state), view.state)
    view.state = np.maximum(np.where(zi == RIGHT_OUT_OF_BOUNDS, ERROR_OUT_OF_BOUNDS, view.state), view.state)
    view.state = np.maximum(np.where(zi == LEFT_OUT_OF_BOUNDS, ERROR_THROUGH_SURFACE, view.state), view.state)


def eval_uvw(fs: OFieldSet, t, z, y, x, view: View | None, want3d: bool):
    """_core/field.py:250-304 (``VectorField.eval`` + ``__getitem__`` error mapping :31-44)."""
    try:
        ei = None if view is None else view.ei[:, -1]
        z, y, x = np.atleast_1d(z), np.atleast_1d(y), np.atleast_1d(x)
        if np.any(np.isnan(t)):
            raise ValueError("Time values cannot be NaN")
        ti, tau = search_time(fs.time, t)
        (zi, zeta), (yi, eta), (xi, xsi) = grid_search(fs.grid, z, y, x, ei)
        if view is not None:
            e = view.ei
            e[:, -1] = ravel_index(fs.grid, zi, yi, xi)  # field.py:307-317 (int64 -> int32 store)
            view.ei = e
        _flag_positions(view, zi, yi, xi)
        pos = {"t": t, "z": z, "y": y, "x": x}
        gp = ((ti, tau), (zi, zeta), (yi, eta), (xi, xsi))
        if fs.interp == "linear":
            u, v, w = xlinear_velocity(fs, pos, gp)
        elif fs.interp == "freeslip":
            u, v, w = spatialslip_velocity(fs, pos, gp, 1.0, 0.0)
        elif fs.interp == "partialslip":
            u, v, w = spatialslip_velocity(fs, pos, gp, 0.5, 0.5)
        elif fs.interp == "nearest":
            u, v, w = xnearest_velocity(fs, pos, gp)
        else:
            from . import curvilinear_oracle as co

            u, v, w = co.cgrid_velocity(fs, pos, gp)
        oob = (xi < 0) | (yi < 0) | (zi < 0)
        for vel in (u, v, w):
            if view is not None and view.n() > 0:
                view.state = np.maximum(np.where(np.isnan(vel), ERROR_INTERPOLATION, view.state), view.state)
            if np.any(oob):
                vel[oob] = 0.0
        return (u, v, w) if want3d else (u, v)
    except OutsideTimeInterval:
        view.state = ERROR_OUTSIDE_TIME_INTERVAL  # plain assignment to the whole view (field.py:31-36)
        return (0, 0, 0) if want3d else (0, 0)


def xlinear_invdist_land(data, ti, tau, zi, zeta, yi, eta, xi, xsi):
    """_xinterpolators.py:556-613 (``XLinearInvdistLandTracer``): XLinear, except where some of the gathered corners are
    land (value ~ 0): all land -> 0; otherwise the inverse-squared-distance mean of the ocean corners, the distance
    measured in (eta, xsi) only and summed over EVERY gathered time / depth level alike; a sample exactly on an ocean
    corner takes the sum of that corner over the gathered levels (:603-610, as written in the reference)."""
    values = xlinear(data, ti, tau, zi, zeta, yi, eta, xi, xsi)
    corner, _ = _corner_block(data, ti, tau, zi, zeta, yi, xi)
    land = np.isclose(corner, 0.0)
    n_land = land.sum(axis=(0, 1, 2, 3))
    n_all = corner.shape[0] * corner.shape[1] * 4
    if np.any(n_land):
        values[n_land == n_all] = 0.0
        some = (n_land > 0) & (n_land < n_all)
        if np.any(some):
            jj = np.arange(2)[None, None, :, None, None]
            ii = np.arange(2)[None, None, None, :, None]
            d2 = (eta[None, None, None, None, :] - jj) ** 2 + (xsi[None, None, None, None, :] - ii) ** 2
            ocean = ~land
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / d2
                num = np.where(ocean, corner * inv, 0.0).sum(axis=(0, 1, 2, 3))
                den = np.where(ocean, inv, 0.0).sum(axis=(0, 1, 2, 3))
                values[some] = num[some] / den[some]
            on_node = (d2 == 0) & ocean
            node_val = np.where(on_node, corner, 0.0).sum(axis=(0, 1, 2, 3))
            pick = some & on_node.any(axis=(0, 1, 2, 3))
            values[pick] = node_val[pick]
    return values


def cgrid_tracer(fs: OFieldSet, data, ti, tau, zi, yi, xi):
    """_xinterpolators.py:335-383 (``CGrid_Tracer``): constant over the cell (the tracer point), linear in time."""
    T, Z, Y, X = data.shape
    off = fs.grid.offsets
    zi = np.clip(zi + off["Z"], 0, Z - 1)
    yi = np.clip(yi + off["Y"], 0, Y - 1)
    xi = np.clip(xi + off["X"], 0, X - 1)
    c0 = _take(data, ti, zi, yi, xi)
    if bool(np.any(tau > 0)):
        return c0 * (1 - tau) + _take(data, np.clip(ti + 1, 0, T - 1), zi, yi, xi) * tau
    return c0


def eval_scalar(fs: OFieldSet, data, method, t, z, y, x, view: View | None):
    """_core/field.py:144-202 (``Field.eval`` + the error mapping of ``__getitem__``) for a scalar field ``data``
    (T, Z, Y, X) on the fieldset's grid; ``method``: "linear" (XLinear), "nearest" (XNearest), "cgrid_tracer".
    A field with one time level has no time dimension (field.py:112-117)."""
    try:
        ei = None if view is None else view.ei[:, -1]
        z, y, x = np.atleast_1d(z), np.atleast_1d(y), np.atleast_1d(x)
        if np.any(np.isnan(t)):
            raise ValueError("Time values cannot be NaN")
        ti, tau = search_time(fs.time if data.shape[0] > 1 else None, t)
        (zi, zeta), (yi, eta), (xi, xsi) = grid_search(fs.grid, z, y, x, ei)
        if view is not None:
            e = view.ei
            e[:, -1] = ravel_index(fs.grid, zi, yi, xi)
            view.ei = e
        _flag_positions(view, zi, yi, xi)
        if method == "linear":
            value = xlinear(data, ti, tau, zi, zeta, yi, eta, xi, xsi)
        elif method == "nearest":
            value = xnearest(data, ti, tau, zi, zeta, yi, eta, xi, xsi)
        elif method == "linear_invdist_land":
            value = xlinear_invdist_land(data, ti, tau, zi, zeta, yi, eta, xi, xsi)
        else:
            value = cgrid_tracer(fs, data, ti, tau, zi, yi, xi)
        if view is not None and view.n() > 0:
            view.state = np.maximum(np.where(np.isnan(value), ERROR_INTERPOLATION, view.state), view.state)
        oob = (xi < 0) | (yi < 0) | (zi < 0)
        if np.any(oob):
            value[oob] = 0.0
        return value
    except OutsideTimeInterval:
        view.state = ERROR_OUTSIDE_TIME_INTERVAL
        return 0


def eval_constant(fs: OFieldSet, name, view: View):
    """``fieldset.Kh_zonal[particles]`` on the constant-field grid (lon=[0], lat=[0], no depth;
    _core/model.py:292-318): the grid search returns index 0 everywhere (index_search.py:45-46),
    ``ei[:, -1]`` is overwritten with 0 (cell counts are 0) and XConstantField returns
    ``data[0,0,0,0] * ones_like(x)`` (_xinterpolators.py:156-166)."""
    e = view.ei
    e[:, -1] = 0
    view.ei = e
    val = np.asarray(fs.constants[name]) * np.ones_like(view.x)
    if view.n() > 0:
        view.state = np.maximum(np.where(np.isnan(val), ERROR_INTERPOLATION, view.state), view.state)
    return val


# ----------------------------------------------------------------------------------------------
# Kernels
# ----------------------------------------------------------------------------------------------
def AdvectionRK4(p: View, fs: OFieldSet):
    """kernels/_advection.py:42-55."""
    (u1, v1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
    x1 = p.x + u1 * 0.5 * p.dt
    y1 = p.y + v1 * 0.5 * p.dt
    (u2, v2) = eval_uvw(fs, p.t + 0.5 * p.dt, p.z, y1, x1, p, False)
    x2 = p.x + u2 * 0.5 * p.dt
    y2 = p.y + v2 * 0.5 * p.dt
    (u3, v3) = eval_uvw(fs, p.t + 0.5 * p.dt, p.z, y2, x2, p, False)
    x3 = p.x + u3 * p.dt
    y3 = p.y + v3 * p.dt
    (u4, v4) = eval_uvw(fs, p.t + p.dt, p.z, y3, x3, p, False)
    p.dx = p.dx + (u1 + 2 * u2 + 2 * u3 + u4) / 6.0 * p.dt
    p.dy = p.dy + (v1 + 2 * v2 + 2 * v3 + v4) / 6.0 * p.dt


def AdvectionRK45(p: View, fs: OFieldSet):
    """kernels/_advection.py:85-155.  ``fs.context``: RK45_tol (already in mesh units: the reference divides it by deg2m
    on spherical meshes when the Kernel is built, kernel.py:144-145), RK45_min_dt, RK45_max_dt."""
    tol, min_dt, max_dt = fs.context["RK45_tol"], fs.context["RK45_min_dt"], fs.context["RK45_max_dt"]
    sign_dt = np.sign(p.dt)
    c = [1.0 / 4.0, 3.0 / 8.0, 12.0 / 13.0, 1.0, 1.0 / 2.0]
    A = [
        [1.0 / 4.0, 0.0, 0.0, 0.0, 0.0],
        [3.0 / 32.0, 9.0 / 32.0, 0.0, 0.0, 0.0],
        [1932.0 / 2197.0, -7200.0 / 2197.0, 7296.0 / 2197.0, 0.0, 0.0],
        [439.0 / 216.0, -8.0, 3680.0 / 513.0, -845.0 / 4104.0, 0.0],
        [-8.0 / 27.0, 2.0, -3544.0 / 2565.0, 1859.0 / 4104.0, -11.0 / 40.0],
    ]
    b4 = [25.0 / 216.0, 0.0, 1408.0 / 2565.0, 2197.0 / 4104.0, -1.0 / 5.0]
    b5 = [16.0 / 135.0, 0.0, 6656.0 / 12825.0, 28561.0 / 56430.0, -9.0 / 50.0, 2.0 / 55.0]
    (u1, v1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
    x1 = p.x + u1 * A[0][0] * p.dt
    y1 = p.y + v1 * A[0][0] * p.dt
    (u2, v2) = eval_uvw(fs, p.t + c[0] * p.dt, p.z, y1, x1, p, False)
    x2 = p.x + (u1 * A[1][0] + u2 * A[1][1]) * p.dt
    y2 = p.y + (v1 * A[1][0] + v2 * A[1][1]) * p.dt
    (u3, v3) = eval_uvw(fs, p.t + c[1] * p.dt, p.z, y2, x2, p, False)
    x3 = p.x + (u1 * A[2][0] + u2 * A[2][1] + u3 * A[2][2]) * p.dt
    y3 = p.y + (v1 * A[2][0] + v2 * A[2][1] + v3 * A[2][2]) * p.dt
    (u4, v4) = eval_uvw(fs, p.t + c[2] * p.dt, p.z, y3, x3, p, False)
    x4 = p.x + (u1 * A[3][0] + u2 * A[3][1] + u3 * A[3][2] + u4 * A[3][3]) * p.dt
    y4 = p.y + (v1 * A[3][0] + v2 * A[3][1] + v3 * A[3][2] + v4 * A[3][3]) * p.dt
    (u5, v5) = eval_uvw(fs, p.t + c[3] * p.dt, p.z, y4, x4, p, False)
    x5 = p.x + (u1 * A[4][0] + u2 * A[4][1] + u3 * A[4][2] + u4 * A[4][3] + u5 * A[4][4]) * p.dt
    y5 = p.y + (v1 * A[4][0] + v2 * A[4][1] + v3 * A[4][2] + v4 * A[4][3] + v5 * A[4][4]) * p.dt
    (u6, v6) = eval_uvw(fs, p.t + c[4] * p.dt, p.z, y5, x5, p, False)
    x_4th = (u1 * b4[0] + u2 * b4[1] + u3 * b4[2] + u4 * b4[3] + u5 * b4[4]) * p.dt
    y_4th = (v1 * b4[0] + v2 * b4[1] + v3 * b4[2] + v4 * b4[3] + v5 * b4[4]) * p.dt
    x_5th = (u1 * b5[0] + u2 * b5[1] + u3 * b5[2] + u4 * b5[3] + u5 * b5[4] + u6 * b5[5]) * p.dt
    y_5th = (v1 * b5[0] + v2 * b5[1] + v3 * b5[2] + v4 * b5[3] + v5 * b5[4] + v6 * b5[5]) * p.dt
    kappa = np.sqrt(np.pow(x_5th - x_4th, 2) + np.pow(y_5th - y_4th, 2))
    good = (kappa <= tol) | (np.fabs(p.dt) <= np.fabs(min_dt))
    p.dx = p.dx + np.where(good, x_5th, 0)
    p.dy = p.dy + np.where(good, y_5th, 0)
    inc = good & (kappa <= tol / 10) & (np.fabs(p.dt * 2) <= np.fabs(max_dt))
    p.next_dt = np.where(inc, p.dt * 2, p.dt)
    p.next_dt = np.where(np.abs(p.next_dt) > np.abs(max_dt), max_dt * sign_dt, p.next_dt)
    p.state = np.where(good, EVALUATE, p.state)
    rep = np.invert(good)
    p.dt = np.where(rep, p.dt / 2, p.dt)
    p.dt = np.where(np.abs(p.dt) < np.abs(min_dt), min_dt * sign_dt, p.dt)
    p.state = np.where(rep, REPEAT, p.state)


def AdvectionRK4_3D(p: View, fs: OFieldSet):
    """kernels/_advection.py:58-75."""
    (u1, v1, w1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, True)
    x1 = p.x + u1 * 0.5 * p.dt
    y1 = p.y + v1 * 0.5 * p.dt
    z1 = p.z + w1 * 0.5 * p.dt
    (u2, v2, w2) = eval_uvw(fs, p.t + 0.5 * p.dt, z1, y1, x1, p, True)
    x2 = p.x + u2 * 0.5 * p.dt
    y2 = p.y + v2 * 0.5 * p.dt
    z2 = p.z + w2 * 0.5 * p.dt
    (u3, v3, w3) = eval_uvw(fs, p.t + 0.5 * p.dt, z2, y2, x2, p, True)
    x3 = p.x + u3 * p.dt
    y3 = p.y + v3 * p.dt
    z3 = p.z + w3 * p.dt
    (u4, v4, w4) = eval_uvw(fs, p.t + p.dt, z3, y3, x3, p, True)
    p.dx = p.dx + (u1 + 2 * u2 + 2 * u3 + u4) / 6 * p.dt
    p.dy = p.dy + (v1 + 2 * v2 + 2 * v3 + v4) / 6 * p.dt
    p.dz = p.dz + (w1 + 2 * w2 + 2 * w3 + w4) / 6 * p.dt


def AdvectionEE(p: View, fs: OFieldSet):
    """kernels/_advection.py:78-82."""
    (u1, v1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
    p.dx = p.dx + u1 * p.dt
    p.dy = p.dy + v1 * p.dt


def AdvectionRK2(p: View, fs: OFieldSet):
    """kernels/_advection.py:20-27."""
    (u1, v1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
    x1 = p.x + u1 * 0.5 * p.dt
    y1 = p.y + v1 * 0.5 * p.dt
    (u2, v2) = eval_uvw(fs, p.t + 0.5 * p.dt, p.z, y1, x1, p, False)
    p.dx = p.dx + u2 * p.dt
    p.dy = p.dy + v2 * p.dt


def AdvectionRK2_3D(p: View, fs: OFieldSet):
    """kernels/_advection.py:30-39."""
    (u1, v1, w1) = eval_uvw(fs, p.t, p.z, p.y, p.x, p, True)
    x1 = p.x + u1 * 0.5 * p.dt
    y1 = p.y + v1 * 0.5 * p.dt
    z1 = p.z + w1 * 0.5 * p.dt
    (u2, v2, w2) = eval_uvw(fs, p.t + 0.5 * p.dt, z1, y1, x1, p, True)
    p.dx = p.dx + u2 * p.dt
    p.dy = p.dy + v2 * p.dt
    p.dz = p.dz + w2 * p.dt


class DiffusionUniformKh:
    """kernels/_advectiondiffusion.py:11-18,120-153.  ``normal(view)`` supplies the two N(0,1)
    draws per particle; the default mirrors the reference's legacy global RandomState
    (``np.random.normal``).  Tests inject the engine's Philox stream to compare the
    deterministic part bit-for-bit."""

    __name__ = "DiffusionUniformKh"

    def __init__(self, normal=None):
        self.normal = normal

    def __call__(self, p: View, fs: OFieldSet):
        if self.normal is None:
            dWx = np.random.normal(0, np.sqrt(np.fabs(p.dt)))
            dWy = np.random.normal(0, np.sqrt(np.fabs(p.dt)))
        else:
            zx, zy = self.normal(p)
            dWx = zx * np.sqrt(np.fabs(p.dt))
            dWy = zy * np.sqrt(np.fabs(p.dt))
        kh_zonal = eval_constant(fs, "Kh_zonal", p)
        kh_meridional = eval_constant(fs, "Kh_meridional", p)
        if fs.const_spherical:
            kh_zonal = kh_zonal / pow(fs.const_deg2m * trig.current().kh_metric(p.y * np.pi / 180), 2)
            kh_meridional = kh_meridional / pow(fs.const_deg2m, 2)
        bx = np.sqrt(2 * kh_zonal)
        by = np.sqrt(2 * kh_meridional)
        p.dx = p.dx + bx * dWx
        p.dy = p.dy + by * dWy


class _AdvectionDiffusion:
    """kernels/_advectiondiffusion.py:11-18,21-117 (``AdvectionDiffusionM1`` / ``AdvectionDiffusionEM``): 2-D
    advection-diffusion with spatially varying diffusivity fields ``Kh_zonal`` / ``Kh_meridional`` (scalar fields on the
    fieldset's grid, ``fs.scalars``) and the finite-difference step ``fs.context["dres"]``.  ``normal(view)`` supplies
    the two N(0,1) draws per particle (default: the reference's legacy global RandomState, so that ``np.random.seed``
    reproduces the reference bit for bit); tests inject the engine's Philox stream."""

    scheme = "M1"

    def __init__(self, normal=None):
        self.normal = normal

    def __call__(self, p: View, fs: OFieldSet):
        if self.normal is None:
            dWx = np.random.normal(0, np.sqrt(np.fabs(p.dt)))
            dWy = np.random.normal(0, np.sqrt(np.fabs(p.dt)))
        else:
            zx, zy = self.normal(p)
            dWx = zx * np.sqrt(np.fabs(p.dt))
            dWy = zy * np.sqrt(np.fabs(p.dt))
        dres = fs.context["dres"]
        khz, mz = fs.scalars["Kh_zonal"]
        khm, mm = fs.scalars["Kh_meridional"]
        sph, deg2m = fs.grid.spherical, fs.grid.deg2m

        def zonal(v, lat):  # meters_to_degrees_zonal (:11-13)
            return v / pow(deg2m * trig.current().m1em_metric(lat * np.pi / 180), 2)

        def merid(v):  # meters_to_degrees_meridional (:16-18)
            return v / pow(deg2m, 2)

        if self.scheme == "EM":
            u, v = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
        Kxp1 = eval_scalar(fs, khz, mz, p.t, p.z, p.y, p.x + dres, p)
        Kxm1 = eval_scalar(fs, khz, mz, p.t, p.z, p.y, p.x - dres, p)
        if sph:
            Kxp1 = zonal(Kxp1, p.y)
            Kxm1 = zonal(Kxm1, p.y)
        dKdx = (Kxp1 - Kxm1) / (2 * dres)
        if self.scheme == "M1":
            u, v = eval_uvw(fs, p.t, p.z, p.y, p.x, p, False)
        kh_zonal = eval_scalar(fs, khz, mz, p.t, p.z, p.y, p.x, p)
        if sph:
            kh_zonal = zonal(kh_zonal, p.y)
        bx = np.sqrt(2 * kh_zonal)
        Kyp1 = eval_scalar(fs, khm, mm, p.t, p.z, p.y + dres, p.x, p)
        Kym1 = eval_scalar(fs, khm, mm, p.t, p.z, p.y - dres, p.x, p)
        if sph:
            Kyp1 = merid(Kyp1)
            Kym1 = merid(Kym1)
        dKdy = (Kyp1 - Kym1) / (2 * dres)
        kh_meridional = eval_scalar(fs, khm, mm, p.t, p.z, p.y, p.x, p)
        if sph:
            kh_meridional = merid(kh_meridional)
        by = np.sqrt(2 * kh_meridional)
        if self.scheme == "M1":  # :64-66
            p.dx = p.dx + (u * p.dt + 0.5 * dKdx * (dWx**2 + p.dt) + bx * dWx)
            p.dy = p.dy + (v * p.dt + 0.5 * dKdy * (dWy**2 + p.dt) + by * dWy)
        else:  # :85,101,115-117
            ax = u + dKdx
            ay = v + dKdy
            p.dx = p.dx + (ax * p.dt + bx * dWx)
            p.dy = p.dy + (ay * p.dt + by * dWy)


class AdvectionDiffusionM1(_AdvectionDiffusion):
    __name__ = "AdvectionDiffusionM1"
    scheme = "M1"


class AdvectionDiffusionEM(_AdvectionDiffusion):
    __name__ = "AdvectionDiffusionEM"
    scheme = "EM"


def DeleteOnError(p: View, fs: OFieldSet):
    """The idiom of the reference's tests (tests/common_kernels.py:12-13,
    tests/test_interpolation.py:357-359): every error state becomes Delete."""
    s = p.state
    p.state = np.where(s >= 50, DELETE, s)


# ----------------------------------------------------------------------------------------------
# Kernel.execute / ParticleSet.execute
# ----------------------------------------------------------------------------------------------
_ERRORS_TO_THROW = (  # order of _core/kernel.py:31-38
    ERROR_OUTSIDE_TIME_INTERVAL,
    ERROR_OUT_OF_BOUNDS,
    ERROR_THROUGH_SURFACE,
    ERROR_INTERPOLATION,
    ERROR_GRID_SEARCHING,
    ERROR,
)


def _remove(pdata, idx):
    """_core/particleset.py:247-250 (np.delete on every array)."""
    for k in pdata:
        pdata[k] = np.delete(pdata[k], idx, axis=0)


def kernel_execute(pdata, fs: OFieldSet, kernels, endtime, dt, max_iters=None):
    """_core/kernel.py:174-247 (``Kernel.execute``) + ``_position_update`` (:108-120).

    ``max_iters`` (testing aid, not in the reference) stops after that many loop iterations.
    Returns the number of particle-steps evaluated.
    """
    sign = 1 if dt > 0 else -1
    pdata["state"][:] = EVALUATE
    nsteps = 0
    it = 0
    rk45_mode = "RK45_tol" in getattr(fs, "context", {})
    max_repeats = 10000
    while len(pdata["state"]) > 0 and np.any(np.isin(pdata["state"], [EVALUATE, REPEAT])):
        if max_iters is not None and it >= max_iters:
            break
        it += 1
        tte = sign * (endtime - pdata["t"])
        ev = np.isin(pdata["state"], [SUCCESS, EVALUATE]) & (tte >= 0)
        if not np.any(ev):
            return nsteps
        if sign == 1:
            pdata["dt"][:] = np.maximum(np.minimum(pdata["dt"], tte), 0)
        else:
            pdata["dt"][:] = np.minimum(np.maximum(pdata["dt"], -tte), 0)
        nsteps += int(np.count_nonzero(ev))
        for f in kernels:
            f(View(pdata, ev), fs)
            rep = pdata["state"] == REPEAT  # kernel.py:212-216
            while np.any(rep):
                if max_repeats is not None:  # testing aid: the reference has no bound
                    max_repeats -= 1
                    if max_repeats < 0:
                        raise RuntimeError("Repeat loop does not terminate")
                f(View(pdata, rep), fs)
                rep = pdata["state"] == REPEAT
        upd = ev & np.isin(pdata["state"], [EVALUATE, SUCCESS])
        if np.any(upd):
            p = View(pdata, upd)
            p.x = p.x + p.dx
            p.y = p.y + p.dy
            p.z = p.z + p.dz
            p.t = p.t + p.dt
            p.dx = 0
            p.dy = 0
            p.dz = 0
            if rk45_mode:  # kernel.py:118-120: `if hasattr(self.fieldset, "RK45_tol")`
                p.dt = p.next_dt
        if not rk45_mode:  # kernel.py:224-226
            pdata["dt"][:] = dt
        eol = (pdata["state"] == EVALUATE) & (pdata["t"] == endtime)
        pdata["state"][eol] = END_OF_LOOP
        dele = np.where(pdata["state"] == DELETE)[0]
        if len(dele) > 0:
            _remove(pdata, dele)
        if np.any(pdata["state"] == STOP_ALL_EXECUTION):
            return nsteps
        for code in _ERRORS_TO_THROW:
            if np.any(pdata["state"] == code):
                raise OracleParticleError(code)
    return nsteps


def to_write_particles(pdata, t):
    """_core/particlefile.py:198-221 (``_to_write_particles``): rows written at output time ``t``."""
    fin = np.isfinite(pdata["t"])
    return np.where(
        (
            np.less_equal(t - np.abs(pdata["dt"] / 2), pdata["t"], where=fin, out=None)
            & np.greater_equal(t + np.abs(pdata["dt"] / 2), pdata["t"], where=fin, out=None)
            | (np.isnan(pdata["dt"]) & np.equal(t, pdata["t"], where=fin, out=None))
        )
        & np.isfinite(pdata["particle_id"])
        & fin
    )[0]


def pset_execute(pdata, fs: OFieldSet, kernels, dt, runtime=None, endtime=None, outputdt=None, on_output=None):
    """_core/particleset.py:355-470 (outer loop) with float-second arguments
    (:497-585: start = first release time, or 0 / interval end when t is NaN)."""
    if len(pdata["state"]) == 0:
        return 0
    if not isinstance(kernels, (list, tuple)):
        kernels = [kernels]
    dt = float(dt)
    sign = 1 if dt > 0 else -1
    pdata["dt"][:] = dt
    first = np.nanmin(pdata["t"]) if sign == 1 else np.nanmax(pdata["t"])
    if np.all(np.isnan(pdata["t"])):
        first = np.nan
    if np.isnan(first):
        start = 0.0 if sign == 1 else float(fs.time[-1] - fs.time[0])
    else:
        start = float(first)
    end = float(endtime) if endtime is not None else start + sign * float(runtime)
    if np.isnan(pdata["t"]).any():
        pdata["t"][:] = start
    next_output = None
    if outputdt is not None:
        if on_output is not None:
            on_output(pdata, start)
        next_output = start + outputdt * sign
    time = start
    total = 0
    while sign * (time - end) < 0:
        if next_output is not None:
            next_time = min(next_output, end) if sign > 0 else max(next_output, end)
        else:
            next_time = end
        total += kernel_execute(pdata, fs, kernels, next_time, dt)
        if next_output is not None and abs(next_time - next_output) < 0.001:
            if on_output is not None:
                on_output(pdata, next_output)
            next_output += outputdt * sign
        time = next_time
    return total
