"""Seeded synthetic inputs shared by the tests and ``oracle/make_golden.py``.

Every case is regenerated from its spec (seed + shape parameters), so only the *reference's
outputs* need to be stored under ``tests/golden/ref_cases.npz``.
"""

from __future__ import annotations

import numpy as np


def peninsula(xdim=100, ydim=50, mesh="flat"):
    """Config 1 field: flow around an idealised peninsula on an A-grid, restated from the
    formulas of the reference dataset (_datasets/structured/generated.py:206-298):
    stream function P = u0 R^2 y / ((x-x0)^2 + y^2) - u0 y, land where P >= 0, f32 arrays."""
    Lx, Ly = 1.0e5, 5.0e4
    xs = np.linspace(0, Lx, xdim, dtype=np.float32)
    ys = np.linspace(0, Ly, ydim, dtype=np.float32)
    u0, x0, R = 1, Lx / 2, 0.32 * Lx / 2
    x, y = np.meshgrid(xs, ys, sparse=True, indexing="xy")
    P = np.zeros((ydim, xdim), dtype=np.float32)
    U = np.zeros_like(P)
    V = np.zeros_like(P)
    r2 = (x - x0) ** 2 + y**2
    P[:, :] = u0 * R**2 * y / r2 - u0 * y
    land = P >= 0.0
    P[land] = 0.0
    U[:, :] = u0 - u0 * R**2 * ((x - x0) ** 2 - y**2) / (r2**2)
    V[:, :] = -2 * u0 * R**2 * ((x - x0) * y) / (r2**2)
    U[land] = 0.0
    V[land] = 0.0
    lon = xs / 1852.0 / 60.0 if mesh == "spherical" else xs
    lat = ys / 1852.0 / 60.0 if mesh == "spherical" else ys
    return lon, lat, U, V, P


def smooth_uvw(rng, lon, lat, depth, nt, ddtype, umax=1.0, wmax=1e-3, noise=0.05):
    """Config-2 style field: a few Fourier modes + seeded noise, (T, Z, Y, X)."""
    nz = 1 if depth is None else len(depth)
    X = (lon - lon[0]) / (lon[-1] - lon[0])
    Y = (lat - lat[0]) / (lat[-1] - lat[0])
    Z = np.zeros(1) if depth is None or len(depth) < 2 else (depth - depth[0]) / (depth[-1] - depth[0])
    tt = np.arange(nt, dtype=np.float64)
    T4, Z4, Y4, X4 = np.meshgrid(tt, Z, Y, X, indexing="ij", sparse=True)
    two_pi = 2 * np.pi
    U = np.sin(two_pi * (2 * X4 + 0.3 * T4)) * np.cos(two_pi * Y4) * (1 - 0.5 * Z4) + 0.3 * np.cos(two_pi * 3 * Y4 + T4)
    V = np.cos(two_pi * (X4 + 0.1 * T4)) * np.sin(two_pi * 2 * Y4) * (1 - 0.3 * Z4) + 0.2 * np.sin(two_pi * 2 * X4)
    W = np.sin(two_pi * X4) * np.sin(two_pi * Y4) * np.sin(np.pi * Z4) * np.cos(0.5 * T4)
    shape = (nt, nz, len(lat), len(lon))
    U = np.broadcast_to(U, shape) / 1.3 + noise * rng.uniform(-1, 1, shape)
    V = np.broadcast_to(V, shape) / 1.2 + noise * rng.uniform(-1, 1, shape)
    W = np.broadcast_to(W, shape) + noise * rng.uniform(-1, 1, shape)
    return (umax * U).astype(ddtype), (umax * V).astype(ddtype), (wmax * W).astype(ddtype)


def curv_mesh(ny, nx, spherical, cdtype, sph_box=(-20.0, 30.0, 35.0, 25.0)):
    """Smooth curvilinear node mesh (rotated 25 deg, stretched, warped): 2-D lon/lat (ny, nx).  Spherical meshes span
    lon0 + dlon * X, lat0 + dlat * Y, sph_box = (lon0, dlon, lat0, dlat)."""
    I, J = np.meshgrid(np.linspace(0, 1, nx), np.linspace(0, 1, ny))
    th = np.deg2rad(25.0)
    a = I + 0.15 * I**2
    b = J + 0.1 * np.sin(np.pi * I) * J
    X = np.cos(th) * a - np.sin(th) * b
    Y = np.sin(th) * a + np.cos(th) * b
    if spherical:
        lon0, dlon, lat0, dlat = sph_box
        lon, lat = lon0 + dlon * X, lat0 + dlat * Y
    else:
        # Warp BOTH grid-line families.  With straight, parallel eta-lines the quadratic coefficient of the
        # reference's bilinear inverse (index_search.py:136) cancels analytically to ~1e-10 -- above its
        # 1e-12 "linear" threshold -- and the root then depends on the BLAS summation order of np.dot,
        # i.e. on the BATCH SIZE inside the reference itself (measured: 1.5 % in xsi).  Parity is only
        # defined on meshes where the reference is reproducible.
        X = X + 0.12 * J**2 * (1 + 0.5 * I)
        Y = Y + 0.10 * I**2 * (1 - 0.4 * J)
        lon, lat = 1e4 * X, 1e4 * Y
    return lon.astype(cdtype), lat.astype(cdtype)


def points_in_mesh(rng, lon, lat, n, margin=0.5):
    """Random points inside the mesh: bilinear blend inside random cells (kept `margin` cells off the rim)."""
    ny, nx = lon.shape
    jj = rng.uniform(margin, ny - 1 - margin, n)
    ii = rng.uniform(margin, nx - 1 - margin, n)
    j0, i0 = jj.astype(int), ii.astype(int)
    fj, fi = jj - j0, ii - i0

    def bl(a):
        a = a.astype(np.float64)
        return ((1 - fj) * (1 - fi) * a[j0, i0] + (1 - fj) * fi * a[j0, i0 + 1] + fj * fi * a[j0 + 1, i0 + 1]
                + fj * (1 - fi) * a[j0 + 1, i0])  # fmt: skip

    return bl(lon), bl(lat)


def _default(spec, k, v):
    return spec[k] if k in spec else v


# name -> spec.  `segments` are successive execute() calls (kwargs runtime=/endtime= in seconds).
CASES = {
    # C2-shaped (coords f64, data f32, spherical, time-varying, 3-D); errors deleted
    "c2_small": dict(seed=1, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=41, ny=33, nz=12, nt=3,
                     tstep=3600.0, n=500, kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=7200.0)],
                     delete=True, margin=-0.02, umax=10.0),
    # same but flat mesh, f32 coords, f64 data (the v3-golden dtype combination)
    "flat_f32c_f64d": dict(seed=2, kind="smooth", cdtype="f4", ddtype="f8", mesh="flat", nx=20, ny=17, nz=6, nt=4,
                           tstep=50.0, n=400, kernels=["AdvectionRK4_3D"], dt=10.0, segments=[dict(runtime=150.0)],
                           delete=True, margin=-0.03),
    # everything f32 (f32 arithmetic at stage 1), time-varying
    "all_f32": dict(seed=3, kind="smooth", cdtype="f4", ddtype="f4", mesh="spherical", nx=30, ny=25, nz=8, nt=3,
                    tstep=1800.0, n=400, kernels=["AdvectionRK4_3D"], dt=300.0, segments=[dict(runtime=3600.0)],
                    delete=True, margin=-0.02),
    # C1: Peninsula, 2-D static field, AdvectionRK4
    "c1_peninsula": dict(seed=4, kind="peninsula", mesh="flat", n=200, kernels=["AdvectionRK4"], dt=1800.0,
                         segments=[dict(runtime=23 * 3600.0)], delete=False),
    "c1_peninsula_sph": dict(seed=5, kind="peninsula", mesh="spherical", n=100, kernels=["AdvectionRK4"], dt=1800.0,
                             segments=[dict(runtime=12 * 3600.0)], delete=False),
    # 2-D advection in a 3-D time-varying field (z stays f32 at every stage)
    "rk4_2d_in_3d": dict(seed=6, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=31, ny=29, nz=7, nt=3,
                         tstep=3600.0, n=300, kernels=["AdvectionRK4"], dt=900.0, segments=[dict(runtime=7200.0)],
                         delete=True, margin=-0.02),
    # delayed release + partial last step + two execute() segments
    "delayed_partial": dict(seed=7, kind="smooth", cdtype="f8", ddtype="f4", mesh="flat", nx=25, ny=21, nz=6, nt=3,
                            tstep=2000.0, n=300, kernels=["AdvectionRK4_3D"], dt=300.0,
                            segments=[dict(runtime=1000.0), dict(runtime=1450.0)], delete=True, margin=0.05,
                            release=("uniform", 0.0, 1700.0)),
    # backward in time
    "backward": dict(seed=8, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=25, ny=21, nz=6, nt=3,
                     tstep=3600.0, n=300, kernels=["AdvectionRK4_3D"], dt=-600.0, segments=[dict(runtime=5400.0)],
                     delete=True, margin=0.05, release=("const", 7200.0)),
    # no error handler: the reference raises FieldOutOfBoundError after the first offending step
    "raise_oob": dict(seed=9, kind="smooth", cdtype="f8", ddtype="f4", mesh="flat", nx=15, ny=13, nz=5, nt=3,
                      tstep=1000.0, n=200, kernels=["AdvectionRK4_3D"], dt=100.0, segments=[dict(runtime=1500.0)],
                      delete=False, margin=0.02, umax=3.0),
    # integrating beyond the field's time axis: OutsideTimeInterval flags the whole view
    "raise_time": dict(seed=10, kind="smooth", cdtype="f8", ddtype="f4", mesh="flat", nx=15, ny=13, nz=5, nt=3,
                       tstep=500.0, n=100, kernels=["AdvectionRK4_3D"], dt=100.0, segments=[dict(runtime=1500.0)],
                       delete=False, margin=0.3),
    # Euler / RK2 on the same machinery
    "ee_2d": dict(seed=11, kind="smooth", cdtype="f4", ddtype="f4", mesh="spherical", nx=22, ny=19, nz=1, nt=3,
                  tstep=3600.0, n=200, kernels=["AdvectionEE"], dt=600.0, segments=[dict(runtime=7200.0)],
                  delete=True, margin=0.02, no_depth=True),
    "rk2_3d": dict(seed=12, kind="smooth", cdtype="f8", ddtype="f8", mesh="flat", nx=22, ny=19, nz=6, nt=3,
                   tstep=400.0, n=200, kernels=["AdvectionRK2_3D"], dt=50.0, segments=[dict(runtime=800.0)],
                   delete=True, margin=0.02),
    "rk2_2d": dict(seed=13, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=22, ny=19, nz=4, nt=1,
                   tstep=400.0, n=200, kernels=["AdvectionRK2"], dt=600.0, segments=[dict(runtime=6000.0)],
                   delete=True, margin=0.02),
    # fused advection + uniform diffusion (reference RNG: np.random.seed(rng_seed) before execute)
    "diffusion": dict(seed=14, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=31, ny=29, nz=7, nt=3,
                      tstep=3600.0, n=300, kernels=["AdvectionRK4_3D", "DiffusionUniformKh"], dt=600.0,
                      segments=[dict(runtime=3600.0)], delete=True, margin=0.1, kh=(100.0, 50.0), rng_seed=1234),
    # strong downward/upward w: through-surface (61) and bottom (60) exits, deleted
    "through_surface": dict(seed=15, kind="smooth", cdtype="f8", ddtype="f4", mesh="flat", nx=15, ny=13, nz=6, nt=2,
                            tstep=4000.0, n=300, kernels=["AdvectionRK4_3D"], dt=200.0, segments=[dict(runtime=4000.0)],
                            delete=True, margin=0.02, wmax=0.2),
    # ---- C-grid (CGrid_Velocity): curvilinear search with hint + spatial-hash fallback ----
    "curv_flat_2d": dict(seed=21, kind="curv", cdtype="f8", mesh="flat", nx=31, ny=23, nz=1, nt=3, tstep=600.0, n=400,
                         kernels=["AdvectionRK4"], dt=60.0, segments=[dict(runtime=600.0)], delete=True, umax=1.5),
    "curv_sph_2d": dict(seed=22, kind="curv", cdtype="f8", mesh="spherical", nx=41, ny=33, nz=1, nt=3, tstep=7200.0, n=500,
                        kernels=["AdvectionRK4"], dt=900.0, segments=[dict(runtime=14400.0)], delete=True, umax=20.0),
    "curv_sph_3d": dict(seed=23, kind="curv", cdtype="f8", mesh="spherical", nx=31, ny=23, nz=6, nt=3, tstep=3600.0, n=400,
                        kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=7200.0)], delete=True, umax=15.0),
    "curv_sph_f32": dict(seed=24, kind="curv", cdtype="f4", mesh="spherical", nx=31, ny=23, nz=1, nt=2, tstep=7200.0, n=300,
                         kernels=["AdvectionRK4"], dt=600.0, segments=[dict(runtime=7200.0)], delete=True, umax=15.0),
    # ---- A-grid interpolation (XLinear_Velocity) on curvilinear meshes: the same search, _xinterpolators.py:112-190 on its result ----
    "curv_lin_flat_2d": dict(seed=41, kind="curv", interp="linear", cdtype="f8", mesh="flat", nx=31, ny=23, nz=1, nt=3, tstep=600.0,
                             n=400, kernels=["AdvectionRK4"], dt=60.0, segments=[dict(runtime=600.0)], delete=True, umax=1.5),
    "curv_lin_sph_3d": dict(seed=42, kind="curv", interp="linear", cdtype="f8", mesh="spherical", nx=31, ny=23, nz=6, nt=3,
                            tstep=3600.0, n=400, kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=7200.0)],
                            delete=True, umax=15.0),
    "curv_lin_sph_f32": dict(seed=43, kind="curv", interp="linear", cdtype="f4", mesh="spherical", nx=31, ny=23, nz=5, nt=2,
                             tstep=7200.0, n=300, kernels=["AdvectionRK4"], dt=600.0, segments=[dict(runtime=7200.0)],
                             delete=True, umax=15.0),
    "cgrid_rect_3d": dict(seed=25, kind="smooth", interp="cgrid_velocity", cdtype="f4", ddtype="f8", mesh="flat", nx=16,
                          ny=13, nz=6, nt=4, tstep=200.0, n=400, kernels=["AdvectionRK4_3D"], dt=50.0,
                          segments=[dict(runtime=600.0)], delete=True, margin=-0.02, umax=4.0),
    "cgrid_rect_sph": dict(seed=26, kind="smooth", interp="cgrid_velocity", cdtype="f8", ddtype="f4", mesh="spherical",
                           nx=21, ny=17, nz=5, nt=3, tstep=3600.0, n=300, kernels=["AdvectionRK4"], dt=600.0,
                           segments=[dict(runtime=7200.0)], delete=True, margin=0.02, umax=10.0),
    # ---- other A-grid vector interpolators (reference _xinterpolators.py:385-560): land = nodes with U = V = 0 ----
    "freeslip_3d": dict(seed=31, kind="smooth", interp="freeslip", land=True, cdtype="f4", ddtype="f8", mesh="flat", nx=16, ny=13,
                        nz=6, nt=4, tstep=200.0, n=400, kernels=["AdvectionRK4_3D"], dt=50.0, segments=[dict(runtime=600.0)],
                        delete=True, margin=-0.02, umax=4.0),
    "partialslip_sph": dict(seed=32, kind="smooth", interp="partialslip", land=True, cdtype="f8", ddtype="f4", mesh="spherical",
                            nx=21, ny=17, nz=5, nt=3, tstep=3600.0, n=300, kernels=["AdvectionRK4"], dt=600.0,
                            segments=[dict(runtime=7200.0)], delete=True, margin=0.02, umax=10.0),
    # 2-D advection at the surface of a 3-D field whose land mask grows with depth: the whole batch has zeta == 0, so the
    # reference's land test looks at the first depth level only (lenZ == 1, _xinterpolators.py:400,426-434)
    "freeslip_surface": dict(seed=34, kind="smooth", interp="freeslip", land="depth", surface=True, cdtype="f8", ddtype="f4",
                             mesh="flat", nx=19, ny=16, nz=5, nt=3, tstep=400.0, n=300, kernels=["AdvectionRK4"], dt=60.0,
                             segments=[dict(runtime=720.0)], delete=True, margin=0.02, umax=4.0),
    # nearest node on float32 data without a time dimension: every RK stage value is float32, so the reference's
    # (u1 + 2*u2 + 2*u3 + u4) / 6 is float32 arithmetic (found by scripts/fuzz_hostsim.py)
    "nearest_f32_static": dict(seed=35, kind="smooth", interp="nearest", cdtype="f4", ddtype="f4", mesh="flat", nx=9, ny=14, nz=3,
                               nt=1, tstep=1000.0, n=120, kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=6000.0)],
                               delete=True, margin=0.1, umax=3.0),
    # ---- spherical edge cases: where the trigonometry of the unit conversion and of the curvilinear search is at its worst ----
    # within +-3 deg of the equator (nodes on it): cos_np's cancellation near 0 and its clamp to 1
    "sph_equator": dict(seed=51, kind="smooth", cdtype="f8", ddtype="f4", mesh="spherical", nx=23, ny=25, nz=5, nt=3,
                        tstep=3600.0, n=300, kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=7200.0)],
                        delete=True, margin=0.02, umax=2.0, lon_range=(-4.0, 4.0), lat_range=(-3.0, 3.0)),
    # 80 - 89.5 deg: a small cos(lat) amplifies every last-bit difference of the zonal conversion; float32 coordinates and data
    "sph_polar_f32": dict(seed=52, kind="smooth", cdtype="f4", ddtype="f4", mesh="spherical", nx=25, ny=20, nz=1, nt=3,
                          tstep=3600.0, n=300, kernels=["AdvectionRK4"], dt=600.0, segments=[dict(runtime=7200.0)],
                          delete=True, margin=0.02, umax=1.0, lon_range=(-30.0, 30.0), lat_range=(80.0, 89.5), no_depth=True),
    # spherical rectilinear C-grid on float32 coordinates: at RK stage 1 the barycentric coordinates, the mid-edge latitudes and
    # their cos are float32 (cgrid.cuh edge_length with L = float)
    "cgrid_rect_sph_f32": dict(seed=53, kind="smooth", interp="cgrid_velocity", cdtype="f4", ddtype="f4", mesh="spherical",
                               nx=21, ny=17, nz=5, nt=3, tstep=3600.0, n=300, kernels=["AdvectionRK4"], dt=600.0,
                               segments=[dict(runtime=7200.0)], delete=True, margin=0.02, umax=10.0),
    # curvilinear spherical C-grid across 90 deg, 135 deg and the antimeridian, longitudes wrapped to [-180, 180) like an ORCA
    # grid: sincos_lon's quadrant switches, cos_np of |lon| > 90 deg (the cold path) and CGrid_Velocity's longitude unwrap
    "curv_sph_dateline": dict(seed=54, kind="curv", cdtype="f8", mesh="spherical", nx=41, ny=25, nz=1, nt=3, tstep=7200.0,
                              n=400, kernels=["AdvectionRK4"], dt=900.0, segments=[dict(runtime=14400.0)], delete=True,
                              umax=20.0, sph_box=(95.0, 110.0, -10.0, 25.0), wrap_lon=True),
    "nearest_3d": dict(seed=33, kind="smooth", interp="nearest", cdtype="f8", ddtype="f4", mesh="spherical", nx=21, ny=17, nz=5,
                       nt=3, tstep=3600.0, n=300, kernels=["AdvectionRK4_3D"], dt=600.0, segments=[dict(runtime=7200.0)],
                       delete=True, margin=0.02, umax=10.0),
}


def build(spec):
    """Materialise a case: grid coords, fields, particles, run parameters."""
    rng = np.random.default_rng(spec["seed"])
    mesh = spec["mesh"]
    n = spec["n"]
    out = dict(mesh=mesh, dt=spec["dt"], segments=spec["segments"], kernels=spec["kernels"],
               delete_on_error=spec["delete"], constants=None, rng_seed=spec.get("rng_seed"))  # fmt: skip
    if spec["kind"] == "peninsula":
        lon, lat, U, V, P = peninsula(mesh=mesh)
        out.update(lon=lon, lat=lat, depth=None, times=None, U=U[None, None], V=V[None, None], W=None, P=P)
        scale = 1.0 if mesh == "flat" else 1 / 1852.0 / 60.0
        out["x"] = np.full(n, 3e3 * scale)
        out["y"] = np.linspace(3e3, 47e3, n) * scale
        out["z"] = np.zeros(n)
        out["t"] = np.zeros(n)
        return out
    if spec["kind"] == "curv":
        cd = np.dtype(spec["cdtype"])
        nx, ny, nz, nt = spec["nx"], spec["ny"], spec["nz"], spec["nt"]
        lon, lat = curv_mesh(ny, nx, mesh == "spherical", cd, **({"sph_box": spec["sph_box"]} if "sph_box" in spec else {}))
        three_d = spec["kernels"][0].endswith("_3D")
        depth = (np.linspace(0, 1, nz) ** 1.4 * 200.0).astype(cd) if nz > 1 else None
        shape = (nt, nz, ny, nx)
        umax = spec["umax"]
        dd = np.dtype(spec.get("ddtype", "f4"))  # float32 velocity data unless the spec asks for another dtype
        U = (umax * rng.uniform(-1, 1, shape)).astype(dd)
        V = (umax * rng.uniform(-1, 1, shape)).astype(dd)
        W = (1e-2 * rng.uniform(-1, 1, shape)).astype(dd) if three_d else None
        x, y = points_in_mesh(rng, lon, lat, n)
        if spec.get("wrap_lon"):  # nodes and releases wrapped to [-180, 180) after the releases were blended
            lon = (((lon.astype(np.float64) + 180.0) % 360.0) - 180.0).astype(cd)
            x = ((x + 180.0) % 360.0) - 180.0
        z = rng.uniform(2.0, 190.0, n) if nz > 1 else np.zeros(n)
        out.update(lon=lon, lat=lat, depth=depth, times=np.arange(nt) * spec["tstep"], U=U, V=V, W=W, x=x, y=y, z=z,
                   t=np.zeros(n), interp=spec.get("interp", "cgrid_velocity"), padding=("low", "low", "high"))  # fmt: skip
        return out
    cd = np.dtype(spec["cdtype"])
    dd = np.dtype(spec["ddtype"])
    nx, ny, nz, nt = spec["nx"], spec["ny"], spec["nz"], spec["nt"]
    if "interp" in spec:
        out["interp"] = spec["interp"]
    if mesh == "spherical":
        lon = np.linspace(*spec.get("lon_range", (-10.0, 10.0)), nx).astype(cd)
        lat = np.linspace(*spec.get("lat_range", (30.0, 50.0)), ny).astype(cd)
        umax = _default(spec, "umax", 1.0)
    else:
        lon = np.linspace(0.0, 2.0e4, nx).astype(cd)
        lat = np.linspace(0.0, 1.5e4, ny).astype(cd)
        umax = _default(spec, "umax", 1.0)
    no_depth = spec.get("no_depth", False)
    depth = None if no_depth else (np.linspace(0, 1, nz) ** 1.6 * 500.0).astype(cd)
    U, V, W = smooth_uvw(rng, lon.astype(np.float64), lat.astype(np.float64),
                         None if depth is None else depth.astype(np.float64), nt, dd,
                         umax=umax, wmax=_default(spec, "wmax", 1e-3))  # fmt: skip
    if spec.get("land"):  # blocks of land: U = V = W = 0 on about a quarter of the nodes, all levels and times
        r = rng.uniform(0, 1, (ny // 3 + 1, nx // 3 + 1))
        for k in range(U.shape[1]):  # land="depth": the land mask grows with depth (bathymetry)
            blk = r < (0.25 if spec["land"] is True else 0.1 + 0.08 * k)
            land = np.kron(blk, np.ones((3, 3), dtype=bool))[:ny, :nx]
            U[:, k][..., land] = 0
            V[:, k][..., land] = 0
            W[:, k][..., land] = 0
    times = np.arange(nt) * spec["tstep"] if nt > 1 else None
    m = spec["margin"]  # negative margin => some particles start outside the domain
    lx, ly = float(lon[-1] - lon[0]), float(lat[-1] - lat[0])
    x = rng.uniform(float(lon[0]) + m * lx, float(lon[-1]) - m * lx, n)
    y = rng.uniform(float(lat[0]) + m * ly, float(lat[-1]) - m * ly, n)
    if depth is None:
        z = np.zeros(n)
    else:
        lz = float(depth[-1] - depth[0])
        z = rng.uniform(float(depth[0]) + m * lz, float(depth[-1]) - m * lz, n)
    if spec["kernels"][0] in ("AdvectionRK4", "AdvectionEE", "AdvectionRK2") and depth is not None:
        z = np.abs(z)  # 2-D kernels: keep particles below the surface
    if spec.get("surface"):  # every particle exactly on the first depth level: zeta == 0 for the whole batch
        z = np.full(n, float(depth[0]))
    rel = spec.get("release", ("const", 0.0))
    t = np.full(n, rel[1]) if rel[0] == "const" else np.round(rng.uniform(rel[1], rel[2], n))
    uses_w = spec["kernels"][0].endswith("_3D")
    out.update(lon=lon, lat=lat, depth=depth, times=times, U=U, V=V, W=W if uses_w else None, x=x, y=y, z=z, t=t)
    if "kh" in spec:
        out["constants"] = {"Kh_zonal": spec["kh"][0], "Kh_meridional": spec["kh"][1]}
    return out
