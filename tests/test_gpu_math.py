"""The hand-written math primitives of the hot kernels, run on the device (pb_debug_math: the very inline functions the kernels
call), against a high-precision reference of the same operation.

* cos_np (common.cuh): cos of a latitude in radians -- the unit conversion of every spherical A-grid kernel and the curvilinear
  query vector;
* sin_lat / sincos_lon (cgrid.cuh): the per-sample trigonometry of the curvilinear search;
* div_by_cached / div_by_cached_guarded (common.cuh): division by a cached reciprocal (bcoords, the RK4 sum / 6, / deg2m);
* box_muller_f32 (common.cuh): the float32 Box-Muller transform of DiffusionUniformKh's Wiener increments;
* cosf / sinf / cos / sin (cgrid.cuh cosf_ool, sinf_ool, cos_ool, sin_ool): CUDA's own functions, as the kernels call them (the
  float32 unit conversions and hash queries, the per-cell table of the curvilinear search).  The oracle's engine-arithmetic mode
  (tests/device_trig.py) evaluates its sin / cos through these ops, so each must be the function its name says: CUDA's documented
  2 ulp of the exact value, float32 ulp for the float32 ops.
  Limit: a bound cannot tell CUDA's cosf from a correctly rounded float64 cos rounded to float32 (both are float32 values within
  2 float32 ulp), so a float32 op wired to (float)cos_ool would pass here.  That wiring is caught by the exact trajectory tests
  instead: afast.cu's stage-1 cos done in float64 and rounded fails test_gpu_parity / test_gpu_fast_kernel's `-exact` cases on the
  device.

Error unit: ulp of the EXACT value y, 2^(floor(log2|y|) - 52) for float64 results (an exact zero must come out as zero).  The
reference is np.longdouble (64-bit mantissa, asserted) for the dense sweeps and mpmath at 50 digits for the edge lists (long double
when mpmath does not import).  Under the host simulation of the kernel sources (PB_HOSTSIM_TEST=1) the sweeps are 2^16 samples
instead of 2^24 (the edge lists stay whole): the polynomial paths are bit-identical to the device there (explicit fma, no
contraction); the cold paths and sincospif are host libm, so only documented bounds are asserted for them.
"""

import os

import numpy as np
import pytest

from philox_ref import philox4x32_10

pytestmark = pytest.mark.gpu

HOSTSIM = os.environ.get("PB_HOSTSIM_TEST") == "1"
N = 2**16 if HOSTSIM else 2**24
N_BM = 2**16 if HOSTSIM else 2**20
N_F32 = 2**16 if HOSTSIM else 2**22

try:
    import mpmath as _mpmath

    MP = _mpmath.MPContext()  # a context of its own: the global mpmath.mp keeps its precision
    MP.dps = 50
except ImportError:  # pragma: no cover -- the edge lists then use long double as well
    MP = None

LD = np.longdouble
HI = 1.5707963267948966  # pi/2 rounded to float64 (below pi/2)
HI_NEXT = np.nextafter(HI, 2.0)  # 1.5707963267948968: the last argument of the polynomial paths of cos_np / sin_lat
HI_NEXT2 = np.nextafter(HI_NEXT, 2.0)  # 1.570796326794897: the first one that takes the cold path

# bounds asserted below (DESIGN.md section 4 states the same)
COS_NP_ULP = 2.5  # the single polynomial's cancellation near the equator (common.cuh)
SIN_LAT_ULP = 2.0
SINCOS_LON_ULP = 2.0
CUDA_TRIG_ULP = 2.0  # CUDA's documented bound for cos / sin / sincos: the cold paths
COS_NP_REGRESSION_X = 9.73785013376847e-09  # cos_np without its clamp returned 1.0000000000000002 here (exact: 0.99999999999999995257...)


@pytest.fixture(scope="module")
def eng():
    from parcels_b200.engine import Engine

    return Engine(0)


def _ld_ok():
    return np.finfo(LD).nmant >= 63


def _mpf(x):
    return MP.mpf(float(x))


def _ulp_err_ld(dev, exact):
    """|dev - exact| in ulp of exact (long double arithmetic); exact == 0 -> 0 if dev == 0 else inf"""
    exact = np.asarray(exact, dtype=LD)
    _, e = np.frexp(np.abs(exact))
    ulp = np.ldexp(LD(1), e - 53)
    with np.errstate(invalid="ignore", divide="ignore"):
        err = (np.abs(np.asarray(dev, dtype=LD) - exact) / ulp).astype(np.float64)
    z = exact == 0
    err[z] = np.where(np.asarray(dev)[z] == 0, 0.0, np.inf)
    return err


def _ulp_err(dev, x, fn_ld, fn_mp, edge):
    """error of dev = f(x) in ulp of the exact f(x): mpmath for edge lists (when it imports), long double otherwise"""
    x = np.asarray(x, dtype=np.float64)
    if edge and MP is not None:
        out = np.empty(x.size)
        for i, (d, xi) in enumerate(zip(np.asarray(dev, dtype=np.float64), x)):
            ex = fn_mp(_mpf(xi))
            if ex == 0:
                out[i] = 0.0 if d == 0 else np.inf
                continue
            _, e = MP.frexp(ex)
            out[i] = float(abs(_mpf(d) - ex) / MP.ldexp(1, int(e) - 53))
        return out
    assert _ld_ok(), f"np.longdouble has a {np.finfo(LD).nmant}-bit mantissa: too coarse as a reference"
    return _ulp_err_ld(dev, fn_ld(x.astype(LD)))


def _nbrs(x, k):
    """x and its k float64 neighbours on either side"""
    x = np.float64(x)
    out, lo, hi = [x], x, x
    for _ in range(k):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [lo, hi]
    return np.array(out)


def _deg2rad_np(d):
    return np.asarray(d, dtype=np.float64) * (np.pi / 180.0)  # np.deg2rad of float64 (deg2rad_np in common.cuh)


def _latitudes_dense(rng):
    uni = rng.uniform(-HI, HI, N)
    mag = np.exp2(-rng.uniform(1.0, 60.0, N))  # log-uniform magnitudes 2^-1 ... 2^-60, both signs
    return uni, mag * rng.choice([-1.0, 1.0], N)


def _latitudes_edge():
    nodes = _deg2rad_np(np.arange(-180, 181) * 0.5)  # every integer and half degree in [-90, 90]
    offs = [np.nextafter(nodes, np.inf), np.nextafter(nodes, -np.inf), nodes + 1e-9, nodes - 1e-9, nodes + 1e-13, nodes - 1e-13]
    pio4 = _nbrs(np.pi / 4, 64)  # Sterbenz boundary of hi - |x|
    top = np.array([HI, HI_NEXT, np.nextafter(HI, 0.0), np.nextafter(np.nextafter(HI, 0.0), 0.0)])
    tiny = np.array([5e-324, 2.2250738585072014e-308, 1e-300, 1e-20, 1e-16, 1.4901161193847656e-08, COS_NP_REGRESSION_X, 1e-4, 2e-4])
    x = np.concatenate([nodes, *offs, pio4, -pio4, top, -top, tiny, -tiny])
    return x[np.abs(x) <= HI_NEXT]


# ------------------------------------------------------------------------------------------------------------------------------
# cos_np
# ------------------------------------------------------------------------------------------------------------------------------
def _cos_np(eng, x):
    return eng.debug_math("cos_np", x)[:, 0]


def test_cos_np_error_bound_on_latitudes(eng):
    rng = np.random.default_rng(20261015)
    for name, x, edge in (*zip(("uniform", "log-uniform"), _latitudes_dense(rng), (False, False)), ("edges", _latitudes_edge(), True)):
        c = _cos_np(eng, x)
        err = _ulp_err(c, x, np.cos, MP.cos if MP else None, edge)
        i = int(np.argmax(err))
        assert err[i] <= COS_NP_ULP, f"cos_np {name}: {err[i]:.3f} ulp at x = {x[i]!r} (bound {COS_NP_ULP})"
        # the range of cos on [-pi/2, pi/2] (the argument HI_NEXT lies just beyond pi/2: its cosine is negative)
        inside = np.abs(x) <= HI
        bad = inside & ~((c >= 0.0) & (c <= 1.0))
        assert not bad.any(), f"{name}: cos_np outside [0, 1] at x = {x[bad][:5].tolist()}: {c[bad][:5].tolist()}"


def test_cos_np_is_even_and_exact_at_zero(eng):
    rng = np.random.default_rng(7)
    x = np.concatenate([*(np.abs(a) for a in _latitudes_dense(rng)), np.abs(_latitudes_edge())])
    c_pos, c_neg = _cos_np(eng, x), _cos_np(eng, -x)
    assert np.array_equal(c_pos.view(np.uint64), c_neg.view(np.uint64)), "cos_np(x) != cos_np(-x) bit for bit"
    assert np.array_equal(_cos_np(eng, np.array([0.0, -0.0])), [1.0, 1.0])


def test_cos_np_regression_value_near_the_equator(eng):
    """The value where cos_np without its clamp (sin(pi/2 - |x|) evaluated at r ~ pi/2) returned 1.0000000000000002."""
    c = _cos_np(eng, np.array([COS_NP_REGRESSION_X, -COS_NP_REGRESSION_X]))
    assert c[0] <= 1.0 and c[1] <= 1.0, c
    assert c[0] == 1.0 and c[1] == 1.0, c  # the correctly rounded value of 0.99999999999999995257...


def test_cos_np_cold_path_and_non_finite(eng):
    """|x| > pi/2 (not a latitude) and non-finite arguments take CUDA's cos (documented <= 2 ulp)."""
    x = np.array([HI_NEXT2, np.nextafter(HI_NEXT2, 3.0), 1.6, 2.0, 3.0, np.pi, 10.0, 100.0, 1e6, 1e15])
    x = np.concatenate([x, -x])
    c = _cos_np(eng, x)
    err = _ulp_err(c, x, np.cos, MP.cos if MP else None, True)
    assert err.max() <= CUDA_TRIG_ULP, (err.max(), x[np.argmax(err)])
    nf = _cos_np(eng, np.array([np.inf, -np.inf, np.nan, -np.nan]))
    assert np.isnan(nf).all(), nf


# ------------------------------------------------------------------------------------------------------------------------------
# sin_lat
# ------------------------------------------------------------------------------------------------------------------------------
def _sin_lat(eng, x):
    return eng.debug_math("sin_lat", x)[:, 0]


def test_sin_lat_error_bound_symmetry_and_range(eng):
    rng = np.random.default_rng(20261016)
    for name, x, edge in (*zip(("uniform", "log-uniform"), _latitudes_dense(rng), (False, False)), ("edges", _latitudes_edge(), True)):
        s = _sin_lat(eng, x)
        err = _ulp_err(s, x, np.sin, MP.sin if MP else None, edge)
        assert err.max() <= SIN_LAT_ULP, f"sin_lat {name}: {err.max():.3f} ulp at x = {x[np.argmax(err)]!r}"
        assert (np.abs(s) <= 1.0).all(), f"sin_lat {name}: |s| > 1 at {x[np.abs(s) > 1.0][:5].tolist()}"
        s_neg = _sin_lat(eng, -x)
        assert np.array_equal((-s).view(np.uint64)[x != 0], s_neg.view(np.uint64)[x != 0]), f"sin_lat {name}: sin_lat(-x) != -sin_lat(x)"
    # a zero latitude gives +0 for either sign (r + r^3 P rounds -0 + +0 to +0): the query vector's z component only enters sums
    # and products, where the sign of a zero is not observable
    assert np.array_equal(_sin_lat(eng, np.array([0.0, -0.0])), [0.0, 0.0])


def test_sin_lat_cold_path_and_non_finite(eng):
    x = np.array([HI_NEXT2, 1.6, 2.0, 3.0, 10.0, 1e6])
    x = np.concatenate([x, -x])
    err = _ulp_err(_sin_lat(eng, x), x, np.sin, MP.sin if MP else None, True)
    assert err.max() <= CUDA_TRIG_ULP, (err.max(), x[np.argmax(err)])
    assert np.isnan(_sin_lat(eng, np.array([np.inf, -np.inf, np.nan]))).all()


# ------------------------------------------------------------------------------------------------------------------------------
# sincos_lon
# ------------------------------------------------------------------------------------------------------------------------------
def _lon_edge():
    k = np.arange(-8, 9)
    mult = np.concatenate([_nbrs(kk * (np.pi / 2), 64) for kk in k])  # +-64 ulp around the float64 nearest to k pi/2
    mult = np.concatenate([mult, np.array([kk * 1.5707963267948966 for kk in k])])  # k * hi (the reduction's own multiples)
    halfq = np.concatenate([_nbrs((kk + 0.5) * (np.pi / 2), 4) for kk in np.arange(-9, 9)])  # where round(x 2/pi) flips
    deg = _deg2rad_np(np.arange(-1440, 1441) * 0.5)  # every half degree in [-720, 720]
    x = np.concatenate([mult, halfq, deg, [13.0, -13.0, np.nextafter(13.0, 0.0), -np.nextafter(13.0, 0.0)]])
    return x[np.abs(x) <= 13.0]


def _check_sincos(eng, x, edge, bound, what):
    out = eng.debug_math("sincos_lon", x)
    s, c = out[:, 0], out[:, 1]
    es = _ulp_err(s, x, np.sin, MP.sin if MP else None, edge)
    ec = _ulp_err(c, x, np.cos, MP.cos if MP else None, edge)
    assert es.max() <= bound, f"sincos_lon {what}: sin {es.max():.3f} ulp at x = {x[np.argmax(es)]!r}"
    assert ec.max() <= bound, f"sincos_lon {what}: cos {ec.max():.3f} ulp at x = {x[np.argmax(ec)]!r}"
    assert (np.abs(s) <= 1.0).all() and (np.abs(c) <= 1.0).all(), what
    pyth = np.abs(s.astype(LD) ** 2 + c.astype(LD) ** 2 - 1)
    assert pyth.max() <= 4 * 2.0**-52, f"sincos_lon {what}: s^2 + c^2 - 1 = {float(pyth.max()):.3g} at x = {x[np.argmax(pyth)]!r}"


def test_sincos_lon_uniform(eng):
    rng = np.random.default_rng(20261017)
    _check_sincos(eng, rng.uniform(-13.0, 13.0, N), False, SINCOS_LON_ULP, "uniform")


def test_sincos_lon_edges(eng):
    _check_sincos(eng, _lon_edge(), True, SINCOS_LON_ULP, "edges")
    z = eng.debug_math("sincos_lon", np.array([0.0, -0.0]))
    assert np.array_equal(z, [[0.0, 1.0], [0.0, 1.0]])  # (sin of -0 is +0, as for sin_lat)


def test_sincos_lon_cold_path_and_non_finite(eng):
    """|x| > 13 takes CUDA's sincos (documented <= 2 ulp)."""
    x = np.array([np.nextafter(13.0, 14.0), 13.5, 20.0, 100.0, 1e4, 1e9])
    x = np.concatenate([x, -x])
    _check_sincos(eng, x, True, CUDA_TRIG_ULP, "cold path")
    nf = eng.debug_math("sincos_lon", np.array([np.inf, -np.inf, np.nan]))
    assert np.isnan(nf).all(), nf


# ------------------------------------------------------------------------------------------------------------------------------
# CUDA's cosf / sinf / cos / sin, out of line as the kernels call them
# ------------------------------------------------------------------------------------------------------------------------------
def _f32_args(rng):
    """float32 radians: uniform on [-4 pi, 4 pi], log-uniform magnitudes 2^-1 ... 2^-40, every half degree in [-720, 720] converted
    like np.deg2rad of float32, and +-8 float32 neighbours of k pi/2 for |k| <= 16"""
    f32 = np.float32
    uni = rng.uniform(-4 * np.pi, 4 * np.pi, N_F32).astype(f32)
    mag = (np.exp2(-rng.uniform(1.0, 40.0, N_F32)) * rng.choice([-1.0, 1.0], N_F32)).astype(f32)
    deg = (np.arange(-1440, 1441) * 0.5).astype(f32) * f32(np.pi / 180.0)
    mult = []
    for k in range(-16, 17):
        x = f32(k * (np.pi / 2))
        lo = hi = x
        mult.append(x)
        for _ in range(8):
            lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
            mult += [lo, hi]
    return np.concatenate([uni, mag, deg, np.array(mult, dtype=f32)])


def _ulp_err_f32(dev, exact):
    """|dev - exact| in float32 ulp of exact (long double arithmetic)"""
    exact = np.asarray(exact, dtype=LD)
    _, e = np.frexp(np.abs(exact))
    ulp = np.ldexp(LD(1), e - 24)
    return (np.abs(np.asarray(dev, dtype=LD) - exact) / ulp).astype(np.float64)


@pytest.mark.parametrize("op, fn", [("cosf", np.cos), ("sinf", np.sin)])
def test_cuda_float32_trig_error_bound(eng, op, fn):
    assert _ld_ok()
    x = _f32_args(np.random.default_rng(20261018))
    out = eng.debug_math(op, x.astype(np.float64))[:, 0]
    assert np.array_equal(out, out.astype(np.float32).astype(np.float64)), f"{op}: a result that is not a float32 value"
    err = _ulp_err_f32(out, fn(x.astype(LD)))
    assert err.max() <= CUDA_TRIG_ULP, f"{op}: {err.max():.3f} float32 ulp at x = {x[np.argmax(err)]!r}"
    z = eng.debug_math(op, np.array([0.0, -0.0]))[:, 0]
    assert np.array_equal(z, [1.0, 1.0] if op == "cosf" else [0.0, -0.0]) and (op == "cosf" or np.signbit(z[1]))
    assert np.isnan(eng.debug_math(op, np.array([np.inf, -np.inf, np.nan]))[:, 0]).all()


def test_cuda_float32_trig_rounds_its_argument_to_float32(eng):
    """The float32 ops see the float32 value carried in the double slot: a float64 argument is rounded first."""
    x = np.array([0.1, 1.0 + 2.0**-40, 2.5], dtype=np.float64)
    for op in ("cosf", "sinf"):
        np.testing.assert_array_equal(eng.debug_math(op, x)[:, 0], eng.debug_math(op, x.astype(np.float32).astype(np.float64))[:, 0])


@pytest.mark.parametrize("op, fn_ld, fn_mp", [("cos", np.cos, "cos"), ("sin", np.sin, "sin")])
def test_cuda_float64_trig_error_bound(eng, op, fn_ld, fn_mp):
    rng = np.random.default_rng(20261019)
    fmp = getattr(MP, fn_mp) if MP else None
    uni = rng.uniform(-4 * np.pi, 4 * np.pi, N)
    err = _ulp_err(eng.debug_math(op, uni)[:, 0], uni, fn_ld, fmp, False)
    assert err.max() <= CUDA_TRIG_ULP, f"{op} uniform: {err.max():.3f} ulp at x = {uni[np.argmax(err)]!r}"
    edge = np.concatenate([_lon_edge(), _latitudes_edge(), [20.0, 100.0, 1e4, -1e9]])
    err = _ulp_err(eng.debug_math(op, edge)[:, 0], edge, fn_ld, fmp, True)
    assert err.max() <= CUDA_TRIG_ULP, f"{op} edges: {err.max():.3f} ulp at x = {edge[np.argmax(err)]!r}"
    assert np.isnan(eng.debug_math(op, np.array([np.inf, -np.inf, np.nan]))[:, 0]).all()


# ------------------------------------------------------------------------------------------------------------------------------
# division by a cached reciprocal
# ------------------------------------------------------------------------------------------------------------------------------
def _bits_equal(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    return both_nan | (a.view(np.uint64) == b.view(np.uint64))


def _division_operands(rng, n):
    """oracle/division_check.c's distributions: bcoord-like 0 <= a <= b over 2^+-20 widths, random mantissas (exponents +-30),
    the hot path's constant divisors 6 and 111120 (deg2m), quotients next to rounding midpoints"""
    m = n // 5
    b1 = np.ldexp(1.0 + rng.random(m), rng.integers(-20, 20, m))
    a1 = b1 * rng.random(m)
    mant = lambda k: rng.integers(0, 2**52, k, dtype=np.uint64)  # noqa: E731
    ex = lambda k: rng.integers(1023 - 30, 1023 + 30, k).astype(np.uint64)  # noqa: E731
    a2 = (mant(m) | (ex(m) << np.uint64(52))).view(np.float64)
    b2 = (mant(m) | (ex(m) << np.uint64(52))).view(np.float64)
    a3 = np.ldexp(1.0 + rng.random(2 * m), rng.integers(-50, 10, 2 * m)) * rng.choice([-1.0, 1.0], 2 * m)
    b3 = np.where(np.arange(2 * m) % 2 == 0, 6.0, 111120.0)
    q = 1.0 + rng.random(m)
    mid = 0.5 * (q + np.nextafter(q, 2.0))
    b4 = 1.0 + rng.random(m)
    a4 = mid * b4
    return np.concatenate([a1, a2, a3, a4]), np.concatenate([b1, b2, b3, b4])


@pytest.mark.parametrize("op", ["div_by_cached", "div_by_cached_guarded"])
def test_division_by_cached_reciprocal_is_correctly_rounded(eng, op):
    rng = np.random.default_rng(20261018)
    a, b = _division_operands(rng, N)
    k = min(N // 5, a.size)
    a = np.concatenate([a, -a[:k], np.zeros(64), b[:k]])  # negative numerators (a particle left of the axis), a == 0, a == b
    b = np.concatenate([b, b[:k], b[:64], b[:k]])
    out = eng.debug_math(op, a, b)
    assert np.array_equal(out[:, 1], 1.0 / b), "the device's reciprocal is not RN(1 / b)"
    ok = _bits_equal(out[:, 0], a / b)
    assert ok.all(), f"{op}: {int((~ok).sum())} of {a.size} differ from a / b, e.g. a = {a[~ok][:3].tolist()}, b = {b[~ok][:3].tolist()}"


def test_div_by_cached_subnormal_numerators_within_one_unit(eng):
    """The unguarded form assumes normal-range intermediates (bcoords): a subnormal numerator is within one unit of 2^-1074 of
    the quotient, not always correctly rounded -- the precondition DESIGN.md states.  Divisors >= 1 (cell widths, 6, deg2m)."""
    rng = np.random.default_rng(20261019)
    n = N // 4
    a = rng.integers(1, 2**52, n, dtype=np.uint64).view(np.float64) * rng.choice([-1.0, 1.0], n)
    b = np.concatenate([np.ldexp(1.0 + rng.random(n - 64), rng.integers(0, 20, n - 64)), np.full(32, 6.0), np.full(32, 111120.0)])
    out = eng.debug_math("div_by_cached", a, b)[:, 0]
    units = np.abs(out - a / b) / 5e-324  # the difference of two subnormals is exact
    assert units.max() <= 1.0, (units.max(), a[np.argmax(units)], b[np.argmax(units)])


def test_div_by_cached_guarded_matches_division_for_every_numerator(eng):
    """Velocities come from data: zeros (sign kept), subnormals, huge values, non-finite ones and the neighbours of the guard's
    1e-280 / 1e280 thresholds must all give exactly a / b."""
    rng = np.random.default_rng(20261020)
    special = np.array([0.0, 5e-324, 1e-310, 2.2250738585072014e-308, 1e-300, 1e300, 1.7976931348623157e308, np.inf, np.nan, 1.0])
    thresholds = np.concatenate([_nbrs(1e-280, 8), _nbrs(1e280, 8)])
    anywhere = rng.integers(0, 2**63, N // 4, dtype=np.uint64).view(np.float64)  # every exponent, subnormals and NaNs included
    a = np.concatenate([special, thresholds, anywhere])
    a = np.concatenate([a, -a])
    widths = np.concatenate([np.ldexp(1.0 + rng.random(a.size - 2), rng.integers(-20, 20, a.size - 2)), [6.0, 111120.0]])
    for b in (widths, np.full(a.size, 6.0), np.full(a.size, 111120.0)):
        out = eng.debug_math("div_by_cached_guarded", a, b)[:, 0]
        with np.errstate(all="ignore"):
            ok = _bits_equal(out, a / b)
        assert ok.all(), f"{int((~ok).sum())} differ, e.g. a = {a[~ok][:3].tolist()}, b = {b[~ok][:3].tolist()}"


# ------------------------------------------------------------------------------------------------------------------------------
# Box-Muller
# ------------------------------------------------------------------------------------------------------------------------------
U32 = 2.0**-24  # float32 unit roundoff
# relative error of zx = rad * c (and zy) against the exact transform of the device's u1, u2 -- from the documented accuracy:
#   logf <= 1 ulp  -> -2 ln u1 relative <= 2 U32, halved by the square root   : U32
#   sqrtf correctly rounded                                                   : U32
#   sincospif <= 1 ulp                                                        : 2 U32
#   rad * c rounded to float32                                                : U32
# (the float64 conversion is exact; u1, u2 are the float32 values the device defines, so they carry no error here)
BM_REL = 5 * U32 * (1 + 1e-6)  # about 2.5 float32 ulp of the result's binade, <= 5 ulp of its own


def _u_from_words(r0, r1):
    f32 = np.float32
    u1 = (np.asarray(r0, dtype=np.uint32).astype(f32) + f32(0.5)) * f32(2.0**-32)
    u2 = (np.asarray(r1, dtype=np.uint32).astype(f32) + f32(0.5)) * f32(2.0**-32)
    return u1, u2


def _bm_exact_ld(u1, u2):
    """sqrt(-2 ln u1) (cos, sin)(2 pi u2) in long double, the angle reduced exactly in half-turns (exact zeros where they are)"""
    assert _ld_ok()
    pi = 4 * np.arctan(LD(1))
    rad = np.sqrt(-2 * np.log(u1.astype(LD)))
    r = np.remainder(2 * u2.astype(np.float64), 2.0)  # exact
    r = np.where(r > 1.0, r - 2.0, r)  # [-1, 1], exact
    a = np.abs(r)
    s = np.copysign(np.sin(pi * np.minimum(a, 1.0 - a).astype(LD)), r.astype(LD))
    c = np.where(a < 0.25, np.cos(pi * a.astype(LD)), np.sin(pi * (0.5 - a).astype(LD)))
    return rad * c, rad * s


def _bm_exact_mp(u1, u2):
    zx, zy = [], []
    for a, b in zip(u1, u2):
        rad = MP.sqrt(-2 * MP.log(_mpf(a)))
        zx.append(rad * MP.cospi(2 * _mpf(b)))
        zy.append(rad * MP.sinpi(2 * _mpf(b)))
    return zx, zy


def _bm_check(eng, r0, r1, edge):
    out = eng.debug_math("box_muller_f32", r0.astype(np.float64), r1.astype(np.float64))
    assert np.isfinite(out).all(), "non-finite Box-Muller output"
    assert np.abs(out).max() <= 6.8, np.abs(out).max()
    # every output is a float32 value
    assert np.array_equal(out.astype(np.float32).astype(np.float64), out)
    u1, u2 = _u_from_words(r0, r1)
    if edge and MP is not None:
        ex = _bm_exact_mp(u1, u2)
        for j in range(2):
            for d, e in zip(out[:, j], ex[j]):
                assert abs(_mpf(d) - e) <= BM_REL * abs(e), (j, d, e)
    else:
        ex = _bm_exact_ld(u1, u2)
        for j in range(2):
            err = np.abs(out[:, j].astype(LD) - ex[j])
            lim = BM_REL * np.abs(ex[j])
            bad = err > lim
            assert not bad.any(), f"component {j}: relative error {float((err / np.abs(ex[j]))[bad].max()):.3g} > {BM_REL:.3g}"
    return out, u1


def test_box_muller_random_words(eng):
    rng = np.random.default_rng(20261021)
    r0 = rng.integers(0, 2**32, N_BM, dtype=np.uint64).astype(np.uint32)
    r1 = rng.integers(0, 2**32, N_BM, dtype=np.uint64).astype(np.uint32)
    _bm_check(eng, r0, r1, False)


def test_box_muller_extreme_words(eng):
    w0 = np.array([0, 1, 2**24 - 1, 2**24, 2**32 - 1], dtype=np.uint32)
    w1 = np.array([0, 2**30, 2**31, 3 * 2**30, 2**32 - 1], dtype=np.uint32)
    r0, r1 = (g.ravel() for g in np.meshgrid(w0, w1, indexing="ij"))
    out, u1 = _bm_check(eng, r0, r1, True)
    top = r0 == 2**32 - 1
    assert (u1[top] == np.float32(1.0)).all()
    assert (out[top] == 0.0).all(), out[top]  # u1 == 1: ln u1 == 0 exactly
    assert np.abs(out[r0 == 0]).max() > 6.7  # u1 = 2^-33 keeps its tail: |z| reaches 6.76


def test_debug_normals_is_box_muller_of_the_philox_words(eng):
    """pb_debug_normals (the kernels' wiener_normals) == box_muller_f32 of the Philox words of tests/philox_ref.py, bit for bit:
    ties the transform checked above to the stream the diffusion kernels draw."""
    seed, rng_call, it = 0xDEADBEEFCAFE, (5 << 32) + 3, 17
    pid = np.concatenate([np.arange(10**6 - 4, dtype=np.int64), [2**33 + 7, 10**12, 2**62, -1]])
    dev = eng.debug_normals(seed=seed, rng_call=rng_call, it=it, particle_id=pid)
    u = pid.view(np.uint64)
    mask = np.uint64(0xFFFFFFFF)
    r0, r1, _, _ = philox4x32_10((u & mask).astype(np.uint32), (u >> np.uint64(32)).astype(np.uint32),
                                 np.full(pid.size, np.uint32(it)), np.full(pid.size, np.uint32(rng_call & 0xFFFFFFFF)),
                                 seed & 0xFFFFFFFF, ((seed >> 32) ^ (rng_call >> 32)) & 0xFFFFFFFF)  # fmt: skip
    bm = eng.debug_math("box_muller_f32", r0.astype(np.float64), r1.astype(np.float64))
    assert np.array_equal(dev.view(np.uint64), bm.view(np.uint64))


def test_debug_math_rejects_bad_arguments(eng):
    from parcels_b200._lib import EngineError

    with pytest.raises(EngineError):
        eng.debug_math("div_by_cached", np.ones(4))  # a binary op without its second operand
    out = eng.debug_math("cos_np", np.zeros(0))
    assert out.shape == (0, 2)
