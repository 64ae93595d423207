// cgrid.cuh -- C-grid policy of advect_kernel (instantiated in cgrid.cu; curva.cu instantiates the curvilinear search with the
// A-grid interpolator): CGrid_Velocity on rectilinear and curvilinear grids
// (reference interpolators/_xinterpolators.py:193-332), the curvilinear cell search with hint
// (_core/index_search.py:94-295) and the device-side spatial-hash query (_core/spatialhash.py:389-535;
// the table is built once on the host and uploaded).
//
// Per particle, in registers: the current cell (yi, xi), its 4 corner lon/lat, on spherical
// curvilinear meshes the cell's tangent-plane basis and projected corners, and the 2 faces x 2
// time levels of U, V, W that CGrid_Velocity reads.  Everything is re-gathered from HBM only when the
// particle changes cell / time level.
#pragma once
#include "common.cuh"
#include "rk45.cuh"

// np.remainder for a positive divisor (floored modulo), in the array dtype
__device__ __forceinline__ float mod_np(float a, float b) {
    float r = fmodf(a, b);
    if (r != 0.f) { if (r < 0.f) r += b; } else r = copysignf(0.f, b);
    return r;
}
__device__ __forceinline__ double mod_np(double a, double b) {
    double r = fmod(a, b);
    if (r != 0.0) { if (r < 0.0) r += b; } else r = copysign(0.0, b);
    return r;
}
// Out-of-line transcendentals: the curvilinear path evaluates ~13 double-precision sin/cos per sample;
// inlining each expansion (~200 SASS instructions) made the kernel overflow the instruction cache
// (ncu: stall_no_inst dominant).  One shared copy each.
static __device__ __noinline__ double cos_ool(double x) { return cos(x); }
static __device__ __noinline__ double sin_ool(double x) { return sin(x); }
static __device__ __noinline__ float cosf_ool(float x) { return cosf(x); }
static __device__ __noinline__ float sinf_ool(float x) { return sinf(x); }
__device__ __forceinline__ float cosx(float x) { return cosf_ool(x); }
__device__ __forceinline__ double cosx(double x) { return cos_np(x); }  // (a latitude: common.cuh's polynomial, inline)
// Per-sample trigonometry of the curvilinear search (out-of-line cos / sin like the ones above would be 24 + 8 calls of ~70
// instructions per warp and step on config 3).  The query's unit vector needs
// sin / cos of a LATITUDE (|x| <= pi/2: one odd polynomial each, like cos_np) and of a LONGITUDE (|x| <= 4 pi: one shared
// quadrant reduction + the two fdlibm kernel polynomials on [-pi/4, pi/4]); <= 2 ulp like CUDA's own, anything outside those
// ranges takes sincos().  The one-time per-cell table (project_cell) keeps CUDA's sin / cos.
static __device__ __noinline__ void sincos_cold(double x, double* s, double* c) { sincos(x, s, c); }
__device__ __forceinline__ double sin_lat(double x) {
    if (!(fabs(x) <= 1.5707963267948968)) { double s, c; sincos_cold(x, &s, &c); return s; }
    return sin_poly_pio2(x);
}
// fdlibm __kernel_sin / __kernel_cos coefficients (highest first), in constant memory like PB_SIN_TAYLOR
static __constant__ double PB_KSIN[6] = {1.58969099521155010221e-10, -2.50507602534068634195e-08, 2.75573137070700676789e-06,
                                         -1.98412698298579493134e-04, 8.33333333332248946124e-03, -1.66666666666666324348e-01};
static __constant__ double PB_KCOS[6] = {-1.13596475577881948265e-11, 2.08757232129817482790e-09, -2.75573143513906633035e-07,
                                         2.48015872894767294178e-05, -1.38888888888741095749e-03, 4.16666666666666019037e-02};
__device__ __forceinline__ void sincos_lon(double x, double& sn, double& cs) {
    if (!(fabs(x) <= 13.0)) { sincos_cold(x, &sn, &cs); return; }
    const double t = x * 0.63661977236758138 + 6755399441055744.0;  // round(x * 2 / pi) by the 1.5 * 2^52 trick
    const double kf = t - 6755399441055744.0;
    const int k = (int)kf;
    double r = fma(-kf, 1.5707963267948966, x);  // Cody-Waite, pi/2 = hi + lo (|k| <= 8)
    r = fma(-kf, 6.123233995736766e-17, r);
    const double z = r * r;
    double ps = PB_KSIN[0], pc = PB_KCOS[0];
#pragma unroll
    for (int j = 1; j < 6; ++j) { ps = fma(ps, z, PB_KSIN[j]); pc = fma(pc, z, PB_KCOS[j]); }
    const double s0 = fma(r * z, ps, r);
    const double c0 = fma(z, fma(z, pc, -0.5), 1.0);
    const double a = (k & 1) ? c0 : s0, b = (k & 1) ? s0 : c0;  // quadrant k & 3: (s, c), (c, -s), (-s, -c), (-c, s)
    sn = (k & 2) ? -a : a;
    cs = ((k + 1) & 2) ? -b : b;
}
__device__ __forceinline__ float sinx(float x) { return sinf_ool(x); }
__device__ __forceinline__ double sinx(double x) { return sin_ool(x); }
__device__ __forceinline__ float sqrt_np(float x) { return sqrtf(x); }
__device__ __forceinline__ double sqrt_np(double x) { return sqrt(x); }

template <class A, class D>
struct CGridCtx {
    AxisCell<A> cz, cy, cx;  // cy, cx: rectilinear grids only
    AxisCell<double> ct;
    int yi, xi;              // horizontal cell of the last search (curvilinear: -3 after a failed search)
    int kyi, kxi;            // cell whose corners are cached below (INT_MIN: none)
    A clon[4], clat[4];      // raw corner lon/lat, CCW from (yi, xi)
    int uyi, uxi;            // curvilinear: cell whose unwrapped corner longitudes are cached in ulon (INT_MIN: none)
    A ulon[4];               // corner longitudes wrapped to [-180, 180) and unwrapped relative to corner 0 (:230-233)
    double pu[4], pv[4];     // spherical curvilinear: corners projected on the cell's tangent plane
    double eu[3], ev[3];     //                        orthonormal basis of that plane
    int fti, fzi, fyi, fxi;  // key of the cached face values
    D fu[4], fv[4], fw[4];   // [time level * 2 + face]
    int state, ei;
    unsigned int refills;
    bool out_of_time;
    signed char len_t, len_z;  // lenT / lenZ of the batch when known (0 / 1), -1: decide per particle (see EvalCtx, agrid.cuh)
};

// ------------------------------------------------------------------------------------------------
// curvilinear point-in-cell (index_search.py:94-239)
// ------------------------------------------------------------------------------------------------
// Tangent-plane basis and projected corners of ONE cell (_spherical_project_cell_and_query, cell part,
// index_search.py:203-236).  out[16] = pu[4], pv[4], eu[3], ev[3], 2 pad.
template <class A>
__device__ __forceinline__ void project_cell(const A (&clon)[4], const A (&clat)[4], double (&pu)[4], double (&pv)[4],
                                             double (&eu)[3], double (&ev)[3]) {
    double cX[4], cY[4], cZ[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double la = deg2rad_np((double)clat[k]), lo = deg2rad_np((double)clon[k]);
        const double cl = cos_ool(la);
        cX[k] = cos_ool(lo) * cl; cY[k] = sin_ool(lo) * cl; cZ[k] = sin_ool(la);
    }
    double ux = (cX[1] + cX[2]) - (cX[0] + cX[3]);
    double uy = (cY[1] + cY[2]) - (cY[0] + cY[3]);
    double uz = (cZ[1] + cZ[2]) - (cZ[0] + cZ[3]);
    double un = sqrt(ux * ux + uy * uy + uz * uz);
    if (un == 0.0) un = 1.0;
    eu[0] = ux / un; eu[1] = uy / un; eu[2] = uz / un;
    double vx = (cX[2] + cX[3]) - (cX[0] + cX[1]);
    double vy = (cY[2] + cY[3]) - (cY[0] + cY[1]);
    double vz = (cZ[2] + cZ[3]) - (cZ[0] + cZ[1]);
    const double d = vx * eu[0] + vy * eu[1] + vz * eu[2];
    vx = vx - d * eu[0]; vy = vy - d * eu[1]; vz = vz - d * eu[2];
    double vn = sqrt(vx * vx + vy * vy + vz * vz);
    if (vn == 0.0) vn = 1.0;
    ev[0] = vx / vn; ev[1] = vy / vn; ev[2] = vz / vn;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        pu[k] = cX[k] * eu[0] + cY[k] * eu[1] + cZ[k] * eu[2];
        pv[k] = cX[k] * ev[0] + cY[k] * ev[1] + cZ[k] * ev[2];
    }
}

// One thread per cell, once per grid upload: the projections every point-in-cell test needs.  Same device
// function as the on-the-fly path => bit-identical values; a candidate test then costs 16 loads, no trig.
template <class A>
__global__ void precompute_cells_kernel(const A* __restrict__ lon, const A* __restrict__ lat, int ny, int nx, double* __restrict__ out) {
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long ncell = (long long)(ny - 1) * (nx - 1);
    if (c >= ncell) return;
    const int j = (int)(c / (nx - 1)), i = (int)(c % (nx - 1));
    const long long o00 = (long long)j * nx + i;
    const A clon[4] = {lon[o00], lon[o00 + 1], lon[o00 + nx + 1], lon[o00 + nx]};
    const A clat[4] = {lat[o00], lat[o00 + 1], lat[o00 + nx + 1], lat[o00 + nx]};
    double pu[4], pv[4], eu[3], ev[3];
    project_cell<A>(clon, clat, pu, pv, eu, ev);
    double* o = out + c * 16;
#pragma unroll
    for (int k = 0; k < 4; ++k) { o[k] = pu[k]; o[4 + k] = pv[k]; }
#pragma unroll
    for (int k = 0; k < 3; ++k) { o[8 + k] = eu[k]; o[11 + k] = ev[k]; }
    o[14] = 0.0; o[15] = 0.0;
}


template <class A, class D>
__device__ __forceinline__ void load_corners(const GridDev& g, CGridCtx<A, D>& e, int j, int i) {
    if (e.kyi == j && e.kxi == i) return;
    e.kyi = j; e.kxi = i;
    const A* __restrict__ lon = (const A*)g.lon;
    const A* __restrict__ lat = (const A*)g.lat;
    const long long nx = g.nx;
    const long long o00 = (long long)j * nx + i;
    e.clon[0] = ldg(lon + o00);          e.clat[0] = ldg(lat + o00);
    e.clon[1] = ldg(lon + o00 + 1);      e.clat[1] = ldg(lat + o00 + 1);
    e.clon[2] = ldg(lon + o00 + nx + 1); e.clat[2] = ldg(lat + o00 + nx + 1);
    e.clon[3] = ldg(lon + o00 + nx);     e.clat[3] = ldg(lat + o00 + nx);
    if (g.spherical) {
        if (g.cellproj) {
            const double2* __restrict__ c = reinterpret_cast<const double2*>(g.cellproj + ((long long)j * (nx - 1) + i) * 16);
            const double2 q0 = __ldg(c), q1 = __ldg(c + 1), q2 = __ldg(c + 2), q3 = __ldg(c + 3), q4 = __ldg(c + 4), q5 = __ldg(c + 5),
                          q6 = __ldg(c + 6);
            e.pu[0] = q0.x; e.pu[1] = q0.y; e.pu[2] = q1.x; e.pu[3] = q1.y;
            e.pv[0] = q2.x; e.pv[1] = q2.y; e.pv[2] = q3.x; e.pv[3] = q3.y;
            e.eu[0] = q4.x; e.eu[1] = q4.y; e.eu[2] = q5.x;
            e.ev[0] = q5.y; e.ev[1] = q6.x; e.ev[2] = q6.y;
        }
        // (no on-the-fly fallback: pb_grid_upload_curvilinear always builds the table for spherical meshes, and keeping
        //  project_cell's ~2000 SASS instructions out of the advect kernel is a quarter of its code size)
    }
}

// _bilinear_inverse (index_search.py:132-149); np.dot(_invA, p) sums left to right.  Out of line (one copy,
// shared by the hint, neighbour and hash-candidate tests) with everything passed and returned in registers.
struct BilinearInv {
    double xsi, eta;
    bool inside;
};
static __device__ __noinline__ BilinearInv bilinear_inverse_v(double px0, double px1, double px2, double px3, double py0, double py1,
                                                       double py2, double py3, double xq, double yq) {
    const double a0 = px0, a1 = px1 - px0, a2 = px3 - px0, a3 = ((px0 - px1) + px2) - px3;
    const double b0 = py0, b1 = py1 - py0, b2 = py3 - py0, b3 = ((py0 - py1) + py2) - py3;
    const double aa = a3 * b2 - a2 * b3;
    const double bb = a3 * b0 - a0 * b3 + a1 * b2 - a2 * b1 + xq * b3 - yq * a3;
    const double cc = a1 * b0 - a0 * b1 + xq * b1 - yq * a1;
    const double det2 = bb * bb - 4 * aa * cc;
    const double det = det2 > 0 ? sqrt(det2) : -1.0;
    BilinearInv r;
    r.eta = fabs(aa) < 1e-12 ? -cc / bb : (det2 > 0 ? (-bb + det) / (2 * aa) : -1.0);
    const double den = a1 + a3 * r.eta;
    r.xsi = fabs(den) < 1e-12 ? ((yq - py0) / (py1 - py0) + (yq - py3) / (py2 - py3)) * 0.5 : (xq - a0 - a2 * r.eta) / den;
    r.inside = r.xsi >= 0 && r.xsi <= 1 && r.eta >= 0 && r.eta <= 1;
    return r;
}
__device__ __forceinline__ bool bilinear_inverse(const double (&px)[4], const double (&py)[4], double xq, double yq,
                                                 double& xsi, double& eta) {
    const BilinearInv r = bilinear_inverse_v(px[0], px[1], px[2], px[3], py[0], py[1], py[2], py[3], xq, yq);
    xsi = r.xsi; eta = r.eta;
    return r.inside;
}

struct Query {  // the sampled point, prepared once per eval
    double x, y;     // degrees (float64, as point_in_cell casts them)
    double qu_x, qu_y, qu_z;  // unit-sphere xyz in float64 (spherical)
};

template <class A, class D>
__device__ __forceinline__ bool point_in_cell(const GridDev& g, CGridCtx<A, D>& e, int j, int i, const Query& q,
                                              double& xsi, double& eta) {
    load_corners(g, e, j, i);
    if (g.spherical) {
        const double qu = q.qu_x * e.eu[0] + q.qu_y * e.eu[1] + q.qu_z * e.eu[2];
        const double qv = q.qu_x * e.ev[0] + q.qu_y * e.ev[1] + q.qu_z * e.ev[2];
        return bilinear_inverse(e.pu, e.pv, qu, qv, xsi, eta);
    }
    double px[4], py[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { px[k] = (double)e.clon[k]; py[k] = (double)e.clat[k]; }
    return bilinear_inverse(px, py, q.x, q.y, xsi, eta);
}

// ------------------------------------------------------------------------------------------------
// spatial-hash query (spatialhash.py:389-535, quantize :647-695, Morton :554-597,698-716)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int dilate10(unsigned int n) {
    n &= 0x000003FFu;
    n = (n | (n << 16)) & 0xFF0000FFu;
    n = (n | (n << 8)) & 0x0300F00Fu;
    n = (n | (n << 4)) & 0x030C30C3u;
    n = (n | (n << 2)) & 0x09249249u;
    return n;
}
// The hash-grid bounds are scalars of the grid's coordinate dtype A (np.nanmin of A-typed arrays), so
// the normalisation runs in Q = promote(dtype of the sampled position, A).
template <class Q, class A, class P>
__device__ __forceinline__ unsigned int quant(P v, double lo_, double hi_, int bw) {
    const A lo = (A)lo_, hi = (A)hi_;
    const A d = hi - lo;
    const Q vn = d != 0 ? ((Q)v - (Q)lo) / (Q)d : (Q)0;
    Q s = vn * (Q)bw;
    s = s < (Q)0 ? (Q)0 : (s > (Q)bw ? (Q)bw : s);  // np.clip (NaN coordinates are rejected by the finite test)
    return (unsigned int)s;
}

// quantised hash-grid coordinates of the sampled point (spatialhash.py:417-431,647-695)
template <class A, class PY, class PX>
__device__ __forceinline__ void hash_coords(const GridDev& g, PY y, PX x, unsigned int& qx, unsigned int& qy, unsigned int& qz) {
    using P = prom_t<PY, PX>;
    using Q = prom_t<P, A>;
    P hx, hy, hz;
    if (g.spherical) {  // trig in the dtype of the sampled position (spatialhash.py:417-421)
        const PY lat = deg2rad_np(y);
        const PX lon = deg2rad_np(x);
        hx = cosx(lon) * cosx(lat);
        hy = sinx(lon) * cosx(lat);
        hz = sinx(lat);
    } else {
        hx = x; hy = y; hz = 0;
    }
    qx = quant<Q, A>(hx, g.hbox[0], g.hbox[1], g.hash_bitwidth);
    qy = quant<Q, A>(hy, g.hbox[2], g.hbox[3], g.hash_bitwidth);
    qz = quant<Q, A>(hz, g.hbox[4], g.hbox[5], g.hash_bitwidth);
}

// same for a float64 position on a spherical mesh whose unit vector is already known: the query vector of the point-in-cell
// tests is cos(lon) cos(lat), sin(lon) cos(lat), sin(lat) of the same float64 radians -- the very expressions above
template <class A>
__device__ __forceinline__ void hash_coords_xyz(const GridDev& g, double hx, double hy, double hz, unsigned int& qx, unsigned int& qy,
                                                unsigned int& qz) {
    qx = quant<double, A>(hx, g.hbox[0], g.hbox[1], g.hash_bitwidth);
    qy = quant<double, A>(hy, g.hbox[2], g.hbox[3], g.hash_bitwidth);
    qz = quant<double, A>(hz, g.hbox[4], g.hbox[5], g.hash_bitwidth);
}

// is face (j, i) listed under hash cell (qx, qy, qz)?  (its quantised bounding box contains the cell)
__device__ __forceinline__ bool face_listed(const GridDev& g, int j, int i, unsigned int qx, unsigned int qy, unsigned int qz) {
    const unsigned long long b = ldg(g.hqbox + (long long)j * (g.nx - 1) + i);
    const unsigned int xl = b & 1023u, xh = (b >> 10) & 1023u, yl = (b >> 20) & 1023u, yh = (b >> 30) & 1023u,
                       zl = (b >> 40) & 1023u, zh = (b >> 50) & 1023u;
    return qx >= xl && qx <= xh && qy >= yl && qy <= yh && qz >= zl && qz <= zh;
}

template <class A, class D>
__device__ __forceinline__ void hash_query(const GridDev& g, CGridCtx<A, D>& e, const Query& q, bool finite, unsigned int qx,
                                           unsigned int qy, unsigned int qz, int& yi, int& xi, double& xsi, double& eta) {
    yi = -3; xi = -3; xsi = -1.0; eta = -1.0;  // GRID_SEARCH_ERROR, coords -1 (spatialhash.py:454-455,511)
    const unsigned int code = (dilate10(qz) << 2) | (dilate10(qy) << 1) | dilate10(qx);
    long long l = 0, h = g.hnkeys;  // np.searchsorted(keys, code) (side="left"), narrowed by the bucket table
    if (g.hbucket) {
        const unsigned int b = code >> g.hbucket_shift;
        l = ldg(g.hbucket + b);
        h = ldg(g.hbucket + b + 1);
    }
    while (l < h) {
        const long long m = (l + h) >> 1;
        if (ldg(g.hkeys + m) < code) l = m + 1; else h = m;
    }
    if (!(l < g.hnkeys && finite && ldg(g.hkeys + l) == code)) return;
    const long long start = ldg(g.hstarts + l), cnt = ldg(g.hcounts + l);
    const int ncol = g.nx - 1;
    for (long long k = 0; k < cnt; ++k) {  // first candidate (ascending face id) that contains the point wins
        const unsigned int face = ldg(g.hfaces + start + k);
        const int j = (int)(face / (unsigned)ncol), i = (int)(face % (unsigned)ncol);
        double cs, ce;
        if (point_in_cell(g, e, j, i, q, cs, ce)) {
            yi = j; xi = i;
            xsi = (double)(float)cs;  // coords_best is float32 (spatialhash.py:511,529)
            eta = (double)(float)ce;
            return;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// CGrid_Velocity arithmetic (typed like NumPy: A corner coords, C face values, TY/TX bcoords)
// ------------------------------------------------------------------------------------------------
// _geodetic_distance (utils/interpolation.py:178-185): result dtype promote(A, L) on spherical meshes,
// A on flat meshes
template <bool SPH, class A, class L>
__device__ __forceinline__ auto edge_length(A lat1, A lat2, A lon1, A lon2, L lat, double deg2m)
    -> typename std::conditional<SPH, decltype(A() * L()), A>::type {
    if constexpr (SPH) {
        using R = decltype(A() * L());
        const L rad_lat = (L)(3.14159265358979323846 / 180.0) * lat;
        const R t1 = ((lon2 - lon1) * (A)deg2m) * cosx(rad_lat);
        const A t2 = (lat2 - lat1) * (A)deg2m;
        return sqrt_np((R)(t1 * t1 + t2 * t2));
    } else {
        const A d1 = lon2 - lon1, d2 = lat2 - lat1;
        return sqrt_np((A)(d1 * d1 + d2 * d2));
    }
}

// `conv` = deg2m * cos_ool(deg2rad(y)) in the dtype of the sampled y (spherical meshes only)
template <bool SPH, class C, class A, class TZ, class TY, class TX, class CV, int NC>
__device__ __forceinline__ void cgrid_finish(const GridDev& g, const A (&px)[4], const A (&py)[4], C cu0, C cu1, C cv0, C cv1,
                                             C cw0, C cw1, TZ zeta, TY eta, TX xsi, CV conv, Val& u, Val& v, Val& w) {
    constexpr bool sph = SPH;
    const auto omx = 1 - xsi;
    const auto ome = 1 - eta;
    // latitude at the middle of each edge: einsum("ij,ji->i", phi2D_lin(., .), py), summed left to right
    const auto l1 = (omx * (TX)1.0) * py[0] + (xsi * (TX)1.0) * py[1] + (xsi * (TX)0.0) * py[2] + (omx * (TX)0.0) * py[3];
    const auto l2 = ((TY)0.0 * ome) * py[0] + ((TY)1.0 * ome) * py[1] + ((TY)1.0 * eta) * py[2] + ((TY)0.0 * eta) * py[3];
    const auto l3 = (omx * (TX)0.0) * py[0] + (xsi * (TX)0.0) * py[1] + (xsi * (TX)1.0) * py[2] + (omx * (TX)1.0) * py[3];
    const auto l4 = ((TY)1.0 * ome) * py[0] + ((TY)0.0 * ome) * py[1] + ((TY)0.0 * eta) * py[2] + ((TY)1.0 * eta) * py[3];
    const auto c1 = edge_length<SPH>(py[0], py[1], px[0], px[1], l1, g.deg2m);
    const auto c2 = edge_length<SPH>(py[1], py[2], px[1], px[2], l2, g.deg2m);
    const auto c3 = edge_length<SPH>(py[2], py[3], px[2], px[3], l3, g.deg2m);
    const auto c4 = edge_length<SPH>(py[3], py[0], px[3], px[0], l4, g.deg2m);
    const auto U0 = cu0 * c4;
    const auto U1 = cu1 * c2;
    const auto Uvel = omx * U0 + xsi * U1;
    const auto V0 = cv0 * c1;
    const auto V1 = cv1 * c3;
    const auto Vvel = ome * V0 + eta * V1;
    // _compute_jacobian_determinant (utils/interpolation.py:188-198)
    const auto dxdxsi = (eta - 1) * px[0] + ome * px[1] + eta * px[2] + (-eta) * px[3];
    const auto dxdeta = (xsi - 1) * px[0] + (-xsi) * px[1] + xsi * px[2] + omx * px[3];
    const auto dydxsi = (eta - 1) * py[0] + ome * py[1] + eta * py[2] + (-eta) * py[3];
    const auto dydeta = (xsi - 1) * py[0] + (-xsi) * py[1] + xsi * py[2] + omx * py[3];
    auto jac = dxdxsi * dydeta - dxdeta * dydxsi;
    if (sph) jac = jac * (decltype(jac))g.deg2m;
    auto uu = ((-ome) * Uvel - omx * Vvel) * px[0] + (ome * Uvel - xsi * Vvel) * px[1] + (eta * Uvel + xsi * Vvel) * px[2] +
              ((-eta) * Uvel + omx * Vvel) * px[3];
    auto vv = ((-ome) * Uvel - omx * Vvel) * py[0] + (ome * Uvel - xsi * Vvel) * py[1] + (eta * Uvel + xsi * Vvel) * py[2] +
              ((-eta) * Uvel + omx * Vvel) * py[3];
    auto ur = uu / jac;
    auto vr = vv / jac;
    if (sph) {  // u /= conversion; v /= conversion (in place: keeps u's dtype)
        ur = (decltype(ur))(ur / conv);
        vr = (decltype(vr))(vr / conv);
    }
    u = Val{(double)ur, std::is_same<decltype(ur), float>::value};
    v = Val{(double)vr, std::is_same<decltype(vr), float>::value};
    if (NC == 3) {
        const auto wr = cw0 * (1 - zeta) + cw1 * zeta;
        w = Val{(double)wr, std::is_same<decltype(wr), float>::value};
    } else {
        w = Val{0.0, u.f32};
    }
}

// ------------------------------------------------------------------------------------------------
// the policy
// ------------------------------------------------------------------------------------------------
// Rectilinear C-grid (1-D lon/lat): bcoords come from the typed 1-D axis search.
template <class A, class D, int NC_>
struct CGridPolicy {
    static constexpr int NC = NC_;
    static constexpr bool RUNTIME_DTYPE = false;
    static constexpr bool FAST_RK4 = false;
    static constexpr bool F32_STAGES = false;
    static constexpr bool BATCH_LEN_T = std::is_same<A, float>::value;
    static constexpr bool BATCH_LEN_Z = false;
    using Ctx = CGridCtx<A, D>;

    __device__ static __forceinline__ void init(Ctx& e, const AdvectParams& p, int ei) {
        e.cx.idx = e.cy.idx = e.cz.idx = e.ct.idx = -100;
        e.cx.lo = e.cx.hi = e.cy.lo = e.cy.hi = e.cz.lo = e.cz.hi = (A)0;
        e.ct.lo = e.ct.hi = 0.0;
        e.kyi = e.kxi = INT_MIN;
        e.uyi = e.uxi = INT_MIN;
        e.fti = e.fzi = e.fyi = e.fxi = INT_MIN;
        e.len_t = e.len_z = -1;
        e.ei = ei;
        // hint of the first search: unravel_index(ei) (basegrid.py:120-152,219-256), floor semantics
        const long long xd = p.g.xdim, yd = p.g.ydim;
        long long r = ei;
        if (p.g.nz > 0 && xd * yd > 0) { const long long pl = xd * yd; r = ((r % pl) + pl) % pl; }
        if (xd > 0) {
            long long yy = r / xd, xx = r % xd;
            if (xx < 0) { xx += xd; yy -= 1; }
            e.yi = (int)yy; e.xi = (int)xx;
        } else {
            e.yi = e.xi = -3;
        }
    }

    __device__ static __forceinline__ void finish(Ctx&, const AdvectParams&) {}

    template <class PZ, class PY, class PX>
    __device__ static __forceinline__ void eval(const AdvectParams& p, Ctx& e, bool no_hint, double t, PZ z, PY y, PX x, Val& u,
                                                Val& v, Val& w) {
        const GridDev& g = p.g;
        const FieldDev& f = p.f;
        using TZ = prom_t<PZ, A>;
        // -- time (index_search.py:65-91)
        double tau = 0.0;
        int ti = 0;
        if (g.nt > 0) {
            if (!(0 <= t && t <= g.time_len)) {
                e.state = PB_ERROR_OUTSIDE_TIME_INTERVAL;
                e.out_of_time = true;
                u = Val{0.0, false}; v = u; w = u;
                return;
            }
            tau = axis_search<double, double>(g.time, g.nt, t, e.ct);
            ti = e.ct.idx;
        }
        // -- depth
        TZ zeta = 0;
        int zi = 0;
        if (g.nz > 0) {
            zeta = axis_search<PZ, A>((const A*)g.depth, g.nz, z, e.cz);
            zi = e.cz.idx;
        }
        int yi, xi;
        A px[4], py[4];
        {
            using TY = prom_t<PY, A>;
            using TX = prom_t<PX, A>;
            const TY eta = axis_search<PY, A>((const A*)g.lat, g.ny, y, e.cy);
            const TX xsi = axis_search<PX, A>((const A*)g.lon, g.nx, x, e.cx);
            yi = e.cy.idx; xi = e.cx.idx;
            long long r = (long long)yi * g.xdim + (long long)xi;
            if (g.nz > 0) r += (long long)zi * (g.ydim * g.xdim);
            e.ei = (int)r;
            int s = e.state;
            if (xi == -1 || yi == -1 || zi == -1) s = max(s, (int)PB_ERROR_OUT_OF_BOUNDS);
            if (zi == -2) s = max(s, (int)PB_ERROR_THROUGH_SURFACE);
            // a horizontal index -2 (left of the axis) is not an error in the reference: it interpolates with the wrapped index
            // and masks the value afterwards -- but its NaN test comes first (field.py:288-290), and a non-finite barycentric
            // coordinate (a position that is -inf or NaN) makes that value NaN whatever the gathered faces are: ErrorInterpolation
            // (with valid indices the NaN test below finds it; this covers the early return)
            if (!isfinite((double)xsi) || !isfinite((double)eta) || (NC_ == 3 && !isfinite((double)zeta))) s = max(s, (int)PB_ERROR_INTERPOLATION);
            e.state = s;
            if (xi < 0 || yi < 0 || zi < 0) { u = Val{0.0, false}; v = u; w = u; return; }
            px[0] = e.cx.lo; px[1] = e.cx.hi; px[2] = e.cx.hi; px[3] = e.cx.lo;  // _xinterpolators.py:218-220
            py[0] = e.cy.lo; py[1] = e.cy.lo; py[2] = e.cy.hi; py[3] = e.cy.hi;
            finish<PZ, PY, TY, TX>(p, e, ti, tau, zi, zeta, yi, eta, xi, xsi, y, px, py, u, v, w);
        }
        if (u.v != u.v || v.v != v.v || w.v != w.v) e.state = max(e.state, (int)PB_ERROR_INTERPOLATION);
    }

    template <class PZ, class PY, class TY, class TX>
    __device__ static __forceinline__ void finish(const AdvectParams& p, Ctx& e, int ti, double tau, int zi, prom_t<PZ, A> zeta,
                                                  int yi, TY eta, int xi, TX xsi, PY y, A (&px)[4], A (&py)[4], Val& u, Val& v,
                                                  Val& w) {
        const GridDev& g = p.g;
        const FieldDev& f = p.f;
        using TZ = prom_t<PZ, A>;
        if (g.spherical) {  // corner longitudes unwrapped relative to corner 0 (_xinterpolators.py:230-233)
#pragma unroll
            for (int k = 0; k < 4; ++k) px[k] = mod_np((A)(px[k] + (A)180.0), (A)360.0) - (A)180.0;
#pragma unroll
            for (int k = 1; k < 4; ++k) if (px[k] - px[0] > (A)180) px[k] = px[k] - (A)360;
#pragma unroll
            for (int k = 1; k < 4; ++k) if (-px[k] + px[0] > (A)180) px[k] = px[k] + (A)360;
        }
        load_faces(g, f, e, ti, zi, yi, xi);
        if (g.spherical) reduce_and_finish<true, TZ, TY, TX, PY>(g, e, px, py, tau, zeta, eta, xsi, y, u, v, w);
        else reduce_and_finish<false, TZ, TY, TX, PY>(g, e, px, py, tau, zeta, eta, xsi, y, u, v, w);
    }

    // the 2 faces x 2 time levels of U, V (, W) this cell needs (_xinterpolators.py:246-330), re-gathered only
    // when the cell or the time level changed
    __device__ static __forceinline__ void load_faces(const GridDev& g, const FieldDev& f, Ctx& e, int ti, int zi, int yi, int xi) {
        if (e.fti != ti || e.fzi != zi || e.fyi != yi || e.fxi != xi) {
            e.fti = ti; e.fzi = zi; e.fyi = yi; e.fxi = xi;
            e.refills++;
            const long long ot[2] = {tslot(f, (long long)min(max(ti, 0), f.T - 1)) * f.sT, tslot(f, up_idx(ti, f.T)) * f.sT};
            const long long oz = (long long)min(max(zi, 0), f.Z - 1) * f.sZ;
            const long long oy0 = (long long)yi * f.sY, oy1 = up_idx(yi, f.Y) * f.sY;
            const long long oyo = (long long)min(max(yi + g.off_y, 0), f.Y - 1) * f.sY;
            const long long ox0 = (long long)xi * f.sX, ox1 = up_idx(xi, f.X) * f.sX;
            const long long oxo = (long long)min(max(xi + g.off_x, 0), f.X - 1) * f.sX;
            const D* __restrict__ U = (const D*)f.p[0];
            const D* __restrict__ V = (const D*)f.p[1];
#pragma unroll
            for (int tl = 0; tl < 2; ++tl) {
                e.fu[tl * 2 + 0] = ldg(U + ot[tl] + oz + oyo + ox0);
                e.fu[tl * 2 + 1] = ldg(U + ot[tl] + oz + oyo + ox1);
                e.fv[tl * 2 + 0] = ldg(V + ot[tl] + oz + oy0 + oxo);
                e.fv[tl * 2 + 1] = ldg(V + ot[tl] + oz + oy1 + oxo);
            }
            if (NC_ == 3) {
                const D* __restrict__ W = (const D*)f.p[2];
                const long long oz0 = (long long)min(max(zi + g.off_z, 0), f.Z - 1) * f.sZ;
                const long long oz1 = (long long)min(max(zi + g.off_z + 1, 0), f.Z - 1) * f.sZ;
#pragma unroll
                for (int tl = 0; tl < 2; ++tl) {
                    e.fw[tl * 2 + 0] = ldg(W + ot[tl] + oz0 + oyo + oxo);
                    e.fw[tl * 2 + 1] = ldg(W + ot[tl] + oz1 + oyo + oxo);
                }
            } else {
                e.fw[0] = e.fw[1] = e.fw[2] = e.fw[3] = (D)0;
            }
        }
    }

    template <bool SPH, class TZ, class TY, class TX, class PY>
    __device__ static __forceinline__ void reduce_and_finish(const GridDev& g, Ctx& e, const A (&px)[4], const A (&py)[4], double tau,
                                                             TZ zeta, TY eta, TX xsi, PY y, Val& u, Val& v, Val& w) {
        const PY conv = SPH ? (PY)g.deg2m * cosx(deg2rad_np(y)) : (PY)1;
        if (e.len_t < 0 ? (tau > 0) : (e.len_t != 0)) {  // lenT == 2: reduce over time in promote(D, float64)
            const double omt = 1 - tau;
            cgrid_finish<SPH, double, A, TZ, TY, TX, PY, NC_>(g, px, py, e.fu[0] * omt + e.fu[2] * tau, e.fu[1] * omt + e.fu[3] * tau,
                                                              e.fv[0] * omt + e.fv[2] * tau, e.fv[1] * omt + e.fv[3] * tau,
                                                              e.fw[0] * omt + e.fw[2] * tau, e.fw[1] * omt + e.fw[3] * tau, zeta,
                                                              eta, xsi, conv, u, v, w);
        } else {
            cgrid_finish<SPH, D, A, TZ, TY, TX, PY, NC_>(g, px, py, e.fu[0], e.fu[1], e.fv[0], e.fv[1], e.fw[0], e.fw[1], zeta, eta,
                                                         xsi, conv, u, v, w);
        }
    }
};


// ------------------------------------------------------------------------------------------------
// Curvilinear C-grid policy.  xsi/eta always come out of the closed-form bilinear inverse as float64
// (float32-rounded on a hash/neighbour hit), so the dtype of the sampled position only matters in three
// small places (depth bcoord, hash-grid quantisation, the spherical conversion factor): they branch at
// run time and the whole search + interpolation is instantiated ONCE per kernel.
// ------------------------------------------------------------------------------------------------
// VEL: 0 = CGrid_Velocity, 1 = XLinear_Velocity (an A-grid on 2-D lon / lat: the reference's XGrid.search feeds the same
// interpolators whatever the grid's shape, _core/xgrid.py:316-356 + interpolators/_xinterpolators.py:112-190)
template <class A, class D>
struct CurvACtx : CGridCtx<A, D> {
    D blk[3][16];  // VEL 1: the (t, z, y, x) corner block of U, V, W of the cached cell, [component][(t*2+z)*4 + y*2 + x]
};
template <class A, class D, int NC_, bool SPH, int VEL = 0>
struct CurvPolicy {
    static constexpr int NC = NC_;
    static constexpr bool RUNTIME_DTYPE = true;
    static constexpr bool FAST_RK4 = false;
    static constexpr bool F32_STAGES = false;
    static constexpr bool BATCH_LEN_T = std::is_same<A, float>::value;
    static constexpr bool BATCH_LEN_Z = false;
    using Ctx = typename std::conditional<VEL == 1, CurvACtx<A, D>, CGridCtx<A, D>>::type;

    __device__ static __forceinline__ void init(Ctx& e, const AdvectParams& p, int ei) { CGridPolicy<A, D, NC_>::init(e, p, ei); }
    __device__ static __forceinline__ void finish(Ctx&, const AdvectParams&) {}

    // XLinear_Velocity behind the curvilinear search: T-lerp, Z-lerp, bilinear in NumPy's dtypes (xsi, eta are float64 -- the
    // closed-form inverse's -- so the value is float64; a float32 block meets a float32 zeta in float32 first)
    __device__ static __forceinline__ void xlinear_rt(const FieldDev& f, Ctx& e, int ti, double tau, int zi, double zeta, bool zeta_f32,
                                                      int yi, double eta, int xi, double xsi, bool two_t, bool two_z, double (&q)[3]) {
        if constexpr (VEL == 1) {
            if (e.fti != ti || e.fzi != zi || e.fyi != yi || e.fxi != xi) {
                e.fti = ti; e.fzi = zi; e.fyi = yi; e.fxi = xi;
                e.refills++;
                const long long ot[2] = {tslot(f, wrap_idx(ti, f.T)) * f.sT, tslot(f, up_idx(ti, f.T)) * f.sT};
                const long long oz[2] = {wrap_idx(zi, f.Z) * f.sZ, up_idx(zi, f.Z) * f.sZ};
                const long long oy[2] = {wrap_idx(yi, f.Y) * f.sY, up_idx(yi, f.Y) * f.sY};
                const long long ox[2] = {wrap_idx(xi, f.X) * f.sX, up_idx(xi, f.X) * f.sX};
#pragma unroll
                for (int c = 0; c < NC_; ++c) {
                    const D* __restrict__ base = (const D*)f.p[c];
#pragma unroll
                    for (int k = 0; k < 16; ++k) e.blk[c][k] = ldg(base + ot[k >> 3] + oz[(k >> 2) & 1] + oy[(k >> 1) & 1] + ox[k & 1]);
                }
            }
            const double omt = 1 - tau;
            const double w00 = (1 - xsi) * (1 - eta), w01 = xsi * (1 - eta), w10 = (1 - xsi) * eta, w11 = xsi * eta;
#pragma unroll
            for (int c = 0; c < NC_; ++c) {
                double r[4];
                if (!two_t && std::is_same<D, float>::value && zeta_f32) {  // float32 block, float32 zeta: the Z-lerp is float32
                    const float zf = (float)zeta, omzf = 1 - zf;
#pragma unroll
                    for (int k = 0; k < 4; ++k) r[k] = two_z ? (double)((float)e.blk[c][k] * omzf + (float)e.blk[c][4 + k] * zf) : (double)e.blk[c][k];
                } else {
                    const double omz = zeta_f32 ? (double)(1 - (float)zeta) : 1 - zeta;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const double a = two_t ? e.blk[c][k] * omt + e.blk[c][8 + k] * tau : (double)e.blk[c][k];
                        const double b = two_t ? e.blk[c][4 + k] * omt + e.blk[c][12 + k] * tau : (double)e.blk[c][4 + k];
                        r[k] = two_z ? a * omz + b * zeta : a;
                    }
                }
                q[c] = w00 * r[0] + w01 * r[1] + w10 * r[2] + w11 * r[3];
            }
        }
    }

    __device__ static __forceinline__ void eval_rt(const AdvectParams& p, Ctx& e, bool no_hint, double t, double z, double y, double x,
                                                   bool xy_f32, bool z_f32, Val& u, Val& v, Val& w) {
        const GridDev& g = p.g;
        const FieldDev& f = p.f;
        u = Val{0.0, false}; v = u; w = u;
        // -- time (index_search.py:65-91)
        double tau = 0.0;
        int ti = 0;
        if (g.nt > 0) {
            if (!(0 <= t && t <= g.time_len)) {
                e.state = PB_ERROR_OUTSIDE_TIME_INTERVAL;
                e.out_of_time = true;
                return;
            }
            tau = axis_search<double, double>(g.time, g.nt, t, e.ct);
            ti = e.ct.idx;
        }
        // -- depth: bcoord dtype = promote(position dtype, A)
        double zeta = 0.0;
        bool zeta_f32 = false;
        int zi = 0;
        if (g.nz > 0) {
            if (z_f32 && std::is_same<A, float>::value) {
                zeta = (double)axis_search<float, A>((const A*)g.depth, g.nz, (float)z, e.cz);
                zeta_f32 = true;
            } else if (z_f32) {
                zeta = (double)axis_search<float, A>((const A*)g.depth, g.nz, (float)z, e.cz);  // float z, float64 axis -> float64
            } else {
                zeta = (double)axis_search<double, A>((const A*)g.depth, g.nz, z, e.cz);
            }
            zi = e.cz.idx;
        }
        // -- _search_indices_curvilinear_2d (index_search.py:242-295): hint, (neighbours,) spatial hash
        Query q;
        q.x = x; q.y = y;
        q.qu_x = q.qu_y = q.qu_z = 0.0;
        double cos_lat = 1.0;  // cos(deg2rad(y)) in float64: also the spherical conversion factor of a float64 position
        if (SPH) {
            const double la = deg2rad_np(y), lo = deg2rad_np(x);
            const double cl = cos_np(la);
            cos_lat = cl;
            double sl, cl2;
            sincos_lon(lo, sl, cl2);
            q.qu_x = cl2 * cl; q.qu_y = sl * cl; q.qu_z = sin_lat(la);
        }
        double xsi = -1.0, eta = -1.0;
        int yi, xi;
        // `if np.any(xi)` (index_search.py:269): a batch whose hinted xi are ALL zero skips the hint test.  The host knows that for
        // the first evaluation of a call (no_hint); a set of ONE particle knows it by itself at every evaluation.
        const bool lone_zero = p.lone_particle && e.xi == 0;
        const bool hint_ok = !no_hint && !lone_zero && e.yi >= 0 && e.xi >= 0 && e.yi < g.ny - 1 && e.xi < g.nx - 1;
        bool found = false;
        if (hint_ok) found = point_in_cell(g, e, e.yi, e.xi, q, xsi, eta);
        if (found) {
            yi = e.yi; xi = e.xi;
        } else {
            // The reference goes straight to the spatial hash.  Most misses are a move into an adjacent cell:
            // test the 8 neighbours first and accept a hit only when (a) the point is SAFELY interior -- then
            // that cell is the only one containing it -- and (b) the hash table lists that face under the
            // point's hash cell (a face whose corner bounding box misses the point is invisible to the
            // reference's query).  Then the hash's "first containing candidate" is this very cell with these
            // very coordinates, float32-rounded like spatialhash.py:511.  Anything else -- edge-grazing
            // points, jumps, no valid hint -- takes the exact hash path.
            unsigned int qx, qy, qz;
            if (xy_f32) hash_coords<A, float, float>(g, (float)y, (float)x, qx, qy, qz);
            else if (SPH) hash_coords_xyz<A>(g, q.qu_x, q.qu_y, q.qu_z, qx, qy, qz);  // no second set of sin/cos
            else hash_coords<A, double, double>(g, y, x, qx, qy, qz);
            bool nb = false;
            if (hint_ok && isfinite(x) && isfinite(y)) {
                const int hj = e.yi, hi = e.xi;
                // the failed hint test says which way the point left the hinted cell: that neighbour is tested first
                // (k = -1), the other seven only if it is not the one (non-overlapping cells: at most one can pass)
                const int gdj = eta > 1 ? 1 : (eta < 0 ? -1 : 0);
                const int gdi = xsi > 1 ? 1 : (xsi < 0 ? -1 : 0);
#pragma unroll 1
                for (int k = -1; k < 8 && !nb; ++k) {
                    int dj, di;
                    if (k < 0) {
                        dj = gdj; di = gdi;
                        if ((dj | di) == 0) continue;
                    } else {
                        dj = (k < 3) ? -1 : ((k < 5) ? 0 : 1);
                        di = (k == 0 || k == 3 || k == 5) ? -1 : ((k == 1 || k == 6) ? 0 : 1);
                        if (dj == gdj && di == gdi) continue;
                    }
                    const int j = hj + dj, i = hi + di;
                    if (j < 0 || i < 0 || j >= g.ny - 1 || i >= g.nx - 1) continue;
                    double cs, ce;
                    if (point_in_cell(g, e, j, i, q, cs, ce) && cs > 1e-6 && cs < 1 - 1e-6 && ce > 1e-6 && ce < 1 - 1e-6 &&
                        face_listed(g, j, i, qx, qy, qz)) {
                        nb = true;
                        yi = j; xi = i;
                        xsi = (double)(float)cs;
                        eta = (double)(float)ce;
                    }
                }
            }
            if (!nb) {
                // (inline on purpose: out of line -- 0.03 queries per warp-step, ~350 instructions -- the call spills the caller's live
                //  registers)
                hash_query(g, e, q, xy_f32 ? isfinite((float)x) && isfinite((float)y) : isfinite(x) && isfinite(y), qx, qy, qz, yi, xi, xsi, eta);
            }
        }
        e.yi = yi; e.xi = xi;
        long long r = (long long)yi * g.xdim + (long long)xi;
        if (g.nz > 0) r += (long long)zi * (g.ydim * g.xdim);
        e.ei = (int)r;
        int s = e.state;
        if (zi == -1) s = max(s, (int)PB_ERROR_OUT_OF_BOUNDS);
        if (xi == -3 || yi == -3) s = max(s, (int)PB_ERROR_GRID_SEARCHING);
        if (zi == -2) s = max(s, (int)PB_ERROR_THROUGH_SURFACE);
        e.state = s;
        if (xi < 0 || yi < 0 || zi < 0) return;

        if constexpr (VEL == 1) {  // -- XLinear_Velocity (_xinterpolators.py:112-190) on the searched cell
            const bool two_t = g.nt > 0 && (e.len_t < 0 ? (tau > 0) : (e.len_t != 0));
            const bool two_z = g.nz > 0 && (e.len_z < 0 ? !(zeta <= 0) : (e.len_z != 0));
            double q[3] = {0.0, 0.0, 0.0};
            xlinear_rt(f, e, ti, tau, zi, zeta, zeta_f32, yi, eta, xi, xsi, two_t, two_z, q);
            if (SPH) {  // u /= deg2m * cos(deg2rad(y)) in the dtype of the sampled y; v /= deg2m  (:182-184)
                const double conv = xy_f32 ? (double)((float)g.deg2m * cosf_ool(deg2rad_np((float)y))) : g.deg2m * cos_lat;
                q[0] = q[0] / conv;
                q[1] = q[1] / g.deg2m;
            }
            u = Val{q[0], false}; v = Val{q[1], false}; w = Val{NC_ == 3 ? q[2] : 0.0, false};
            if (u.v != u.v || v.v != v.v || w.v != w.v) e.state = max(e.state, (int)PB_ERROR_INTERPOLATION);
            return;
        }
        // -- CGrid_Velocity (_xinterpolators.py:193-332)
        load_corners(g, e, yi, xi);
        const bool two_t = e.len_t < 0 ? (tau > 0) : (e.len_t != 0);  // lenT: the batch's decision when known
        A px[4], py[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) py[k] = e.clat[k];
        if (SPH) {  // corner longitudes unwrapped relative to corner 0 (:230-233): a property of the cell, redone on a cell change only
            if (e.uyi != yi || e.uxi != xi) {
                e.uyi = yi; e.uxi = xi;
#pragma unroll
                for (int k = 0; k < 4; ++k) e.ulon[k] = mod_np((A)(e.clon[k] + (A)180.0), (A)360.0) - (A)180.0;
#pragma unroll
                for (int k = 1; k < 4; ++k) if (e.ulon[k] - e.ulon[0] > (A)180) e.ulon[k] = e.ulon[k] - (A)360;
#pragma unroll
                for (int k = 1; k < 4; ++k) if (-e.ulon[k] + e.ulon[0] > (A)180) e.ulon[k] = e.ulon[k] + (A)360;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) px[k] = e.ulon[k];
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) px[k] = e.clon[k];
        }
        CGridPolicy<A, D, NC_>::load_faces(g, f, e, ti, zi, yi, xi);
        // spherical conversion factor in the dtype of the sampled y
        double conv = 1.0;
        if (SPH) conv = xy_f32 ? (double)((float)g.deg2m * cosf_ool(deg2rad_np((float)y))) : g.deg2m * cos_lat;
        Val wdummy;
        if constexpr (SPH || std::is_same<A, double>::value) {
            // every operand the face values meet is float64 (edge lengths are float64: float64 bcoords on a
            // spherical mesh / float64 corner coordinates), so they convert exactly: ONE float64 code path
            double c[6];
            if (two_t) {
                const double omt = 1 - tau;
                c[0] = e.fu[0] * omt + e.fu[2] * tau; c[1] = e.fu[1] * omt + e.fu[3] * tau;
                c[2] = e.fv[0] * omt + e.fv[2] * tau; c[3] = e.fv[1] * omt + e.fv[3] * tau;
            } else {
                c[0] = (double)e.fu[0]; c[1] = (double)e.fu[1]; c[2] = (double)e.fv[0]; c[3] = (double)e.fv[1];
            }
            cgrid_finish<SPH, double, A, double, double, double, double, 2>(g, px, py, c[0], c[1], c[2], c[3], 0.0, 0.0, 0.0, eta, xsi,
                                                                            conv, u, v, wdummy);
        } else {  // flat mesh with float32 corner coordinates: edge lengths are float32, the face dtype matters
            if (two_t) {
                const double omt = 1 - tau;
                cgrid_finish<SPH, double, A, double, double, double, double, 2>(g, px, py, e.fu[0] * omt + e.fu[2] * tau,
                                                                                e.fu[1] * omt + e.fu[3] * tau, e.fv[0] * omt + e.fv[2] * tau,
                                                                                e.fv[1] * omt + e.fv[3] * tau, 0.0, 0.0, 0.0, eta, xsi, conv, u,
                                                                                v, wdummy);
            } else {
                cgrid_finish<SPH, D, A, double, double, double, double, 2>(g, px, py, e.fu[0], e.fu[1], e.fv[0], e.fv[1], (D)0, (D)0, 0.0, eta,
                                                                           xsi, conv, u, v, wdummy);
            }
        }
        if (NC_ == 3) {  // W: linear in zeta between the two Z faces (:316-330); dtype as NumPy would promote
            const bool tl = two_t;
            if (!tl && std::is_same<D, float>::value && zeta_f32) {
                const float zf = (float)zeta;
                const float wr = (float)e.fw[0] * (1 - zf) + (float)e.fw[1] * zf;
                w = Val{(double)wr, true};
            } else {
                const double omt = 1 - tau;
                const double w0 = tl ? e.fw[0] * omt + e.fw[2] * tau : (double)e.fw[0];
                const double w1 = tl ? e.fw[1] * omt + e.fw[3] * tau : (double)e.fw[1];
                const double omz = zeta_f32 ? (double)(1 - (float)zeta) : 1 - zeta;
                w = Val{w0 * omz + w1 * zeta, false};
            }
        } else {
            w = Val{0.0, u.f32};
        }
        if (u.v != u.v || v.v != v.v || w.v != w.v) e.state = max(e.state, (int)PB_ERROR_INTERPOLATION);
    }
};

// ------------------------------------------------------------------------------------------------
// Scalar Field.eval on CURVILINEAR grids (reference _core/field.py:144-202): CGrid_Tracer (_xinterpolators.py:335-383, the
// tracer point of the cell the curvilinear search finds -- NEMO temperature / salinity on an ORCA grid) and XNearest
// (:515-560).  Neither does arithmetic on the barycentric coordinates, so the float32-typed coordinates of the reference's
// hash path (DESIGN.md waiver 4) cannot show: values, cells and states are the reference's exactly.
// The search below is CurvPolicy::eval_rt's (time, depth, hint -> neighbours -> spatial hash), restated for one sample so
// that the advection kernel's code stays exactly what the profiles measured.
// ------------------------------------------------------------------------------------------------
template <class A, class D, bool SPH>
__global__ void sample_scalar_curv_kernel(const SampleParams s, int mode /* 3: XLinear, 4: XNearest, 5: CGrid_Tracer */, int has_time) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n) return;
    const GridDev& g = s.g;
    const FieldDev& f = s.f;
    AdvectParams p{};
    p.g = g;
    CGridCtx<A, D> e;
    CGridPolicy<A, D, 2>::init(e, p, s.ei_hint ? s.ei_hint[i] : 0);
    e.uyi = e.uxi = INT_MIN;
    int state = PB_EVALUATE;
    const bool f32 = s.pos_f32 != 0;
    const double t = s.t[i];
    const double z = f32 ? (double)(float)s.z[i] : s.z[i], y = f32 ? (double)(float)s.y[i] : s.y[i], x = f32 ? (double)(float)s.x[i] : s.x[i];
    double value = 0.0;
    bool value_f32 = std::is_same<D, float>::value;
    int ei = e.ei;
    do {
        // -- time (index_search.py:65-91); a field without a time dimension is not searched (field.py:112-117)
        double tau = 0.0;
        int ti = 0;
        if (has_time) {
            if (!(0 <= t && t <= g.time_len)) { state = PB_ERROR_OUTSIDE_TIME_INTERVAL; break; }
            tau = axis_search<double, double>(g.time, g.nt, t, e.ct);
            ti = e.ct.idx;
        }
        // -- depth
        double zeta = 0.0;
        int zi = 0;
        if (g.nz > 0) {
            zeta = f32 ? (double)axis_search<float, A>((const A*)g.depth, g.nz, (float)z, e.cz) : (double)axis_search<double, A>((const A*)g.depth, g.nz, z, e.cz);
            zi = e.cz.idx;
        }
        // -- _search_indices_curvilinear_2d (index_search.py:242-295)
        Query q;
        q.x = x; q.y = y;
        if (SPH) {
            const double la = deg2rad_np(y), lo = deg2rad_np(x);
            const double cl = cos_np(la);
            double sl, cl2;
            sincos_lon(lo, sl, cl2);
            q.qu_x = cl2 * cl; q.qu_y = sl * cl; q.qu_z = sin_lat(la);
        }
        double xsi = -1.0, eta = -1.0;
        int yi, xi;
        const bool no_hint = s.no_hint || !s.ei_hint;
        const bool hint_ok = !no_hint && e.yi >= 0 && e.xi >= 0 && e.yi < g.ny - 1 && e.xi < g.nx - 1;
        bool found = false;
        if (hint_ok) found = point_in_cell(g, e, e.yi, e.xi, q, xsi, eta);
        if (found) {
            yi = e.yi; xi = e.xi;
        } else {
            unsigned int qx, qy, qz;
            if (f32) hash_coords<A, float, float>(g, (float)y, (float)x, qx, qy, qz);
            else hash_coords<A, double, double>(g, y, x, qx, qy, qz);
            hash_query(g, e, q, f32 ? isfinite((float)x) && isfinite((float)y) : isfinite(x) && isfinite(y), qx, qy, qz, yi, xi, xsi, eta);
        }
        long long r = (long long)yi * g.xdim + (long long)xi;
        if (g.nz > 0) r += (long long)zi * (g.ydim * g.xdim);
        ei = (int)r;
        if (zi == -1) state = max(state, (int)PB_ERROR_OUT_OF_BOUNDS);
        if (xi == -3 || yi == -3) state = max(state, (int)PB_ERROR_GRID_SEARCHING);
        if (zi == -2) state = max(state, (int)PB_ERROR_THROUGH_SURFACE);
        if (xi < 0 || yi < 0 || zi < 0) break;  // masked to 0 (field.py:189)
        if (mode == 3) {
            // -- XLinear (_xinterpolators.py:112-153) on the searched cell: T-lerp, Z-lerp, bilinear in NumPy's dtypes.  xsi / eta are
            // the closed-form inverse's float64 values (float32-ROUNDED after a hash hit: DESIGN.md waiver 4), so the value is float64.
            const int bf = s.batch_flags ? *s.batch_flags : -1;
            const bool two_t = has_time && (bf >= 0 ? (bf & 1) != 0 : (tau > 0));
            const bool two_z = g.nz > 0 && (bf >= 0 ? (bf & 2) != 0 : !(zeta <= 0));
            const bool zeta_f32 = f32 && std::is_same<A, float>::value;
            const long long ot[2] = {wrap_idx(ti, f.T) * f.sT, up_idx(ti, f.T) * f.sT};
            const long long oz[2] = {wrap_idx(zi, f.Z) * f.sZ, up_idx(zi, f.Z) * f.sZ};
            const long long oy[2] = {wrap_idx(yi, f.Y) * f.sY, up_idx(yi, f.Y) * f.sY};
            const long long ox[2] = {wrap_idx(xi, f.X) * f.sX, up_idx(xi, f.X) * f.sX};
            const D* __restrict__ P = (const D*)f.p[0];
            const double omt = 1 - tau;
            double rr[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const long long o = oy[k >> 1] + ox[k & 1];
                const D a0 = ldg(P + ot[0] + oz[0] + o), a1 = ldg(P + ot[0] + oz[1] + o);
                if (!two_t && std::is_same<D, float>::value && zeta_f32) {  // float32 data, float32 zeta: the Z-lerp is float32
                    const float zf = (float)zeta;
                    rr[k] = two_z ? (double)((float)a0 * (1 - zf) + (float)a1 * zf) : (double)a0;
                } else {
                    double lo = (double)a0, hi = (double)a1;
                    if (two_t) {
                        lo = lo * omt + (double)ldg(P + ot[1] + oz[0] + o) * tau;
                        hi = hi * omt + (double)ldg(P + ot[1] + oz[1] + o) * tau;
                    }
                    const double omz = zeta_f32 ? (double)(1 - (float)zeta) : 1 - zeta;
                    rr[k] = two_z ? lo * omz + hi * zeta : lo;
                }
            }
            value = (1 - xsi) * (1 - eta) * rr[0] + xsi * (1 - eta) * rr[1] + (1 - xsi) * eta * rr[2] + xsi * eta * rr[3];
            value_f32 = false;
            if (value != value) state = max(state, (int)PB_ERROR_INTERPOLATION);
            break;
        }
        // -- the node: CGrid_Tracer = index + SGRID offset, XNearest = the near side of each axis; both clipped like the gathers
        int kz, ky, kx;
        if (mode == 5) {
            kz = zi + g.off_z; ky = yi + g.off_y; kx = xi + g.off_x;
        } else {
            kz = zeta <= 0.5 ? zi : zi + 1; ky = eta <= 0.5 ? yi : yi + 1; kx = xsi <= 0.5 ? xi : xi + 1;
        }
        const long long oz = (long long)min(max(kz, 0), f.Z - 1) * f.sZ, oy = (long long)min(max(ky, 0), f.Y - 1) * f.sY,
                        ox = (long long)min(max(kx, 0), f.X - 1) * f.sX;
        const D* __restrict__ P = (const D*)f.p[0];
        const D c0 = ldg(P + (long long)min(max(ti, 0), f.T - 1) * f.sT + oz + oy + ox);
        if (s.batch_flags ? ((*s.batch_flags & 1) != 0) : (tau > 0)) {  // lenT == 2 (the batch's decision, from the pre-pass): linear in time in promote(D, float64)
            const D c1 = ldg(P + up_idx(ti, f.T) * f.sT + oz + oy + ox);
            value = (double)c0 * (1 - tau) + (double)c1 * tau;
            value_f32 = false;
        } else {
            value = (double)c0;
        }
        if (value != value) state = max(state, (int)PB_ERROR_INTERPOLATION);
    } while (false);
    s.u[i] = value;
    if (s.f32_out) s.f32_out[i] = value_f32 ? 1 : 0;
    s.ei_out[i] = ei;
    s.state_out[i] = state;
}

