// afast.cu -- the headline hot path: AdvectionRK4 / AdvectionRK4_3D with XLinear_Velocity (reference kernels/_advection.py:42-75,
// interpolators/_xinterpolators.py:78-190, _core/field.py:250-405) on a rectilinear A-grid with FLOAT64 coordinates, FLOAT32
// data and a time axis, every level resident (BASELINE configs 2, 4, 5 and the north-star workload).  Same arithmetic, operation
// by operation, as the generic AGridPolicy<double, float, true, NC, 0> of agrid.cuh (which stays the kernel of every other
// dtype / scheme / interpolator combination and is the cross-check of this one: tests/test_gpu_fast_kernel.py, bit for bit);
// what differs is the schedule:
//
//  * The common case -- the sample is still inside the cached cell of every axis -- is straight-line code: three bcoord divisions
//    through cached reciprocals, the cos of the latitude (one polynomial), Z-lerp, bilinear, unit conversion.  Everything else (a
//    cell change, a sentinel index, a sample on the first node of an axis, outside the time axis) is a rare side path.
//  * Everything a lane caches lives in SHARED MEMORY as 16-byte columns ([chunk][lane]: LDS.128 / STS.128, conflict-free): the raw
//    2x2x2x2 block (float32), the T-LERPED block (float64: the sample time of stage 3 equals stage 2's and stage 1's equals the
//    previous step's stage 4, so the 24 time lerps are done twice per step instead of four times), the cells {lo, hi} of z, y,
//    x, t, the reciprocals of their widths and the cell indices = 560 B per lane, 384 lanes per SM.  The raw block holds the corner
//    NODE RECORDS {u, v, w, 0} as the refill loads them (transposing them into per-component chunks was 48 register moves per cell
//    change); the T-lerp reads two corners' records at a time and feeds the Z-lerp / bilinear sum directly.  The cells are re-read at
//    every evaluation (volatile loads): they only change in the side path, and keeping them in registers costs moves and spills.
//  * A refill reads the NODE-INTERLEAVED copy of U, V, W ({u, v, w, 0} per node, built on the device at upload,
//    interleave_kernel below): 16 x 16-byte loads instead of 48 scattered 4-byte ones, a fifth of the DRAM traffic.
//  * On a cell miss the two neighbouring cells are tried before the full binary search (a particle crosses one face at a time).
//
// TWO SCHEDULES of the same evaluation (template parameter SCHED; the instruction cache decides):
//   SCHED 2 (advection-only lists): a TWO-stage loop body -- a stage that reuses the T-lerped block and one that renews it, the
//     choice a compile-time constant, run twice per step, both side-path copies inline.
//   SCHED 1 (lists with DiffusionUniformKh): ONE evaluation site in a four-trip stage loop, "renew" a run-time flag
//     -- next to the Philox / Box-Muller block only one copy of the hit and side paths fits the cache.
//   Tried and measured slower: all four stages written out (5000 SASS instructions: instruction-fetch stalls), the
//   side path or the diffusion increment out of line (every call spills the hit path's live registers).
#include <cmath>

#include "agrid.cuh"

#ifndef PB_FAST_BLOCK
#define PB_FAST_BLOCK PB_BLOCK
#endif

// ------------------------------------------------------------------------------------------------
// node-interleaved field copy
// ------------------------------------------------------------------------------------------------
__global__ void interleave_kernel(const float* __restrict__ u, const float* __restrict__ v, const float* __restrict__ w, long long n,
                                  float4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 r;
    r.x = u[i];
    r.y = v[i];
    r.z = w ? w[i] : 0.f;
    r.w = 0.f;
    out[i] = r;
}

cudaError_t launch_interleave(const float* u, const float* v, const float* w, long long nodes, void* out, cudaStream_t s) {
    if (nodes <= 0) return cudaSuccess;
    interleave_kernel<<<(unsigned)((nodes + 255) / 256), 256, 0, s>>>(u, v, w, nodes, (float4*)out);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// axis search of the side path: the cell only (no bcoord division), neighbours of the cached cell first.
// Same cell / sentinel as axis_search (common.cuh; reference _core/index_search.py:20-62).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void axis_locate(const double* __restrict__ arr, int n, double x, AxisCell<double>& c) {
    if (n < 2) {  // index_search.py:45-46
        c.idx = 0;
        return;
    }
    if (c.idx >= 0) {
        // lo < x <= hi of a cell inside the axis is exactly searchsorted(side="left") - 1 == that cell
        if (x > c.lo && x <= c.hi) return;
        if (x > c.hi && c.idx + 2 <= n - 1) {
            const double nh = ldg(arr + c.idx + 2);
            if (x <= nh) { c.lo = c.hi; c.hi = nh; c.idx += 1; return; }
        } else if (x <= c.lo && c.idx >= 1) {
            const double nl = ldg(arr + c.idx - 1);
            if (x > nl) { c.hi = c.lo; c.lo = nl; c.idx -= 1; return; }
        }
    }
    int l = 0, h = n;  // first i with arr[i] >= x   (side="left")
    while (l < h) {
        const int m = (l + h) >> 1;
        if (ldg(arr + m) < x) l = m + 1; else h = m;
    }
    if (x != x) l = n;  // NaN sorts last
    const int i = min(max(l - 1, 0), n - 2);
    c.lo = ldg(arr + i);
    c.hi = ldg(arr + i + 1);
    c.idx = i;
    if (x < ldg(arr)) c.idx = -2;          // LEFT_OUT_OF_BOUNDS
    if (x > ldg(arr + n - 1)) c.idx = -1;  // RIGHT_OUT_OF_BOUNDS
}
// bcoord of x in the located cell (also of a clipped one: sentinels keep the cell of the nearest edge)
__device__ __forceinline__ double axis_bcoord(int n, double x, const AxisCell<double>& c) {
    return n < 2 ? 0.0 : (x - c.lo) / (c.hi - c.lo);
}

// The general evaluation of ONE component from a lane's raw block (special samples only: a sentinel index, a sample on the first
// node of the time / depth axis -- lenT or lenZ == 1 for this particle): agrid.cuh's xlinear, the all-float64 path.  Out of line:
// it is rare, and keeping its 16-value block out of the hot kernel's register allocation matters more than a call.
template <int NV>
__device__ __noinline__ double special_component(const float4* raw, int comp, double tau, double zeta, double eta, double xsi, int two_t,
                                                 int two_z) {
    float blk[16];
#pragma unroll
    for (int k = 0; k < NV; ++k) {  // record k = (t * 2 + z) * 4 + y * 2 + x (NV 16) | t * 4 + y * 2 + x (NV 8)
        const float4 r = raw[k * PB_FAST_BLOCK];
        blk[k] = comp == 0 ? r.x : (comp == 1 ? r.y : r.z);
    }
    if (NV == 8) {  // (t, y, x) -> the generic (t, z, y, x) order with the one depth level twice
#pragma unroll
        for (int j = 3; j >= 0; --j) { blk[8 + j] = blk[4 + j]; blk[12 + j] = blk[4 + j]; }
#pragma unroll
        for (int j = 3; j >= 0; --j) blk[4 + j] = blk[j];
    }
    return xlinear<float, double, double, double, double>(blk, tau, zeta, eta, xsi, two_t != 0, two_z != 0).v;
}

// a 16-byte shared-memory load the compiler must issue where it is written (no hoisting, no store-to-load forwarding)
__device__ __forceinline__ double2 lds_volatile(const double2* p) {
#ifdef PB_HOSTSIM
    return *p;
#else
    double2 r;
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "r"(a));
    return r;
#endif
}


struct SideResult {
    double u, v, w;
    int state;
    int flags;  // SIDE_*
};
enum { SIDE_FINAL = 1, SIDE_OUT_OF_TIME = 2, SIDE_REFILLED = 4, SIDE_SEARCHED = 8 };

struct FastCtx {
    double lerp_t;  // sample time the T-lerped block in shared memory belongs to (-1: none)
    float4* raw;    // this lane's column of 16-byte chunks
    int state;
    int ei;
    unsigned int refills;
    bool searched;
    bool out_of_time;
    signed char len_t, len_z;  // (interface of the generic kernel skeleton; unused here)
};

// NC: components sampled (2: fieldset.UV, 3: fieldset.UVW).  HZ: the grid has a depth axis with >= 2 levels.  SCHED: see the head
// of this file (2: two-stage loop body, 1: one evaluation site in a four-trip loop).
template <int NC_, bool HZ, int SCHED>
struct AFastPolicy {
    static constexpr int NC = NC_;
    static constexpr int NV = HZ ? 16 : 8;          // raw values per component: (t, [z,] y, x) corners
    static constexpr int NL = NV / 2;               // T-lerped values per component
    static constexpr int RAW_CHUNKS = NV;           // float4 columns: the corner NODE RECORDS {u, v, w, 0} as loaded (no transposition)
    static constexpr int LRP_CHUNKS = NC * NL / 2;  // double2 columns
    static constexpr int CELL_CHUNKS = 4;           // double2 columns {lo, hi}: z, y, x, t
    static constexpr int RCP_CHUNKS = 2;            // {1 / dz, 1 / dy}, {1 / dx, 1 / dt} of the current cells
    static constexpr int IDX_CHUNKS = 1;            // int4 {ti, zi, yi, xi} of the last search (-100: none)
    static constexpr size_t SMEM = (size_t)(RAW_CHUNKS + LRP_CHUNKS + CELL_CHUNKS + RCP_CHUNKS + IDX_CHUNKS) * 16 * PB_FAST_BLOCK;
    static constexpr bool RUNTIME_DTYPE = false;
    static constexpr bool FAST_RK4 = true;
    static constexpr bool FAST_UNROLLED = SCHED == 2;
    static constexpr bool F32_STAGES = false;
    static constexpr bool BATCH_LEN_T = false;
    static constexpr bool BATCH_LEN_Z = false;
    using Ctx = FastCtx;

    __device__ static __forceinline__ double2* lrp(float4* raw) { return reinterpret_cast<double2*>(raw + (size_t)RAW_CHUNKS * PB_FAST_BLOCK); }
    __device__ static __forceinline__ double2* cell(float4* raw, int k) {  // 0: z, 1: y, 2: x, 3: t
        return reinterpret_cast<double2*>(raw + (size_t)(RAW_CHUNKS + LRP_CHUNKS + k) * PB_FAST_BLOCK);
    }
    __device__ static __forceinline__ double2* rcp(float4* raw) {
        return reinterpret_cast<double2*>(raw + (size_t)(RAW_CHUNKS + LRP_CHUNKS + CELL_CHUNKS) * PB_FAST_BLOCK);
    }
    __device__ static __forceinline__ int4* idx(float4* raw) {
        return reinterpret_cast<int4*>(raw + (size_t)(RAW_CHUNKS + LRP_CHUNKS + CELL_CHUNKS + RCP_CHUNKS) * PB_FAST_BLOCK);
    }

    __device__ static __forceinline__ void init(Ctx& e, const AdvectParams&, int ei) {
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        extern __shared__ __align__(16) unsigned char pb_smem[];
        e.raw = reinterpret_cast<float4*>(pb_smem) + threadIdx.x;
        double2 d;
        d.x = nan; d.y = nan;
#pragma unroll
        for (int k = 0; k < CELL_CHUNKS; ++k) *cell(e.raw, k) = d;
        int4 none;
        none.x = none.y = none.z = none.w = -100;
        *idx(e.raw) = none;
        e.lerp_t = -1.0;  // valid sample times are >= 0
        e.ei = ei;
        e.searched = false;
        e.len_t = e.len_z = -1;
    }
    // ravel_index (basegrid.py:259-278) over the axes present of the last completed search; int64 arithmetic stored to int32
    __device__ static __forceinline__ void finish(Ctx& e, const AdvectParams& p) {
        if (!e.searched) return;
        const int4 ix = *idx(e.raw);
        int gxi = ix.w;
        if (p.g.decomposed && gxi >= 0) gxi += p.g.xi_offset;  // mode D: local column -> global column
        long long r = (long long)ix.z * p.g.xdim + (long long)gxi;
        if (p.g.nz > 0) r += (long long)(HZ ? ix.y : 0) * (p.g.ydim * p.g.xdim);
        e.ei = (int)r;
    }

    // gather the (t, z, y, x) corner block of every component from the node-interleaved copy into this lane's raw columns
    __device__ static __forceinline__ void refill(const FieldDev& f, float4* raw, int ti, int zi, int yi, int xi) {
        const long long ot[2] = {wrap_idx(ti, f.T) * f.sT, up_idx(ti, f.T) * f.sT};
        const long long oz[2] = {wrap_idx(zi, f.Z) * f.sZ, up_idx(zi, f.Z) * f.sZ};
        const long long oy[2] = {wrap_idx(yi, f.Y) * f.sY, up_idx(yi, f.Y) * f.sY};
        const long long ox[2] = {wrap_idx(xi, f.X) * f.sX, up_idx(xi, f.X) * f.sX};
        const float4* __restrict__ base = (const float4*)f.il;
#pragma unroll
        for (int pl = 0; pl < NV / 4; ++pl) {
            // records k = 4 pl .. 4 pl + 3,  k = (t * 2 + z) * 4 + y * 2 + x (HZ) | t * 4 + y * 2 + x: stored as they are loaded
            const long long o = ot[HZ ? (pl >> 1) : pl] + (HZ ? oz[pl & 1] : 0);
            raw[(4 * pl + 0) * PB_FAST_BLOCK] = ldg(base + o + oy[0] + ox[0]);
            raw[(4 * pl + 1) * PB_FAST_BLOCK] = ldg(base + o + oy[0] + ox[1]);
            raw[(4 * pl + 2) * PB_FAST_BLOCK] = ldg(base + o + oy[1] + ox[0]);
            raw[(4 * pl + 3) * PB_FAST_BLOCK] = ldg(base + o + oy[1] + ox[1]);
        }
    }

    // ---------------- side path: searches, states, refill; special samples are finished here ----------------
    // Inline at every evaluation site (out of line it costs the spill / reload of the hit path's live registers at every trip:
    // measured).  Reads and rewrites the lane's cells / reciprocals / indices / raw block in shared memory; what the caller
    // has in registers comes in as arguments and goes back through `out`.
    __device__ static __forceinline__
    void side_path(const AdvectParams* pp, float4* raw, int k, double ts, double zs, double ys, double xs, int state, SideResult* out) {
        const GridDev& g = pp->g;
        const FieldDev& f = pp->f;
        int flags = 0;
        if (!(0 <= ts && ts <= g.time_len)) {  // OutsideTimeInterval (index_search.py:85-86): state 70, sample (0, 0, 0)
            out->u = out->v = out->w = 0.0;
            out->state = PB_ERROR_OUTSIDE_TIME_INTERVAL;
            out->flags = SIDE_FINAL | SIDE_OUT_OF_TIME;
            return;
        }
        const double2 bz = HZ ? *cell(raw, 0) : double2{0.0, 0.0}, by = *cell(raw, 1), bx = *cell(raw, 2), bt = *cell(raw, 3);
        const int4 old = *idx(raw);  // key of the raw block: {ti, zi, yi, xi}
        AxisCell<double> ct{old.x, bt.x, bt.y}, cz{old.y, bz.x, bz.y}, cy{old.z, by.x, by.y}, cx{old.w, bx.x, bx.y};
        const double wt = ct.hi - ct.lo, wz = cz.hi - cz.lo, wy = cy.hi - cy.lo, wx = cx.hi - cx.lo;  // (NaN for a poisoned cell)
        if (old.x >= 0 && !(ct.lo == ct.lo)) ct.idx = -100;  // (a poisoned cell is not a neighbour-search seed)
        if (old.y >= 0 && !(cz.lo == cz.lo)) cz.idx = -100;
        if (old.z >= 0 && !(cy.lo == cy.lo)) cy.idx = -100;
        if (old.w >= 0 && !(cx.lo == cx.lo)) cx.idx = -100;
        axis_locate(g.time, g.nt, ts, ct);
        const int ti = ct.idx;
        int zi = 0;
        if (HZ) {
            axis_locate((const double*)g.depth, g.nz, zs, cz);
            zi = cz.idx;
        }
        axis_locate((const double*)g.lat, g.ny, ys, cy);
        axis_locate((const double*)g.lon, g.nx, xs, cx);
        const int yi = cy.idx, xi = cx.idx;
        {   // cell widths changed: new reciprocals (the division itself: correctly rounded)
            double2* const rp = rcp(raw);
            const double nwt = ct.hi - ct.lo, nwz = cz.hi - cz.lo, nwy = cy.hi - cy.lo, nwx = cx.hi - cx.lo;
            if ((HZ && !(nwz == wz)) || !(nwy == wy)) {
                double2 d;
                d.x = 1.0 / nwz; d.y = 1.0 / nwy;
                rp[0] = d;
            }
            if (!(nwx == wx) || !(nwt == wt)) {
                double2 d;
                d.x = 1.0 / nwx; d.y = 1.0 / nwt;
                rp[PB_FAST_BLOCK] = d;
            }
        }
        int4 now;
        now.x = ti; now.y = zi; now.z = yi; now.w = xi;
        *idx(raw) = now;
        flags |= SIDE_SEARCHED;
        if (g.decomposed) {  // mode D: a sentinel at a slab edge that is not the edge of the global domain = halo too small
            if ((xi == -2 && !g.left_global) || (xi == -1 && !g.right_global)) state = max(state, 99);
        }
        int s = state;
        if (xi == -1 || yi == -1 || zi == -1) s = max(s, (int)PB_ERROR_OUT_OF_BOUNDS);  // field.py:327-356
        if (zi == -2) s = max(s, (int)PB_ERROR_THROUGH_SURFACE);
        if (old.x != ti || (HZ && old.y != zi) || old.z != yi || old.w != xi) {
            refill(f, raw, ti, zi, yi, xi);
            flags |= SIDE_REFILLED;
        }
        // special: a sentinel index, or a sample not strictly inside (lo, hi] of the time / depth cell (tau or zeta == 0 on the
        // first node: lenT / lenZ == 1 for this particle, _xinterpolators.py:130-131; NaN; a degenerate cell)
        const bool t_in = ts > ct.lo && ts <= ct.hi, z_in = !HZ || (zs > cz.lo && zs <= cz.hi);
        const bool special = xi < 0 || yi < 0 || zi < 0 || !t_in || !z_in;
        {   // write the cells back; the ones a special sample involved are poisoned so that the lane comes back here next time
            const double nan = __longlong_as_double(0x7ff8000000000000LL);
            double2 d;
            d.x = ct.lo; d.y = ct.hi; if (!t_in) { d.x = nan; d.y = nan; }
            *cell(raw, 3) = d;
            if (HZ) { d.x = cz.lo; d.y = cz.hi; if (zi < 0 || !z_in) { d.x = nan; d.y = nan; } *cell(raw, 0) = d; }
            d.x = cy.lo; d.y = cy.hi; if (yi < 0) { d.x = nan; d.y = nan; }
            *cell(raw, 1) = d;
            d.x = cx.lo; d.y = cx.hi; if (xi < 0) { d.x = nan; d.y = nan; }
            *cell(raw, 2) = d;
        }
        if (special) {
            const double tau = axis_bcoord(g.nt, ts, ct), zeta = HZ ? axis_bcoord(g.nz, zs, cz) : 0.0;
            const double eta = axis_bcoord(g.ny, ys, cy), xsi = axis_bcoord(g.nx, xs, cx);
            const bool two_t = tau > 0;             // lenT, per particle (float64 grid: no dtype depends on the batch)
            const bool two_z = HZ && !(zeta <= 0);  // lenZ, per particle (a NaN depth must poison the value)
            double u = special_component<NV>(raw, 0, tau, zeta, eta, xsi, two_t, two_z);
            double v = special_component<NV>(raw, 1, tau, zeta, eta, xsi, two_t, two_z);
            double w = NC == 3 ? special_component<NV>(raw, 2, tau, zeta, eta, xsi, two_t, two_z) : 0.0;
            if (g.spherical) spherical(g, k == 0, ys, u, v);
            if (u != u || v != v || w != w) s = max(s, (int)PB_ERROR_INTERPOLATION);
            if (xi < 0 || yi < 0 || zi < 0) { u = 0.0; v = 0.0; w = 0.0; }
            out->u = u; out->v = v; out->w = w;
            flags |= SIDE_FINAL;
        }
        out->state = s;
        out->flags = flags;
    }

    // Z-lerp (:141-145) and bilinear (:147-152, left to right) of one component's T-lerped values
    __device__ static __forceinline__ double zxy(const double (&L)[NL], double zeta, double omz, double w00, double w01, double w10, double w11) {
        double r[4];
        if (HZ) {
#pragma unroll
            for (int j = 0; j < 4; ++j) r[j] = L[j] * omz + L[4 + j] * zeta;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) r[j] = L[j];
        }
        return w00 * r[0] + w01 * r[1] + w10 * r[2] + w11 * r[3];
    }

    // One VectorField.eval (field.py:250-304) at an RK4 stage position.  Odd stages sample a new time: the T-lerped block is
    // renewed; even stages reuse it.  RENEW = 0 / 1: decided at compile time (SCHED 2: the loop body holds a reusing and a renewing
    // copy of this function and runs twice per step); RENEW = -1: `renew_rt` decides (SCHED 1: one copy, four trips).
    template <int RENEW>
    __device__ static __forceinline__ void eval_fast(const AdvectParams& p, Ctx& e, const bool renew_rt, const bool first, const double ts,
                                                     const double zs, const double ys, const double xs, double& u, double& v, double& w) {
        const GridDev& g = p.g;
        const bool renew = RENEW < 0 ? renew_rt : (RENEW != 0);
        float4* const raw = e.raw;
        bool lerp_now = renew;
        double2 bz, by, bx, bt;  // {lo, hi} of the current cells
        // The cells are READ FROM SHARED MEMORY at every evaluation, on purpose (volatile loads: neither NVVM nor ptxas may forward
        // them): they only change in the side path, and keeping them in registers across evaluations costs moves and spills.
#pragma unroll 1
        for (int trip = 0;; ++trip) {
            bz = HZ ? lds_volatile(cell(raw, 0)) : double2{0.0, 0.0};
            by = lds_volatile(cell(raw, 1));
            bx = lds_volatile(cell(raw, 2));
            bt = (renew || trip) ? lds_volatile(cell(raw, 3)) : double2{0.0, 0.0};  // (even stages test the cached lerp's time)
            bool hit = xs > bx.x && xs <= bx.y && ys > by.x && ys <= by.y;
            if (HZ) hit = hit && zs > bz.x && zs <= bz.y;
            hit = hit && (renew ? (ts > bt.x && ts <= bt.y) : (ts == e.lerp_t));
            if (hit || trip) break;
            SideResult r;
            side_path(&p, raw, first ? 0 : 1, ts, zs, ys, xs, e.state, &r);
            e.state = r.state;
            if (r.flags & SIDE_OUT_OF_TIME) e.out_of_time = true;
            if (r.flags & SIDE_SEARCHED) e.searched = true;
            if (r.flags & SIDE_REFILLED) { e.refills++; e.lerp_t = -1.0; }
            if (r.flags & SIDE_FINAL) {
                u = r.u; v = r.v; w = r.w;
                return;
            }
            lerp_now = true;  // (an even stage after a cell change: its block has to be lerped for this sample time first)
        }
        // ---------------- straight-line path: every cell is current, 0 < bcoord <= 1 on every axis ----------------
        // bcoord = (x - lo) / (hi - lo), index_search.py:57 (denominator in the axis dtype), with the cell width's cached reciprocal
        const double2 r_zy = rcp(raw)[0], r_xt = rcp(raw)[PB_FAST_BLOCK];
        const double zeta = HZ ? div_by_cached(zs - bz.x, bz.y - bz.x, r_zy.x) : 0.0;
        const double eta = div_by_cached(ys - by.x, by.y - by.x, r_zy.y);
        const double xsi = div_by_cached(xs - bx.x, bx.y - bx.x, r_xt.x);
        const double omz = 1 - zeta;
        const double w00 = (1 - xsi) * (1 - eta), w01 = xsi * (1 - eta), w10 = (1 - xsi) * eta, w11 = xsi * eta;
        double2* const lp = lrp(raw);
        double q[3] = {0.0, 0.0, 0.0};
        if (lerp_now) {
            const double tau = div_by_cached(ts - bt.x, bt.y - bt.x, r_xt.y);
            const double omt = 1 - tau;
            // two corners (y, x) at a time: their node records at both depth and both time levels -> the T-lerp of every component
            // (_xinterpolators.py:135-139), stored pairwise into the T-lerped block, then straight on: Z-lerp (:141-145) and the
            // bilinear sum (:147-152) accumulated corner by corner in the reference's left-to-right order
            constexpr int NZ = HZ ? 2 : 1;
            const double wgt[4] = {w00, w01, w10, w11};
#pragma unroll
            for (int pr = 0; pr < 2; ++pr) {
                double L[3][NZ][2];
#pragma unroll
                for (int zz = 0; zz < NZ; ++zz) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int k = zz * 4 + 2 * pr + h;  // corner (z, y, x) within a time level
                        const float4 a = raw[k * PB_FAST_BLOCK], b = raw[(NL + k) * PB_FAST_BLOCK];
                        L[0][zz][h] = (double)a.x * omt + (double)b.x * tau;
                        L[1][zz][h] = (double)a.y * omt + (double)b.y * tau;
                        if (NC == 3) L[2][zz][h] = (double)a.z * omt + (double)b.z * tau;
                    }
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        double2 d;
                        d.x = L[c][zz][0]; d.y = L[c][zz][1];
                        lp[(c * (NL / 2) + (zz * 4 + 2 * pr) / 2) * PB_FAST_BLOCK] = d;
                    }
                }
#pragma unroll
                for (int c = 0; c < NC; ++c) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const double r = HZ ? L[c][0][h] * omz + L[c][NZ - 1][h] * zeta : L[c][0][h];
                        q[c] = (pr == 0 && h == 0) ? wgt[0] * r : q[c] + wgt[2 * pr + h] * r;
                    }
                }
            }
            e.lerp_t = ts;
        } else {
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                double L[NL];
#pragma unroll
                for (int j = 0; j < NL / 2; ++j) {
                    const double2 d = lp[(c * (NL / 2) + j) * PB_FAST_BLOCK];
                    L[2 * j] = d.x; L[2 * j + 1] = d.y;
                }
                q[c] = zxy(L, zeta, omz, w00, w01, w10, w11);
            }
        }
        u = q[0]; v = q[1]; w = NC == 3 ? q[2] : 0.0;
        if (g.spherical) spherical(g, first, ys, u, v);
        if (u != u || v != v || w != w) e.state = max(e.state, (int)PB_ERROR_INTERPOLATION);  // field.py:288-290
    }

    // u /= deg2m * cos(deg2rad(y)); v /= deg2m (_xinterpolators.py:182-184).  Stage 1 samples at the particle's own float32
    // latitude: the factor is float32 arithmetic there (and the float64 value is divided by its float64 promotion).
    __device__ static __forceinline__ void spherical(const GridDev& g, bool first, double ys, double& u, double& v) {
        double conv;
        if (first) conv = (double)((float)g.deg2m * cos_np(deg2rad_np((float)ys)));
        else conv = g.deg2m * cos_np(deg2rad_np(ys));
        u = u / conv;
        v = div_by_cached_guarded(v, g.deg2m, g.inv_deg2m);
    }

    // the generic skeleton's entry point is not used by a FAST_RK4 policy
    template <class PZ, class PY, class PX>
    __device__ static __forceinline__ void eval(const AdvectParams&, Ctx&, bool, double, PZ, PY, PX, Val&, Val&, Val&) {}
};

// ------------------------------------------------------------------------------------------------
// launch
// ------------------------------------------------------------------------------------------------
bool agrid_fast_applies(const AdvectParams& p, bool coord_f64, bool data_f64, bool has_time, int nc) {
    if (!coord_f64 || data_f64 || !has_time || !p.f.il || p.f.windowed || p.g.curvilinear) return false;
    if (!(p.scheme == PB_ADVECTION_RK4 || p.scheme == PB_ADVECTION_RK4_3D)) return false;
    if (nc == 3 && p.g.nz < 2) return false;
    return p.g.nt >= 2 && p.g.nx >= 2 && p.g.ny >= 2;
}

template <int NC, bool HZ, int SCHED, bool DIFF>
static cudaError_t launch_fast2(const AdvectParams& p, cudaStream_t s) {
    using Pol = AFastPolicy<NC, HZ, SCHED>;
    const long long grid = (p.P.n + PB_FAST_BLOCK - 1) / PB_FAST_BLOCK;
    if (Pol::SMEM > 48 * 1024) {
        cudaError_t ce = cudaFuncSetAttribute(advect_kernel<Pol, DIFF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Pol::SMEM);
        if (ce != cudaSuccess) return ce;
    }
    advect_kernel<Pol, DIFF><<<(unsigned)grid, PB_FAST_BLOCK, Pol::SMEM, s>>>(p);
    return cudaGetLastError();
}
// (each schedule is instantiated for the lists it is the kernel of, plus the advection-only form of SCHED 1 for A/B runs)
template <int NC, bool HZ>
static cudaError_t launch_fast1(const AdvectParams& p, int sched, cudaStream_t s) {
    if (p.diffusion) return sched == 2 ? launch_fast2<NC, HZ, 2, true>(p, s) : launch_fast2<NC, HZ, 1, true>(p, s);
    return sched == 2 ? launch_fast2<NC, HZ, 2, false>(p, s) : launch_fast2<NC, HZ, 1, false>(p, s);
}

cudaError_t launch_agrid_fast(const AdvectParams& p, int nc, int sched, cudaStream_t s) {
    const bool hz = p.g.nz >= 2;
    if (nc == 3) return launch_fast1<3, true>(p, sched, s);
    return hz ? launch_fast1<2, true>(p, sched, s) : launch_fast1<2, false>(p, sched, s);
}
