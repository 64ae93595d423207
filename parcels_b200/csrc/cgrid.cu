// cgrid.cu -- instantiations and launchers of the C-grid kernels (cgrid.cuh): CGrid_Velocity on rectilinear and curvilinear
// grids, AdvectionRK45 on them, scalar Field.eval on curvilinear grids.
#include "cgrid.cuh"

cudaError_t launch_precompute_cells(const void* lon, const void* lat, int ny, int nx, bool coord_f64, double* out, cudaStream_t s) {
    const long long ncell = (long long)(ny - 1) * (nx - 1);
    const unsigned grid = (unsigned)((ncell + 127) / 128);
    if (coord_f64) precompute_cells_kernel<double><<<grid, 128, 0, s>>>((const double*)lon, (const double*)lat, ny, nx, out);
    else precompute_cells_kernel<float><<<grid, 128, 0, s>>>((const float*)lon, (const float*)lat, ny, nx, out);
    return cudaGetLastError();
}

template <class A, class D>
static cudaError_t scalar_curv_ad(const SampleParams& p, int mode, bool has_time, cudaStream_t s) {
    const unsigned grid = (unsigned)((p.n + 127) / 128);
    if (p.g.spherical) sample_scalar_curv_kernel<A, D, true><<<grid, 128, 0, s>>>(p, mode, has_time ? 1 : 0);
    else sample_scalar_curv_kernel<A, D, false><<<grid, 128, 0, s>>>(p, mode, has_time ? 1 : 0);
    return cudaGetLastError();
}
// mode: 4 XNearest, 5 CGrid_Tracer (the numbering of agrid.cuh)
cudaError_t launch_sample_scalar_curv(const SampleParams& p, int mode, bool coord_f64, bool data_f64, bool has_time, cudaStream_t s) {
    if (coord_f64) return data_f64 ? scalar_curv_ad<double, double>(p, mode, has_time, s) : scalar_curv_ad<double, float>(p, mode, has_time, s);
    return data_f64 ? scalar_curv_ad<float, double>(p, mode, has_time, s) : scalar_curv_ad<float, float>(p, mode, has_time, s);
}

static constexpr int ADVECT_BLOCK = 128;
int cgrid_launch_block() { return ADVECT_BLOCK; }

template <class Policy>
static cudaError_t launch_policy(const AdvectParams& p, cudaStream_t s) {
    const int block = ADVECT_BLOCK;
    const long long grid = (p.P.n + block - 1) / block;
    // (advection-only launches carry neither the Philox / Box-Muller code nor its registers in the time loop)
    if (Policy::RUNTIME_DTYPE && !p.diffusion) advect_kernel<Policy, false><<<(unsigned)grid, block, 0, s>>>(p);
    else advect_kernel<Policy><<<(unsigned)grid, block, 0, s>>>(p);
    return cudaGetLastError();
}

template <class A, class D>
static cudaError_t launch_ad(const AdvectParams& p, int nc, cudaStream_t s) {
    if (p.g.curvilinear && p.g.decomposed) {  // column slabs (mode D)
        if (p.g.spherical)
            return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, true, CURV_COLUMNS>>(p, s) : launch_policy<CurvPolicy<A, D, 2, true, CURV_COLUMNS>>(p, s);
        return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, false, CURV_COLUMNS>>(p, s) : launch_policy<CurvPolicy<A, D, 2, false, CURV_COLUMNS>>(p, s);
    }
    if (p.g.curvilinear) {
        if (p.g.spherical) return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, true>>(p, s) : launch_policy<CurvPolicy<A, D, 2, true>>(p, s);
        return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, false>>(p, s) : launch_policy<CurvPolicy<A, D, 2, false>>(p, s);
    }
    return nc == 3 ? launch_policy<CGridPolicy<A, D, 3>>(p, s) : launch_policy<CGridPolicy<A, D, 2>>(p, s);
}

cudaError_t launch_cgrid(const AdvectParams& p, bool coord_f64, bool data_f64, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? launch_ad<double, double>(p, nc, s) : launch_ad<double, float>(p, nc, s);
    return data_f64 ? launch_ad<float, double>(p, nc, s) : launch_ad<float, float>(p, nc, s);
}

// AdvectionRK45 on C-grids (rk45.cuh): rectilinear CGridPolicy and curvilinear CurvPolicy, 2-D (fieldset.UV)
template <class Policy>
static cudaError_t rk45_policy(const Rk45Params& q, cudaStream_t s) {
    const int block = 128;
    rk45_kernel<Policy><<<(unsigned)((q.base.P.n + block - 1) / block), block, 0, s>>>(q);
    return cudaGetLastError();
}
template <class A, class D>
static cudaError_t rk45_ad(const Rk45Params& q, cudaStream_t s) {
    if (q.base.g.curvilinear && q.base.g.decomposed)  // column slabs (mode D)
        return q.base.g.spherical ? rk45_policy<CurvPolicy<A, D, 2, true, CURV_COLUMNS>>(q, s) : rk45_policy<CurvPolicy<A, D, 2, false, CURV_COLUMNS>>(q, s);
    if (q.base.g.curvilinear) return q.base.g.spherical ? rk45_policy<CurvPolicy<A, D, 2, true>>(q, s) : rk45_policy<CurvPolicy<A, D, 2, false>>(q, s);
    return rk45_policy<CGridPolicy<A, D, 2>>(q, s);
}
cudaError_t launch_rk45_cgrid(const AdvectParams& p, double* dt, double* next_dt, int* iters, int next_dt_f32, double tol, double min_dt,
                              double max_dt, bool coord_f64, bool data_f64, cudaStream_t s) {
    Rk45Params q{p, dt, next_dt, iters, next_dt_f32, tol, min_dt, max_dt};
    if (coord_f64) return data_f64 ? rk45_ad<double, double>(q, s) : rk45_ad<double, float>(q, s);
    return data_f64 ? rk45_ad<float, double>(q, s) : rk45_ad<float, float>(q, s);
}

// Column slabs (mode D), the classify pass of the collective transport: dest[i] = the rank whose cell columns [edges[r], edges[r+1])
// hold the cell particle i's next search finds -- the ownership test the advection kernels run at the top of an iteration, with
// the hint rule of that iteration (iters: per-particle iteration counts of the call, NULL: every particle at its first) -- or -1
// when the particle stays (state not Evaluate, no cell found, a cell of this rank).  counts[r]: leavers per rank, counts[nranks]:
// stayers.
template <class Policy>
__global__ void classify_columns_kernel(const AdvectParams p, const int* __restrict__ iters, int no_hint, const double* __restrict__ edges,
                                        int nranks, int rank, int* dest, unsigned long long* counts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.P.n) return;
    int d = -1;
    if (p.P.state[i] == PB_EVALUATE) {
        typename Policy::Ctx e;
        Policy::init(e, p, p.P.ei[i]);
        const int col = Policy::owner_search(p, e, no_hint && (!iters || iters[i] == 0), p.P.x[i], p.P.y[i]);
        if (col >= 0) {
            int r = 0;
            while (r + 1 < nranks && (double)col >= edges[r + 1]) ++r;
            if (r != rank) d = r;
        }
    }
    dest[i] = d;
    atomicAdd(&counts[d < 0 ? nranks : d], 1ULL);
}
template <class A>
static void classify_columns_a(const AdvectParams& p, const int* iters, int no_hint, const double* edges, int nranks, int rank, int* dest,
                               unsigned long long* counts, cudaStream_t s) {
    const unsigned grid = (unsigned)((p.P.n + 127) / 128);
    if (p.g.spherical)
        classify_columns_kernel<CurvPolicy<A, float, 2, true, CURV_COLUMNS>><<<grid, 128, 0, s>>>(p, iters, no_hint, edges, nranks, rank, dest, counts);
    else
        classify_columns_kernel<CurvPolicy<A, float, 2, false, CURV_COLUMNS>><<<grid, 128, 0, s>>>(p, iters, no_hint, edges, nranks, rank, dest, counts);
}
cudaError_t launch_classify_columns(const AdvectParams& p, bool coord_f64, const int* iters, int no_hint, const double* edges, int nranks,
                                    int rank, int* dest, unsigned long long* counts, cudaStream_t s) {
    if (coord_f64) classify_columns_a<double>(p, iters, no_hint, edges, nranks, rank, dest, counts, s);
    else classify_columns_a<float>(p, iters, no_hint, edges, nranks, rank, dest, counts, s);
    return cudaGetLastError();
}

template <class Policy>
static cudaError_t sample_policy(const SampleParams& p, cudaStream_t s) {
    sample_kernel<Policy><<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p);
    return cudaGetLastError();
}
template <class A, class D>
static cudaError_t sample_ad(const SampleParams& p, int nc, cudaStream_t s) {
    if (p.g.curvilinear) {
        if (p.g.spherical) return nc == 3 ? sample_policy<CurvPolicy<A, D, 3, true>>(p, s) : sample_policy<CurvPolicy<A, D, 2, true>>(p, s);
        return nc == 3 ? sample_policy<CurvPolicy<A, D, 3, false>>(p, s) : sample_policy<CurvPolicy<A, D, 2, false>>(p, s);
    }
    return nc == 3 ? sample_policy<CGridPolicy<A, D, 3>>(p, s) : sample_policy<CGridPolicy<A, D, 2>>(p, s);
}
cudaError_t launch_sample_cgrid(const SampleParams& p, bool coord_f64, bool data_f64, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? sample_ad<double, double>(p, nc, s) : sample_ad<double, float>(p, nc, s);
    return data_f64 ? sample_ad<float, double>(p, nc, s) : sample_ad<float, float>(p, nc, s);
}

// pb_debug_math: the math primitives the kernels call, one element per lane (here because sin_lat / sincos_lon are cgrid.cuh's)
__global__ void debug_math_kernel(int op, long long n, const double* a, const double* b, double* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = a[i];
    double o0 = 0.0, o1 = 0.0;
    switch (op) {
        case PB_MATH_COS_NP: o0 = cos_np(x); break;
        case PB_MATH_SIN_LAT: o0 = sin_lat(x); break;
        case PB_MATH_SINCOS_LON: sincos_lon(x, o0, o1); break;
        case PB_MATH_DIV_BY_CACHED: o1 = 1.0 / b[i]; o0 = div_by_cached(x, b[i], o1); break;
        case PB_MATH_DIV_BY_CACHED_GUARDED: o1 = 1.0 / b[i]; o0 = div_by_cached_guarded(x, b[i], o1); break;
        case PB_MATH_BOX_MULLER_F32: box_muller_f32((uint32_t)x, (uint32_t)b[i], o0, o1); break;
        case PB_MATH_COSF: o0 = (double)cosf_ool((float)x); break;
        case PB_MATH_SINF: o0 = (double)sinf_ool((float)x); break;
        case PB_MATH_COS: o0 = cos_ool(x); break;
        case PB_MATH_SIN: o0 = sin_ool(x); break;
    }
    out[2 * i] = o0;
    out[2 * i + 1] = o1;
}
cudaError_t launch_debug_math(int op, long long n, const double* a, const double* b, double* out, cudaStream_t s) {
    debug_math_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(op, n, a, b, out);
    return cudaGetLastError();
}
