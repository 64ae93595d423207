// curva.cu -- XLinear_Velocity on CURVILINEAR grids (an A-grid whose lon / lat are 2-D): the curvilinear search of cgrid.cuh
// (reference _core/index_search.py:242-295 behind _core/xgrid.py:316-356) feeding the A-grid interpolator
// (interpolators/_xinterpolators.py:112-190).  Its own translation unit: the C-grid kernels of cgrid.cu stay the measured builds.
#include "cgrid.cuh"

static constexpr int ADVECT_BLOCK = 128;
int curva_launch_block() { return ADVECT_BLOCK; }

template <class Policy>
static cudaError_t launch_policy(const AdvectParams& p, cudaStream_t s) {
    const int block = ADVECT_BLOCK;
    advect_kernel<Policy><<<(unsigned)((p.P.n + block - 1) / block), block, 0, s>>>(p);
    return cudaGetLastError();
}
template <class A, class D>
static cudaError_t launch_ad(const AdvectParams& p, int nc, cudaStream_t s) {
    if (p.g.decomposed) {  // column slabs (mode D)
        if (p.g.spherical)
            return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, true, CURV_XLINEAR | CURV_COLUMNS>>(p, s) : launch_policy<CurvPolicy<A, D, 2, true, CURV_XLINEAR | CURV_COLUMNS>>(p, s);
        return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, false, CURV_XLINEAR | CURV_COLUMNS>>(p, s) : launch_policy<CurvPolicy<A, D, 2, false, CURV_XLINEAR | CURV_COLUMNS>>(p, s);
    }
    if (p.g.spherical) return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, true, 1>>(p, s) : launch_policy<CurvPolicy<A, D, 2, true, 1>>(p, s);
    return nc == 3 ? launch_policy<CurvPolicy<A, D, 3, false, 1>>(p, s) : launch_policy<CurvPolicy<A, D, 2, false, 1>>(p, s);
}
cudaError_t launch_curv_agrid(const AdvectParams& p, bool coord_f64, bool data_f64, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? launch_ad<double, double>(p, nc, s) : launch_ad<double, float>(p, nc, s);
    return data_f64 ? launch_ad<float, double>(p, nc, s) : launch_ad<float, float>(p, nc, s);
}

template <class Policy>
static cudaError_t sample_policy(const SampleParams& p, cudaStream_t s) {
    sample_kernel<Policy><<<(unsigned)((p.n + 127) / 128), 128, 0, s>>>(p);
    return cudaGetLastError();
}
template <class A, class D>
static cudaError_t sample_ad(const SampleParams& p, int nc, cudaStream_t s) {
    if (p.g.spherical) return nc == 3 ? sample_policy<CurvPolicy<A, D, 3, true, 1>>(p, s) : sample_policy<CurvPolicy<A, D, 2, true, 1>>(p, s);
    return nc == 3 ? sample_policy<CurvPolicy<A, D, 3, false, 1>>(p, s) : sample_policy<CurvPolicy<A, D, 2, false, 1>>(p, s);
}
cudaError_t launch_sample_curv_agrid(const SampleParams& p, bool coord_f64, bool data_f64, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? sample_ad<double, double>(p, nc, s) : sample_ad<double, float>(p, nc, s);
    return data_f64 ? sample_ad<float, double>(p, nc, s) : sample_ad<float, float>(p, nc, s);
}
