// agrid.cu -- launchers of the XLinear_Velocity A-grid kernels (the headline hot path); device code in agrid.cuh
#include "agrid.cuh"

int agrid_launch_block() { return PB_BLOCK; }

template <class A, class D, bool HT, int NC>
static cudaError_t launch1(const AdvectParams& p, cudaStream_t s) {
    const int block = PB_BLOCK;
    const long long grid = (p.P.n + block - 1) / block;
#ifdef PB_SMEM_CACHE
    const size_t smem = (size_t)NC * 16 * sizeof(typename decltype(EvalCtx<A, D, NC>::cor)::S) * PB_BLOCK;
    if (smem > 48 * 1024) {
        cudaError_t ce = cudaFuncSetAttribute(advect_kernel<AGridPolicy<A, D, HT, NC>>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (ce != cudaSuccess) return ce;
    }
#else
    const size_t smem = 0;
#endif
    advect_kernel<AGridPolicy<A, D, HT, NC>><<<(unsigned)grid, block, smem, s>>>(p);
    return cudaGetLastError();
}

template <class A, class D>
static cudaError_t launch_ad(const AdvectParams& p, bool ht, int nc, cudaStream_t s) {
    if (ht) return nc == 3 ? launch1<A, D, true, 3>(p, s) : launch1<A, D, true, 2>(p, s);
    return nc == 3 ? launch1<A, D, false, 3>(p, s) : launch1<A, D, false, 2>(p, s);
}

cudaError_t launch_agrid(const AdvectParams& p, bool coord_f64, bool data_f64, bool has_time, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? launch_ad<double, double>(p, has_time, nc, s) : launch_ad<double, float>(p, has_time, nc, s);
    return data_f64 ? launch_ad<float, double>(p, has_time, nc, s) : launch_ad<float, float>(p, has_time, nc, s);
}

template <class A, class D, bool HT, int NC>
static cudaError_t sample1(const SampleParams& p, cudaStream_t s) {
#ifdef PB_SMEM_CACHE
    const size_t smem = (size_t)NC * 16 * sizeof(typename decltype(EvalCtx<A, D, NC>::cor)::S) * PB_BLOCK;
    if (smem > 48 * 1024) {
        cudaError_t ce = cudaFuncSetAttribute(sample_kernel<AGridPolicy<A, D, HT, NC>>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (ce != cudaSuccess) return ce;
    }
#else
    const size_t smem = 0;
#endif
    sample_kernel<AGridPolicy<A, D, HT, NC>><<<(unsigned)((p.n + PB_BLOCK - 1) / PB_BLOCK), PB_BLOCK, smem, s>>>(p);
    return cudaGetLastError();
}
template <class A, class D>
static cudaError_t sample_ad(const SampleParams& p, bool ht, int nc, cudaStream_t s) {
    if (ht) return nc == 3 ? sample1<A, D, true, 3>(p, s) : sample1<A, D, true, 2>(p, s);
    return nc == 3 ? sample1<A, D, false, 3>(p, s) : sample1<A, D, false, 2>(p, s);
}
cudaError_t launch_sample_agrid(const SampleParams& p, bool coord_f64, bool data_f64, bool has_time, int nc, cudaStream_t s) {
    if (coord_f64) return data_f64 ? sample_ad<double, double>(p, has_time, nc, s) : sample_ad<double, float>(p, has_time, nc, s);
    return data_f64 ? sample_ad<float, double>(p, has_time, nc, s) : sample_ad<float, float>(p, has_time, nc, s);
}
