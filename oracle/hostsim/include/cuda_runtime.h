// TEST INFRASTRUCTURE ONLY (oracle/hostsim) -- NOT part of the product, never loaded by parcels_b200 on its own.
//
// A minimal stand-in for <cuda_runtime.h> that lets g++ compile the product's CUDA sources (parcels_b200/csrc/*.cu, after
// oracle/hostsim/build.py has rewritten the `kernel<<<...>>>(...)` launch statements into HS_LAUNCH calls) for the HOST.
// The result, oracle/_build/hostsim/libparcels_b200_hostsim.so, exports the product's C-ABI with "device memory" = malloc
// and every kernel executed one thread at a time.  Purpose: check the LOGIC of the kernels' source against the oracle on
// machines without a GPU (tests/test_hostsim_cpu.py).  It says nothing about the GPU build's numerics beyond what the
// shared source implies (libm instead of libdevice), and nothing at all about performance.
#pragma once
#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>

#define PB_HOSTSIM 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define HS_NOINLINE __attribute__((noinline))  // build.py rewrites __noinline__ (a reserved spelling inside libstdc++) to this
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n)
#define __SM_32_INTRINSICS_DECL__

// ---- execution model: ONE thread runs at a time; every thread is lane 0 of its own warp and thread 0 of its own block ----
struct hs_dim3 {
    unsigned x = 1, y = 1, z = 1;
};
inline hs_dim3 threadIdx, blockIdx, blockDim, gridDim;
alignas(16) inline unsigned char pb_smem[256 * 1024];  // `extern __shared__ unsigned char pb_smem[]` of the kernels

// Warp reductions of the kernels' reports.  Convention of the sources: counters that are SUMMED are unsigned, values that
// are MAX/MIN-reduced are signed -- a lone lane contributes 0 to a sum and itself to an extremum.
inline unsigned long long __shfl_xor_sync(unsigned, unsigned long long, int) { return 0; }
inline unsigned __shfl_xor_sync(unsigned, unsigned, int) { return 0; }
inline long long __shfl_xor_sync(unsigned, long long v, int) { return v; }
inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
inline long long __shfl_up_sync(unsigned, long long v, int) { return v; }  // only in kernels hostsim replaces (sel_scan)
#define __grid_constant__
#define __constant__ const
inline void __syncthreads() {}
inline int __syncthreads_count(int p) { return p ? 1 : 0; }
inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }

template <class T>
inline T __ldg(const T* p) { return *p; }
struct double2 {
    double x, y;
};
struct float2 {
    float x, y;
};
struct alignas(16) int4 {
    int x, y, z, w;
};
struct alignas(16) float4 {
    float x, y, z, w;
};
inline double __longlong_as_double(long long v) { double r; std::memcpy(&r, &v, 8); return r; }

template <class T>
inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T>
inline T atomicAdd_system(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T>
inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T>
inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T>
inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }

inline long long __double_as_longlong(double d) { long long r; std::memcpy(&r, &d, 8); return r; }
inline void sincospi(double x, double* s, double* c) {  // exact reduction to [-0.5, 0.5] half-turns, then libm
    double r = std::fmod(x, 2.0);
    if (r > 1.0) r -= 2.0;
    if (r < -1.0) r += 2.0;
    *s = std::sin(3.14159265358979323846 * r);
    *c = std::cos(3.14159265358979323846 * r);
}
// exact reduction in half-turns to an argument where the result is not small, libm in double, one rounding to float: within
// CUDA's documented 1 ulp (exact zeros at the integers and half-integers, like CUDA's)
inline void sincospif(float x, float* s, float* c) {
    const double r = std::remainder((double)x, 2.0);  // [-1, 1], exact
    const double a = std::fabs(r);
    *s = (float)std::copysign(std::sin(3.14159265358979323846 * std::min(a, 1.0 - a)), r);  // 1 - a: exact where it is the min
    *c = (float)(a < 0.25 ? std::cos(3.14159265358979323846 * a) : std::sin(3.14159265358979323846 * (0.5 - a)));  // 0.5 - a: exact
}
using std::isfinite;
// CUDA's min / max accept mixed integer types
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline long long min(long long a, int b) { return a < b ? a : b; }
inline long long max(long long a, int b) { return a > b ? a : b; }
inline long long min(int a, long long b) { return a < b ? a : b; }
inline long long max(int a, long long b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }

// ---- runtime API: "device" memory is host memory, streams are synchronous ----
typedef int cudaError_t;
struct hs_stream {
    int id;
};
typedef hs_stream* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNoDevice = 100 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyHostToHost = 0 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct hs_event {
    std::chrono::steady_clock::time_point t;
};
typedef hs_event* cudaEvent_t;
struct cudaDeviceProp {
    char name[256];
    int major, minor, multiProcessorCount;
    size_t totalGlobalMem;
};

inline bool hs_enabled() {  // the simulation only answers to the test harness
    const char* e = std::getenv("PB_HOSTSIM_TEST");
    return e && e[0] == '1';
}
inline cudaError_t cudaGetDeviceCount(int* n) { *n = hs_enabled() ? 1 : 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return hs_enabled() ? cudaSuccess : cudaErrorNoDevice; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    std::memset(p, 0, sizeof(*p));
    std::snprintf(p->name, sizeof(p->name), "hostsim (kernel sources compiled for the CPU; tests only)");
    p->major = 9; p->minor = 0;  // the engine insists on sm_90: the simulated device claims to be one
    p->multiProcessorCount = 1;
    return cudaSuccess;
}
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
// CUDA IPC: the simulated "device" memory is private to the process -- peers of the same process are linked by address
struct cudaIpcMemHandle_t {
    char reserved[64];
};
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void*) { std::memset(h, 0, sizeof(*h)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) { return cudaErrorInvalidValue; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "hostsim error"; }
template <class T>
inline cudaError_t cudaMalloc(T** p, size_t n) { *p = (T*)std::malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T>
inline cudaError_t cudaMallocHost(T** p, size_t n) { *p = (T*)std::calloc(1, n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = new hs_stream{1}; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new hs_event(); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
    return cudaSuccess;
}
template <class F>
inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }

// Opt-in launch trace: when PB_HOSTSIM_TRACE names a file, every launch appends the (mangled) symbol of its kernel to it, one per
// line, so that a test can tell which template instantiations a run launched.  Without the variable it does nothing.
inline void hs_trace(const void* f) {
    const char* path = std::getenv("PB_HOSTSIM_TRACE");
    if (!path || !path[0]) return;
    Dl_info info;
    if (!dladdr(f, &info) || !info.dli_sname) return;
    if (FILE* out = std::fopen(path, "a")) {
        std::fprintf(out, "%s\n", info.dli_sname);
        std::fclose(out);
    }
}

// ---- kernel launches: build.py rewrites `k<<<grid, block, smem, stream>>>(args)` into HS_LAUNCH((k), grid, block, smem, stream, args)
template <class F, class... Args>
inline void hs_launch(F f, unsigned long long grid, unsigned long long block, Args... args) {
    hs_trace((const void*)f);
    const unsigned long long n = grid * block;  // kernels index with blockIdx.x * blockDim.x + threadIdx.x and guard i < n themselves
    blockDim.x = 1; gridDim.x = (unsigned)n; threadIdx.x = 0;
    for (unsigned long long i = 0; i < n; ++i) {
        blockIdx.x = (unsigned)i;
        f(args...);
    }
}
#define HS_LAUNCH(k, grid, block, smem, stream, ...) hs_launch(k, (unsigned long long)(grid), (unsigned long long)(block), __VA_ARGS__)
// block-cooperative kernels (ballot / __syncthreads scans) are replaced by per-block host functions injected by build.py
template <class F, class... Args>
inline void hs_launch_blocks(F f, unsigned long long grid, unsigned long long block, Args... args) {
    blockDim.x = (unsigned)block; gridDim.x = (unsigned)grid; threadIdx.x = 0;
    for (unsigned long long b = 0; b < grid; ++b) {
        blockIdx.x = (unsigned)b;
        f(args...);
    }
}
#define HS_LAUNCH_BLOCKS(k, grid, block, smem, stream, ...) hs_launch_blocks(k, (unsigned long long)(grid), (unsigned long long)(block), __VA_ARGS__)
