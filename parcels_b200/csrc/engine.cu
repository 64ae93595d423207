// engine.cu -- libparcels_b200.so: hand-written sm_90a CUDA for the Parcels hot path
//   ParticleSet.execute(AdvectionRK4 | AdvectionRK4_3D | AdvectionEE | AdvectionRK2[_3D]
//                       [+ DiffusionUniformKh] [+ delete-on-error])
// behind the C-ABI declared in include/parcels_b200.h.
//
// Design (DESIGN.md has the long version):
//  * one lane per particle; the WHOLE dt loop of Kernel.execute (reference _core/kernel.py:174-247)
//    runs in-kernel with the particle in registers, so particle state crosses HBM once per call;
//  * the 2x2x2x2 (t,z,y,x) corner block of U,V,W that brackets a particle (16 values / component,
//    reference interpolators/_xinterpolators.py:78-96) is kept in REGISTERS together with the cell
//    bounds; a particle stays in its cell for tens of steps, so the 4 RK stages of most steps need
//    no memory traffic at all -- the field is gathered from HBM only when a stage position leaves
//    the cached cell ("corner cache refill");
//  * all arithmetic reproduces NumPy's dtype promotion of the reference (f32 particle positions,
//    f32/f64 grid coordinates and data, f64 time) operation by operation, with FMA contraction OFF
//    (-fmad=false), so cell indices are bit-exact and trajectories agree to the last f32 ulp
//    (transcendentals aside);
//  * no tensor cores: this is a gather + fp64 lerp path, there is no contraction to map on wgmma.
//
// This file is compiled ONLY for sm_90a (H100).  There is no CPU fallback anywhere in the product.

#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"

// NVTX ranges per phase (upload / advect / download / migrate / output ...): visible in Nsight Systems / ncu --nvtx, free when no
// tool is attached (header-only nvtx3: the injection library is looked up at the first call)
#ifndef PB_HOSTSIM
#include <nvtx3/nvToolsExt.h>
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
#else
struct NvtxRange {
    explicit NvtxRange(const char*) {}
};
#endif
#define PB_RANGE(name) NvtxRange pb_nvtx_range_(name)

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int32_t fail(int32_t code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(PB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// whole-view OutsideTimeInterval flag (index_search.py:85-86 + field.py:31-44)
__global__ void flag_view_kernel(ParticlesDev P, double dt, double endtime, int new_state) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const int sign = dt > 0 ? 1 : -1;
    const int s = P.state[i];
    const double tte = sign * (endtime - P.t[i]);
    if ((s == PB_SUCCESS || s == PB_EVALUATE) && tte >= 0) P.state[i] = new_state;
}

__global__ void normals_kernel(unsigned long long seed, unsigned long long rng_call, long long iter, long long n,
                               const long long* pid, double* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double zx, zy;
    wiener_normals(seed, rng_call, iter, pid[i], zx, zy);
    out[2 * i] = zx;
    out[2 * i + 1] = zy;
}


// ------------------------------------------------------------------------------------------------
// migration kernels (mode D)
// ------------------------------------------------------------------------------------------------
// (MigRecord: common.cuh)

// dest[i] = destination rank of particle i, or -1 if it stays.  A particle moves iff it still has to be
// advanced (state Evaluate) and its x lies outside this rank's owned interval [bounds[rank], bounds[rank+1]).
__global__ void mig_classify(ParticlesDev P, const double* __restrict__ bounds, int nranks, int rank, int* dest,
                             unsigned long long* counts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    int d = -1;
    if (P.state[i] == PB_EVALUATE) {
        const double x = (double)P.x[i];
        int r = 0;
        while (r + 1 < nranks && x >= bounds[r + 1]) ++r;  // rank 0 owns (-inf, b1), the last rank [b_{n-1}, +inf)
        if (x != x) r = rank;                             // NaN stays (the kernel flags it)
        if (r != rank) d = r;
    }
    dest[i] = d;
    atomicAdd(&counts[d < 0 ? nranks : d], 1ULL);
}

// rsend (NULL: none) receives each leaver's resumable state R at the index of its record
__global__ void mig_pack(ParticlesDev P, ResumeDev R, const int* __restrict__ dest, int nranks, unsigned long long* cursors,
                         MigRecord* send, MigResume* rsend, long long* keep_idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const int d = dest[i];
    if (d < 0) {
        keep_idx[atomicAdd(&cursors[nranks], 1ULL)] = i;
    } else {
        MigRecord r;
        r.t = P.t[i]; r.pid = P.pid[i];
        r.x = P.x[i]; r.y = P.y[i]; r.z = P.z[i];
        r.dx = P.dx[i]; r.dy = P.dy[i]; r.dz = P.dz[i];
        r.state = P.state[i]; r.ei = P.ei[i];
        const unsigned long long k = atomicAdd(&cursors[d], 1ULL);
        send[k] = r;
        if (rsend) rsend[k] = MigResume{R.dt[i], R.next_dt[i], R.iters[i], 0};
    }
}

// rs / rd: the resumable state, carried when rd.dt is not NULL
__global__ void mig_compact(ParticlesDev src, ParticlesDev dst, ResumeDev rs, ResumeDev rd, const long long* __restrict__ keep_idx,
                            long long n_keep) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_keep) return;
    const long long i = keep_idx[k];
    dst.x[k] = src.x[i]; dst.y[k] = src.y[i]; dst.z[k] = src.z[i];
    dst.dx[k] = src.dx[i]; dst.dy[k] = src.dy[i]; dst.dz[k] = src.dz[i];
    dst.t[k] = src.t[i]; dst.state[k] = src.state[i]; dst.ei[k] = src.ei[i]; dst.pid[k] = src.pid[i];
    if (rd.dt) { rd.dt[k] = rs.dt[i]; rd.next_dt[k] = rs.next_dt[i]; rd.iters[k] = rs.iters[i]; }
}

__global__ void mig_unpack(ParticlesDev dst, ResumeDev rd, long long base, const MigRecord* __restrict__ recv,
                           const MigResume* __restrict__ rrecv, long long n_in) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_in) return;
    const MigRecord r = recv[k];
    const long long j = base + k;
    dst.x[j] = r.x; dst.y[j] = r.y; dst.z[j] = r.z;
    dst.dx[j] = r.dx; dst.dy[j] = r.dy; dst.dz[j] = r.dz;
    dst.t[j] = r.t; dst.state[j] = r.state; dst.ei[j] = r.ei; dst.pid[j] = r.pid;
    if (rd.dt) {
        const MigResume s = rrecv[k];
        rd.dt[j] = s.dt; rd.next_dt[j] = s.next_dt; rd.iters[j] = s.iters;
    }
}


// ------------------------------------------------------------------------------------------------
// output path (SURVEY.md 8f-2): order-preserving selection / compaction on the device.
//   SEL_OUTPUT:  ParticleFile.write's rule (reference _core/particlefile.py:198-221, `_to_write_particles`):
//                finite t and  t_out - |dt/2| <= t <= t_out + |dt/2|
//   SEL_ALIVE:   state != Delete   (Kernel.remove_deleted + ParticleSet.remove_indices, kernel.py:98-106,
//                particleset.py:247-250: np.delete keeps the storage order)
// Three passes: per-block count, one-block scan of the block counts, per-block ordered scatter of the indices.
// ------------------------------------------------------------------------------------------------
//   SEL_RESIDENT: state != PB_STATE_MIGRATED  (mode D with in-kernel migration: the record was stored in its new owner's inbox)
enum { SEL_OUTPUT = 0, SEL_ALIVE = 1, SEL_RESIDENT = 2 };
constexpr int SEL_BLOCK = 256;

struct SelectRule {
    int mode;
    double lo, hi;  // SEL_OUTPUT: t_out -/+ |dt/2|
};

__device__ __forceinline__ bool sel_flag(const ParticlesDev& P, const SelectRule& r, long long i) {
    if (r.mode == SEL_ALIVE) return P.state[i] != PB_DELETE;
    if (r.mode == SEL_RESIDENT) return P.state[i] != PB_STATE_MIGRATED;
    const double t = P.t[i];
    return isfinite(t) && r.lo <= t && r.hi >= t;
}

__global__ void __launch_bounds__(SEL_BLOCK) sel_count(ParticlesDev P, SelectRule r, unsigned int* __restrict__ block_counts) {
    const long long i = (long long)blockIdx.x * SEL_BLOCK + threadIdx.x;
    const bool f = i < P.n && sel_flag(P, r, i);
    const int c = __syncthreads_count(f);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = (unsigned)c;
}

// exclusive scan of block_counts[0..nb) in place -> block_offsets (long long); total to *total.  One block.
__global__ void __launch_bounds__(1024) sel_scan(const unsigned int* __restrict__ block_counts, long long* __restrict__ block_offsets,
                                                 long long nb, long long* total) {
    __shared__ long long warp_sums[32];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long base = 0; base < nb; base += 1024) {
        const long long i = base + threadIdx.x;
        const long long v = i < nb ? (long long)block_counts[i] : 0;
        long long incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            long long w = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long up = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += up;
            }
            warp_sums[lane] = w;  // inclusive over warps
        }
        __syncthreads();
        const long long before = carry + (warp ? warp_sums[warp - 1] : 0) + incl - v;
        if (i < nb) block_offsets[i] = before;
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(SEL_BLOCK) sel_scatter(ParticlesDev P, SelectRule r, const long long* __restrict__ block_offsets,
                                                         long long* __restrict__ idx) {
    __shared__ int warp_counts[SEL_BLOCK / 32];
    const long long i = (long long)blockIdx.x * SEL_BLOCK + threadIdx.x;
    const bool f = i < P.n && sel_flag(P, r, i);
    const unsigned ballot = __ballot_sync(0xffffffffu, f);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_counts[warp] = __popc(ballot);
    __syncthreads();
    if (f) {
        int before = __popc(ballot & ((1u << lane) - 1u));
        for (int w = 0; w < warp; ++w) before += warp_counts[w];
        idx[block_offsets[blockIdx.x] + before] = i;
    }
}

// compacted copies of the written columns (Particle variables with to_write: x, y, z, t, particle_id)
__global__ void out_gather(ParticlesDev P, const long long* __restrict__ idx, long long m, float* x, float* y, float* z, double* t,
                           long long* pid) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    const long long i = idx[k];
    if (x) x[k] = P.x[i];
    if (y) y[k] = P.y[i];
    if (z) z[k] = P.z[i];
    if (t) t[k] = P.t[i];
    if (pid) pid[k] = P.pid[i];
}

// ------------------------------------------------------------------------------------------------
// host-side engine
// ------------------------------------------------------------------------------------------------
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    int32_t ensure(size_t n) {
        if (n <= bytes) return PB_OK;
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
        CK(cudaMalloc(&p, n));
        bytes = n;
        return PB_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

// The resident particle set: one device column per pointer of ParticlesDev, in its order.  The snapshot keeps whole columns
// back to back in this order, the ids (when resident) last.
struct ParticleSoA {
    struct Column {
        size_t es;            // bytes per element
        bool zero_if_absent;  // a NULL host column uploads as zeros (dx, dy, dz)
        bool optional;        // resident only when the host passes it (particle_id)
    };
    static constexpr int NCOL = 10, PID = 9;
    static constexpr Column cols[NCOL] = {
        {4, false, false}, {4, false, false}, {4, false, false},  // x y z
        {4, true, false},  {4, true, false},  {4, true, false},   // dx dy dz
        {8, false, false}, {4, false, false}, {4, false, false},  // t state ei
        {8, false, true}};                                        // particle_id
    static_assert(offsetof(ParticlesDev, n) == NCOL * sizeof(void*), "one column per ParticlesDev pointer");
    DevBuf col[NCOL];
    // each lane's resumable state (ResumeDev: dt, next_dt, iters), resident beside the columns above while pb_engine::resume_on;
    // in the snapshot after them
    static constexpr int NRES = 3;
    static constexpr size_t res_es[NRES] = {8, 8, 4};
    static constexpr size_t res_row_bytes = 20;
    DevBuf res[NRES];
    ResumeDev resume(long long lo = 0) const {
        void* c[NRES];
        for (int k = 0; k < NRES; ++k) c[k] = res[k].p ? (char*)res[k].p + (size_t)lo * res_es[k] : nullptr;
        return ResumeDev{(double*)c[0], (double*)c[1], (int*)c[2]};
    }

    // bytes per particle of the snapshot
    static constexpr size_t row_bytes(bool with_pid) {
        size_t b = 0;
        for (const Column& c : cols)
            if (with_pid || !c.optional) b += c.es;
        return b;
    }
    // particles [lo, lo + n)
    ParticlesDev view(long long n, long long lo = 0) const {
        void* c[NCOL];
        for (int k = 0; k < NCOL; ++k) c[k] = col[k].p ? (char*)col[k].p + (size_t)lo * cols[k].es : nullptr;
        return ParticlesDev{(float*)c[0], (float*)c[1], (float*)c[2], (float*)c[3], (float*)c[4], (float*)c[5],
                            (double*)c[6], (int*)c[7], (int*)c[8], (long long*)c[9], n};
    }
};

struct pb_engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, tev0 = nullptr, tev1 = nullptr;
    // grid
    DevBuf lon, lat, depth, time, hkeys, hstarts, hcounts, hfaces, hbucket, cellproj, hqbox;
    // float64 rectilinear grids: the cell tables of lon, lat, depth, time back to back (AxisCellRec); cellp[k] NULL: none
    DevBuf cells;
    const AxisCellRec* cellp[4] = {};
    int interp = 0;  // enum pb_interp
    GridDev g{};
    long long hash_nent = 0;  // entries of the resident spatial-hash table
    bool have_grid = false;
    int coord_f64 = 0;
    // fields
    DevBuf fbuf[PB_MAX_FIELDS];       // slots 0..2: U, V, W; 3..: scalar fields (Field.eval)
    const void* fptr[PB_MAX_FIELDS] = {};
    int f_f64[PB_MAX_FIELDS] = {};
    long long fshape[PB_MAX_FIELDS][4] = {};
    // node-interleaved {u, v, w, 0} copy of U, V, W for the specialised RK4 kernel (afast.cu); rebuilt when a component changes
    DevBuf il;
    bool il_valid = false;
    int last_variant = 0;  // kernel family of the last advect launch: 0 generic, 1 specialised RK4 (afast.cu)
    // time-slab streaming: ring of (window + 1) levels per windowed slot, loads on a dedicated copy stream; one window for all
    int ring = 0;                    // 0: every level resident
    bool fwin[PB_MAX_FIELDS] = {};   // the slot holds a ring of levels (pb_field_window_create), not the whole field
    long long win_first = 0, win_n = 0;
    cudaStream_t copy_stream = nullptr;
    // pb_advect_host: one in-order stream per chunk slot (H2D -> kernel -> D2H), created on first use
    static constexpr int PIPE = 4;
    cudaStream_t pipe_stream[PIPE] = {};
    cudaEvent_t pipe_done[PIPE] = {};
    cudaEvent_t pipe_fork = nullptr;
    cudaEvent_t copy_done = nullptr;
    std::vector<double> time_host;   // seconds since the interval start
    // particles
    ParticleSoA cur;
    DevBuf snap;  // snapshot of all particle arrays
    long long snap_n = -1;  // particle count the snapshot was taken at (-1: none); a new upload / compaction invalidates it
    bool snap_pid = false;  // the snapshot holds the particle ids too
    bool resume_on = false;    // the resumable-state columns (ParticleSoA::res) are resident (pb_particles_upload_resume)
    bool snap_resume = false;  // the snapshot holds them too
    // alternate SoA for compaction and migration (rebuild_resident); mode D (domain decomposition) migration work buffers
    ParticleSoA alt;
    DevBuf mdest, mkeep, mcount, mbounds;
    // output path: block counts / offsets of the ordered selection, selected indices, compacted columns
    DevBuf sblock, soffs, sidx, sout;
    DevBuf samp_d, samp_i;  // scratch of pb_sample_velocity / pb_sample_scalar (grown on demand, reused across calls)
    DevBuf ad_iters;        // time-slab streaming: pb_advect_diffusion's per-particle iteration counts across resumed launches
    long long* h_sel_total = nullptr;  // pinned
    long long n_selected = -1;
    // in-kernel migration over peer memory: own inbox allocation, every rank's inbox as mapped here, the slot of this round
    unsigned char* mig_base = nullptr;
    unsigned char* mig_peer[PB_MIG_MAX_RANKS] = {};
    bool mig_ipc_opened[PB_MIG_MAX_RANKS] = {};
    long long mig_cap = 0;
    int mig_slot = 0;
    bool mig_on = false;
    unsigned long long* h_mig_count = nullptr;  // pinned
    int nranks = 1, rank = 0;
    long long n_keep = 0, n_send = 0;
    std::vector<long long> send_counts;
    long long n = 0;
    bool have_pid = false;
    // report
    ReportDev* d_rep = nullptr;
    ReportDev* h_rep = nullptr;  // pinned
    pb_report last{};
    bool pending = false;
};

// The bracket of an advect call's launches: a zeroed report and ev0 before them, ev1 and the report's copy back after them;
// pb_last_report waits for both.
static int32_t begin_launch(pb_engine* e) {
    ReportDev& r = *e->h_rep;
    memset(&r, 0, sizeof(r));
    r.first_error_iter = LLONG_MAX;
    r.wait_t_min_bits = ~0ULL;
    CK(cudaMemcpyAsync(e->d_rep, e->h_rep, sizeof(ReportDev), cudaMemcpyHostToDevice, e->stream));
    CK(cudaEventRecord(e->ev0, e->stream));
    return PB_OK;
}

static int32_t end_launch(pb_engine* e) {
    CK(cudaEventRecord(e->ev1, e->stream));
    CK(cudaMemcpyAsync(e->h_rep, e->d_rep, sizeof(ReportDev), cudaMemcpyDeviceToHost, e->stream));
    e->pending = true;
    return PB_OK;
}

// host-side column passes (pb_host_*): a column split over a few C++ threads
#ifndef PB_HOSTSIM
#include <thread>
template <class F>
static void host_parallel(int64_t n, F&& f) {
    // a few threads saturate one socket's memory channels; small columns are not worth a thread start (~20 us each)
    int nt = (int)std::min<int64_t>(8, std::max<int64_t>(1, n / (1 << 19)));
    const unsigned hc = std::thread::hardware_concurrency();
    if (hc && (unsigned)nt > hc) nt = (int)hc;
    if (nt <= 1) { f(0, 0, n); return; }
    std::vector<std::thread> th;
    const int64_t per = (n + nt - 1) / nt;
    for (int k = 1; k < nt; ++k) th.emplace_back([=, &f] { f(k, std::min<int64_t>(n, k * per), std::min<int64_t>(n, (k + 1) * per)); });
    f(0, 0, std::min<int64_t>(n, per));
    for (auto& t : th) t.join();
}
#else
template <class F>
static void host_parallel(int64_t n, F&& f) { f(0, 0, n); }
#endif


extern "C" {

int32_t pb_abi_version(void) { return PB_ABI_VERSION; }
const char* pb_last_error_string(void) { return g_err.c_str(); }

int32_t pb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int32_t pb_engine_create(int32_t device, pb_engine** out) {
    if (!out) return fail(PB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    int n = pb_device_count();
    if (n <= 0) return fail(PB_ERR_NO_DEVICE, "no CUDA device visible: parcels_b200 has no CPU fallback");
    if (device < 0 || device >= n) return fail(PB_ERR_INVALID, "device %d out of range (0..%d)", device, n - 1);
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)  // sm_90a code loads on compute capability 9.0 only
        return fail(PB_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    pb_engine* e = new pb_engine();
    e->device = device;
    CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&e->ev0));
    CK(cudaEventCreate(&e->ev1));
    CK(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&e->copy_done, cudaEventDisableTiming));
    CK(cudaEventCreate(&e->tev0));
    CK(cudaEventCreate(&e->tev1));
    CK(cudaMalloc(&e->d_rep, sizeof(ReportDev)));
    CK(cudaMallocHost(&e->h_rep, sizeof(ReportDev)));
    CK(cudaMallocHost(&e->h_sel_total, sizeof(long long)));
    *out = e;
    return PB_OK;
}

void pb_engine_destroy(pb_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    for (ParticleSoA* s : {&e->cur, &e->alt}) {
        for (DevBuf& b : s->col) b.release();
        for (DevBuf& b : s->res) b.release();
    }
    for (DevBuf& b : e->fbuf) b.release();
    e->il.release();
    for (DevBuf* b : {&e->mdest, &e->mkeep, &e->mcount, &e->mbounds, &e->hqbox, &e->hbucket, &e->cellproj, &e->hkeys, &e->hstarts,
                      &e->hcounts, &e->hfaces, &e->lon, &e->lat, &e->depth, &e->time, &e->cells, &e->snap, &e->sblock, &e->soffs, &e->sidx,
                      &e->sout, &e->samp_d, &e->samp_i, &e->ad_iters})
        b->release();
    for (int r = 0; r < PB_MIG_MAX_RANKS; ++r)
        if (e->mig_ipc_opened[r]) cudaIpcCloseMemHandle(e->mig_peer[r]);
    if (e->mig_base) cudaFree(e->mig_base);
    if (e->h_mig_count) cudaFreeHost(e->h_mig_count);
    if (e->d_rep) cudaFree(e->d_rep);
    if (e->h_rep) cudaFreeHost(e->h_rep);
    if (e->h_sel_total) cudaFreeHost(e->h_sel_total);
    cudaEventDestroy(e->ev0);
    cudaEventDestroy(e->ev1);
    cudaStreamDestroy(e->copy_stream);
    for (int k = 0; k < pb_engine::PIPE; ++k) {
        if (e->pipe_stream[k]) cudaStreamDestroy(e->pipe_stream[k]);
        if (e->pipe_done[k]) cudaEventDestroy(e->pipe_done[k]);
    }
    if (e->pipe_fork) cudaEventDestroy(e->pipe_fork);
    cudaEventDestroy(e->copy_done);
    cudaEventDestroy(e->tev0);
    cudaEventDestroy(e->tev1);
    cudaStreamDestroy(e->stream);
    delete e;
}

int32_t pb_engine_synchronize(pb_engine* e) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_timer_begin(pb_engine* e) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    CK(cudaSetDevice(e->device));
    CK(cudaEventRecord(e->tev0, e->stream));
    return PB_OK;
}

int32_t pb_timer_end_ms(pb_engine* e, float* ms) {
    if (!e || !ms) return fail(PB_ERR_INVALID, "NULL argument");
    CK(cudaSetDevice(e->device));
    CK(cudaEventRecord(e->tev1, e->stream));
    CK(cudaEventSynchronize(e->tev1));
    CK(cudaEventElapsedTime(ms, e->tev0, e->tev1));
    return PB_OK;
}

static int32_t upload(pb_engine* e, DevBuf& b, const void* src, size_t bytes) {
    int32_t rc = b.ensure(bytes ? bytes : 1);
    if (rc) return rc;
    if (bytes) CK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, e->stream));
    return PB_OK;
}

// depth + time axes and the scalar grid description shared by both grid kinds
static int32_t upload_zt(pb_engine* e, const void* depth, int64_t nz, int32_t coord_is_f64, const double* time_s, int64_t nt,
                         int32_t spherical, double deg2m, int64_t xdim_cells, int64_t ydim_cells, int64_t zdim_cells) {
    const size_t es = coord_is_f64 ? 8 : 4;
    int32_t rc;
    if (!depth) nz = 0;
    if ((rc = upload(e, e->depth, depth, nz * es))) return rc;
    std::vector<double> tnorm;
    if (!time_s || nt < 2) nt = 0;
    if (nt) {  // seconds since the interval start (index_search.py:88)
        tnorm.resize(nt);
        for (int64_t k = 0; k < nt; ++k) tnorm[k] = time_s[k] - time_s[0];
        for (int64_t k = 1; k < nt; ++k)
            if (!(tnorm[k] > tnorm[k - 1])) return fail(PB_ERR_INVALID, "time axis must be strictly increasing");
    }
    if ((rc = upload(e, e->time, tnorm.data(), nt * sizeof(double)))) return rc;
    CK(cudaStreamSynchronize(e->stream));  // tnorm goes out of scope
    GridDev& g = e->g;
    g.lon = e->lon.p; g.lat = e->lat.p; g.depth = nz ? e->depth.p : nullptr;
    g.time = nt ? (const double*)e->time.p : nullptr;
    g.nz = (int)nz; g.nt = (int)nt;
    g.spherical = spherical ? 1 : 0;
    g.deg2m = spherical ? deg2m : 1.0;
    g.inv_deg2m = 1.0 / g.deg2m;  // correctly rounded (host division): div_by_cached in afast.cu
    g.time_len = nt ? tnorm[nt - 1] : 0.0;
    e->time_host = tnorm;
    g.xdim = xdim_cells; g.ydim = ydim_cells; g.zdim = zdim_cells;
    e->coord_f64 = coord_is_f64 ? 1 : 0;
    e->have_grid = true;
    return PB_OK;
}

// the cell tables of a float64 rectilinear grid (AxisCellRec), from the axes just uploaded
static int32_t build_axis_cells(pb_engine* e) {
    for (const AxisCellRec*& c : e->cellp) c = nullptr;
    if (!e->coord_f64 || e->g.curvilinear) return PB_OK;
    const GridDev& g = e->g;
    const double* axes[4] = {(const double*)g.lon, (const double*)g.lat, (const double*)g.depth, g.time};
    const int n[4] = {g.nx, g.ny, g.nz, g.nt};
    size_t off[4], recs = 0;
    for (int k = 0; k < 4; ++k) {
        off[k] = recs;
        if (axes[k] && n[k] >= 2) recs += (size_t)n[k] - 1;
    }
    if (!recs) return PB_OK;
    int32_t rc = e->cells.ensure(recs * sizeof(AxisCellRec));
    if (rc) return rc;
    for (int k = 0; k < 4; ++k) {
        if (!axes[k] || n[k] < 2) continue;
        AxisCellRec* out = (AxisCellRec*)e->cells.p + off[k];
        cudaError_t ce = launch_axis_cells(axes[k], n[k], out, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "axis_cells_kernel launch failed: %s", cudaGetErrorString(ce));
        e->cellp[k] = out;
    }
    return PB_OK;
}

int32_t pb_grid_upload_rectilinear(pb_engine* e, const void* lon, int64_t nx, const void* lat, int64_t ny,
                                   const void* depth, int64_t nz, int32_t coord_is_f64, const double* time_s,
                                   int64_t nt, int32_t spherical, double deg2m, int64_t xdim_cells,
                                   int64_t ydim_cells, int64_t zdim_cells) {
    PB_RANGE("pb_grid_upload_rectilinear");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    // a length-1 axis is allowed: the 1-D search returns index 0, coordinate 0 there (index_search.py:45-46)
    if (!lon || !lat || nx < 1 || ny < 1)
        return fail(PB_ERR_INVALID, "rectilinear grid needs lon and lat nodes (got nx=%lld ny=%lld)", (long long)nx, (long long)ny);
    if (nx > INT_MAX || ny > INT_MAX || nz > INT_MAX || nt > INT_MAX) return fail(PB_ERR_INVALID, "axis too long");
    CK(cudaSetDevice(e->device));
    const size_t es = coord_is_f64 ? 8 : 4;
    int32_t rc;
    if ((rc = upload(e, e->lon, lon, nx * es))) return rc;
    if ((rc = upload(e, e->lat, lat, ny * es))) return rc;
    e->g.nx = (int)nx; e->g.ny = (int)ny;
    e->g.curvilinear = 0;
    e->g.hkeys = nullptr; e->g.hstarts = nullptr; e->g.hcounts = nullptr; e->g.hfaces = nullptr; e->g.hnkeys = 0;
    e->g.hbucket = nullptr; e->g.cellproj = nullptr; e->g.hqbox = nullptr;
    if ((rc = upload_zt(e, depth, nz, coord_is_f64, time_s, nt, spherical, deg2m, xdim_cells, ydim_cells, zdim_cells))) return rc;
    return build_axis_cells(e);
}

int32_t pb_grid_upload_curvilinear(pb_engine* e, const void* lon2d, const void* lat2d, int64_t ny, int64_t nx,
                                   const void* depth, int64_t nz, int32_t coord_is_f64, const double* time_s, int64_t nt,
                                   int32_t spherical, double deg2m, int64_t xdim_cells, int64_t ydim_cells,
                                   int64_t zdim_cells, const uint32_t* hash_keys, const int64_t* hash_starts,
                                   const int64_t* hash_counts, int64_t n_keys, const uint32_t* hash_faces,
                                   int64_t n_entries, const double* hash_box6, int32_t hash_bitwidth,
                                   const uint64_t* face_qbox) {
    PB_RANGE("pb_grid_upload_curvilinear");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!lon2d || !lat2d || nx < 2 || ny < 2) return fail(PB_ERR_INVALID, "curvilinear grid needs (ny, nx) lon/lat with ny, nx >= 2");
    if (nx > INT_MAX || ny > INT_MAX || nz > INT_MAX || nt > INT_MAX) return fail(PB_ERR_INVALID, "axis too long");
    const bool host_table = hash_keys || hash_starts || hash_counts || hash_faces;
    if (!hash_box6 || !face_qbox) return fail(PB_ERR_INVALID, "curvilinear grid needs its hash box and per-face quantised boxes");
    if (host_table && (!hash_keys || !hash_starts || !hash_counts || !hash_faces || n_keys < 1 || n_entries < 1))
        return fail(PB_ERR_INVALID, "incomplete host-built spatial-hash table (pass all four arrays, or none to build it on the device)");
    if (hash_bitwidth < 1 || hash_bitwidth > 1023) return fail(PB_ERR_INVALID, "hash bitwidth must be in 1..1023");
    CK(cudaSetDevice(e->device));
    const size_t es = coord_is_f64 ? 8 : 4;
    const int bucket_bits = 20;  // bucket table over the top bits of the 30-bit Morton key: narrows the binary search to a few keys
    int32_t rc;
    if ((rc = upload(e, e->lon, lon2d, (size_t)nx * ny * es))) return rc;
    if ((rc = upload(e, e->lat, lat2d, (size_t)nx * ny * es))) return rc;
    if ((rc = upload(e, e->hqbox, face_qbox, (size_t)(ny - 1) * (nx - 1) * 8))) return rc;
    GridDev& g = e->g;
    if (host_table) {
        if ((rc = upload(e, e->hkeys, hash_keys, n_keys * 4))) return rc;
        if ((rc = upload(e, e->hstarts, hash_starts, n_keys * 8))) return rc;
        if ((rc = upload(e, e->hcounts, hash_counts, n_keys * 8))) return rc;
        if ((rc = upload(e, e->hfaces, hash_faces, n_entries * 4))) return rc;
        const int shift = 30 - bucket_bits;
        const long long nb = 1LL << bucket_bits;
        std::vector<int> bucket(nb + 1);
        long long k = 0;
        for (long long b = 0; b <= nb; ++b) {
            while (k < n_keys && (long long)(hash_keys[k] >> shift) < b) ++k;
            bucket[b] = (int)k;
        }
        if ((rc = upload(e, e->hbucket, bucket.data(), (size_t)(nb + 1) * sizeof(int)))) return rc;
        CK(cudaStreamSynchronize(e->stream));
    } else {
        // the table is a pure integer function of the quantised boxes: expanded, sorted and compressed on the device
        HashTableDev t;
        cudaError_t ce = build_hash_table_device((const unsigned long long*)e->hqbox.p, (long long)(ny - 1) * (nx - 1), bucket_bits, t, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "device spatial-hash build failed: %s", cudaGetErrorString(ce));
        n_keys = t.nkeys; n_entries = t.nent;
        e->hkeys.release(); e->hkeys.p = t.keys; e->hkeys.bytes = (size_t)n_keys * 4;
        e->hstarts.release(); e->hstarts.p = t.starts; e->hstarts.bytes = (size_t)n_keys * 8;
        e->hcounts.release(); e->hcounts.p = t.counts; e->hcounts.bytes = (size_t)n_keys * 8;
        e->hfaces.release(); e->hfaces.p = t.faces; e->hfaces.bytes = (size_t)n_entries * 4;
        e->hbucket.release(); e->hbucket.p = t.bucket; e->hbucket.bytes = (size_t)((1LL << bucket_bits) + 1) * 4;
    }
    e->hash_nent = n_entries;
    g.nx = (int)nx; g.ny = (int)ny;
    g.curvilinear = 1;
    for (const AxisCellRec*& c : e->cellp) c = nullptr;  // (the tables of a rectilinear grid uploaded before)
    g.hash_bitwidth = hash_bitwidth;
    g.hkeys = (const unsigned int*)e->hkeys.p;
    g.hstarts = (const long long*)e->hstarts.p;
    g.hcounts = (const long long*)e->hcounts.p;
    g.hfaces = (const unsigned int*)e->hfaces.p;
    g.hnkeys = n_keys;
    g.hqbox = (const unsigned long long*)e->hqbox.p;
    for (int k = 0; k < 6; ++k) g.hbox[k] = hash_box6[k];
    g.hbucket = (const int*)e->hbucket.p;
    g.hbucket_shift = 30 - bucket_bits;
    g.cellproj = nullptr;
    if (spherical) {  // per-cell tangent-plane projections, computed once on the device
        const size_t ncell = (size_t)(ny - 1) * (nx - 1);
        if ((rc = e->cellproj.ensure(ncell * 16 * sizeof(double)))) return rc;
        cudaError_t ce = launch_precompute_cells(e->lon.p, e->lat.p, (int)ny, (int)nx, coord_is_f64 != 0, (double*)e->cellproj.p, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "precompute_cells launch failed: %s", cudaGetErrorString(ce));
        g.cellproj = (const double*)e->cellproj.p;
    }
    return upload_zt(e, depth, nz, coord_is_f64, time_s, nt, spherical, deg2m, xdim_cells, ydim_cells, zdim_cells);
}

int32_t pb_hash_table_size(pb_engine* e, int64_t* n_keys, int64_t* n_entries) {
    if (!e || !n_keys || !n_entries) return fail(PB_ERR_INVALID, "NULL argument");
    if (!e->g.curvilinear) return fail(PB_ERR_STATE, "no curvilinear grid uploaded");
    *n_keys = e->g.hnkeys;
    *n_entries = e->hash_nent;
    return PB_OK;
}

int32_t pb_hash_table_download(pb_engine* e, uint32_t* keys, int64_t* starts, int64_t* counts, uint32_t* faces) {
    if (!e || !keys || !starts || !counts || !faces) return fail(PB_ERR_INVALID, "NULL argument");
    if (!e->g.curvilinear) return fail(PB_ERR_STATE, "no curvilinear grid uploaded");
    CK(cudaSetDevice(e->device));
    const size_t nk = (size_t)e->g.hnkeys, ne = (size_t)e->hash_nent;
    CK(cudaMemcpyAsync(keys, e->hkeys.p, nk * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(starts, e->hstarts.p, nk * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(counts, e->hcounts.p, nk * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(faces, e->hfaces.p, ne * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

// kernel family of aslip.cu: 1 = _Spatialslip, 2 = nearest node; 0 = not an alternative A-grid interpolator
static int agrid_alt_mode(int interp) {
    if (interp == PB_INTERP_XFREESLIP || interp == PB_INTERP_XPARTIALSLIP) return 1;
    return interp == PB_INTERP_XNEAREST_VELOCITY ? 2 : 0;
}

int32_t pb_set_interpolation(pb_engine* e, int32_t method, int32_t off_x, int32_t off_y, int32_t off_z) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (method < PB_INTERP_XLINEAR_VELOCITY || method > PB_INTERP_XNEAREST_VELOCITY) return fail(PB_ERR_INVALID, "unknown interpolation %d", method);
    if ((off_x | off_y | off_z) & ~1) return fail(PB_ERR_INVALID, "staggering offsets must be 0 or 1");
    e->interp = method;
    e->g.off_x = off_x; e->g.off_y = off_y; e->g.off_z = off_z;
    // _Spatialslip(a, b): XFreeslip (1, 0), XPartialslip (0.5, 0.5)  (_xinterpolators.py:483-506)
    e->g.slip_a = method == PB_INTERP_XPARTIALSLIP ? 0.5f : 1.0f;
    e->g.slip_b = method == PB_INTERP_XPARTIALSLIP ? 0.5f : 0.0f;
    return PB_OK;
}

static int32_t set_field(pb_engine* e, int32_t slot, const void* dev, int32_t is_f64, int64_t T, int64_t Z, int64_t Y, int64_t X) {
    e->fptr[slot] = dev;
    e->fwin[slot] = false;
    if (slot < 3) e->il_valid = false;
    e->f_f64[slot] = is_f64 ? 1 : 0;
    e->fshape[slot][0] = T; e->fshape[slot][1] = Z; e->fshape[slot][2] = Y; e->fshape[slot][3] = X;
    return PB_OK;
}

int32_t pb_field_upload(pb_engine* e, int32_t slot, const void* data, int32_t data_is_f64, int64_t T, int64_t Z,
                        int64_t Y, int64_t X) {
    PB_RANGE("pb_field_upload");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (slot < 0 || slot >= PB_MAX_FIELDS) return fail(PB_ERR_INVALID, "bad field slot %d", slot);
    if (!data || T < 1 || Z < 1 || Y < 1 || X < 1) return fail(PB_ERR_INVALID, "bad field shape");
    if (T > INT_MAX || Z > INT_MAX || Y > INT_MAX || X > INT_MAX) return fail(PB_ERR_INVALID, "field dim too long");
    CK(cudaSetDevice(e->device));
    const size_t bytes = (size_t)T * Z * Y * X * (data_is_f64 ? 8 : 4);
    int32_t rc = upload(e, e->fbuf[slot], data, bytes);
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->stream));
    return set_field(e, slot, e->fbuf[slot].p, data_is_f64, T, Z, Y, X);
}

int32_t pb_field_attach_device(pb_engine* e, int32_t slot, const void* dev_data, int32_t data_is_f64, int64_t T,
                               int64_t Z, int64_t Y, int64_t X) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (slot < 0 || slot >= PB_MAX_FIELDS) return fail(PB_ERR_INVALID, "bad field slot %d", slot);
    if (!dev_data || T < 1 || Z < 1 || Y < 1 || X < 1) return fail(PB_ERR_INVALID, "bad field shape");
    if (T > INT_MAX || Z > INT_MAX || Y > INT_MAX || X > INT_MAX) return fail(PB_ERR_INVALID, "field dim too long");
    e->fbuf[slot].release();
    return set_field(e, slot, dev_data, data_is_f64, T, Z, Y, X);
}

int32_t pb_field_clear(pb_engine* e, int32_t slot) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (slot < 0 || slot >= PB_MAX_FIELDS) return fail(PB_ERR_INVALID, "bad field slot %d", slot);
    e->fbuf[slot].release();
    e->fptr[slot] = nullptr;
    e->fwin[slot] = false;
    if (slot < 3) e->il_valid = false;
    return PB_OK;
}

int32_t pb_particles_upload(pb_engine* e, int64_t n, const float* x, const float* y, const float* z, const float* dx,
                            const float* dy, const float* dz, const double* t, const int32_t* state, const int32_t* ei,
                            const int64_t* particle_id) {
    PB_RANGE("pb_particles_upload");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (n < 0) return fail(PB_ERR_INVALID, "n < 0");
    if (n && (!x || !y || !z || !t || !state || !ei)) return fail(PB_ERR_INVALID, "NULL particle array");
    CK(cudaSetDevice(e->device));
    const void* src[ParticleSoA::NCOL] = {x, y, z, dx, dy, dz, t, state, ei, particle_id};
    e->have_pid = particle_id != nullptr;
    for (int k = 0; k < ParticleSoA::NCOL; ++k) {
        const ParticleSoA::Column& c = ParticleSoA::cols[k];
        if (c.optional && !src[k]) continue;
        DevBuf& b = e->cur.col[k];
        int32_t rc = b.ensure(n ? n * c.es : 1);
        if (rc) return rc;
        if (!n) continue;
        if (src[k]) CK(cudaMemcpyAsync(b.p, src[k], n * c.es, cudaMemcpyHostToDevice, e->stream));
        else if (c.zero_if_absent) CK(cudaMemsetAsync(b.p, 0, n * c.es, e->stream));
    }
    e->n = n;
    e->snap_n = -1;
    e->resume_on = false;  // (a new set: pb_particles_upload_resume gives it resumable state)
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_particles_upload_resume(pb_engine* e, int64_t n, const double* dt, const double* next_dt, const int32_t* iters) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (n != e->n) return fail(PB_ERR_INVALID, "resumable state of %lld particles but %lld are resident", (long long)n, (long long)e->n);
    CK(cudaSetDevice(e->device));
    const void* src[ParticleSoA::NRES] = {dt, next_dt, iters};
    for (int k = 0; k < ParticleSoA::NRES; ++k) {
        const size_t bytes = (size_t)n * ParticleSoA::res_es[k];
        int32_t rc = e->cur.res[k].ensure(n ? bytes : 1);
        if (rc) return rc;
        if (!n) continue;
        if (src[k]) CK(cudaMemcpyAsync(e->cur.res[k].p, src[k], bytes, cudaMemcpyHostToDevice, e->stream));
        else CK(cudaMemsetAsync(e->cur.res[k].p, 0, bytes, e->stream));
    }
    CK(cudaStreamSynchronize(e->stream));
    e->resume_on = true;
    return PB_OK;
}

int32_t pb_particles_download_resume(pb_engine* e, int64_t n, double* dt, double* next_dt, int32_t* iters) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!e->resume_on) return fail(PB_ERR_STATE, "no resumable state resident (pb_particles_upload_resume)");
    if (n != e->n) return fail(PB_ERR_INVALID, "download of %lld particles but %lld are resident", (long long)n, (long long)e->n);
    CK(cudaSetDevice(e->device));
    void* dst[ParticleSoA::NRES] = {dt, next_dt, iters};
    for (int k = 0; k < ParticleSoA::NRES; ++k)
        if (dst[k] && n) CK(cudaMemcpyAsync(dst[k], e->cur.res[k].p, (size_t)n * ParticleSoA::res_es[k], cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_particles_download(pb_engine* e, int64_t n, float* x, float* y, float* z, float* dx, float* dy, float* dz,
                              double* t, int32_t* state, int32_t* ei) {
    PB_RANGE("pb_particles_download");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (n != e->n) return fail(PB_ERR_INVALID, "download of %lld particles but %lld are resident", (long long)n, (long long)e->n);
    CK(cudaSetDevice(e->device));
    void* dst[ParticleSoA::PID] = {x, y, z, dx, dy, dz, t, state, ei};  // (the ids: pb_particles_download_ids)
    for (int k = 0; k < ParticleSoA::PID; ++k)
        if (dst[k] && n) CK(cudaMemcpyAsync(dst[k], e->cur.col[k].p, n * ParticleSoA::cols[k].es, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_particles_download_ids(pb_engine* e, int64_t n, int64_t* particle_id) {
    if (!e || (n && !particle_id)) return fail(PB_ERR_INVALID, "NULL argument");
    if (n != e->n) return fail(PB_ERR_INVALID, "download of %lld ids but %lld particles are resident", (long long)n, (long long)e->n);
    if (!e->have_pid && n) return fail(PB_ERR_STATE, "no particle ids resident");
    CK(cudaSetDevice(e->device));
    if (n) CK(cudaMemcpyAsync(particle_id, e->cur.col[ParticleSoA::PID].p, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

// Snapshot layout: whole columns back to back in ParticleSoA order, at offsets that are multiples of the particle count AT
// SNAPSHOT TIME; particle_id (last) only when ids are resident.
int32_t pb_particles_snapshot(pb_engine* e) {
    PB_RANGE("pb_particles_snapshot");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    CK(cudaSetDevice(e->device));
    const size_t n = (size_t)e->n;
    int32_t rc = e->snap.ensure(n ? n * (ParticleSoA::row_bytes(true) + (e->resume_on ? ParticleSoA::res_row_bytes : 0)) : 1);
    if (rc) return rc;
    size_t off = 0;
    for (int k = 0; k < ParticleSoA::NCOL; ++k) {
        const ParticleSoA::Column& c = ParticleSoA::cols[k];
        if (c.optional && !e->have_pid) continue;
        if (n) CK(cudaMemcpyAsync((char*)e->snap.p + off, e->cur.col[k].p, n * c.es, cudaMemcpyDeviceToDevice, e->stream));
        off += n * c.es;
    }
    for (int k = 0; e->resume_on && k < ParticleSoA::NRES; ++k) {
        if (n) CK(cudaMemcpyAsync((char*)e->snap.p + off, e->cur.res[k].p, n * ParticleSoA::res_es[k], cudaMemcpyDeviceToDevice, e->stream));
        off += n * ParticleSoA::res_es[k];
    }
    e->snap_n = (long long)n;
    e->snap_pid = e->have_pid;
    e->snap_resume = e->resume_on;
    return PB_OK;
}

// Restores the resident set to the snapshot: columns AND particle count (a domain-decomposed pass changes the count through
// migration; the ids travel with the particles and come back with the snapshot).
int32_t pb_particles_restore(pb_engine* e) {
    PB_RANGE("pb_particles_restore");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    CK(cudaSetDevice(e->device));
    if (e->snap_n < 0 ||
        e->snap.bytes < (size_t)e->snap_n * (ParticleSoA::row_bytes(e->snap_pid) + (e->snap_resume ? ParticleSoA::res_row_bytes : 0)))
        return fail(PB_ERR_STATE, "no snapshot of the resident set to restore (the set was replaced or compacted since pb_particles_snapshot)");
    const size_t n = (size_t)e->snap_n;  // (stream-ordered after a pending advect launch: restore + launch sequences need no host sync)
    if (e->snap_n != e->n && !e->snap_pid)
        return fail(PB_ERR_STATE, "snapshot of %lld particles without ids cannot replace %lld resident ones", e->snap_n, (long long)e->n);
    size_t off = 0;
    for (int k = 0; k < ParticleSoA::NCOL; ++k) {
        const ParticleSoA::Column& c = ParticleSoA::cols[k];
        if (c.optional && !e->snap_pid) continue;
        DevBuf& b = e->cur.col[k];
        int32_t rc = b.ensure(n ? n * c.es : 1);  // (after a migration the current buffers may be the smaller alternates)
        if (rc) return rc;
        if (n) CK(cudaMemcpyAsync(b.p, (char*)e->snap.p + off, n * c.es, cudaMemcpyDeviceToDevice, e->stream));
        off += n * c.es;
    }
    for (int k = 0; e->snap_resume && k < ParticleSoA::NRES; ++k) {
        DevBuf& b = e->cur.res[k];
        int32_t rc = b.ensure(n ? n * ParticleSoA::res_es[k] : 1);
        if (rc) return rc;
        if (n) CK(cudaMemcpyAsync(b.p, (char*)e->snap.p + off, n * ParticleSoA::res_es[k], cudaMemcpyDeviceToDevice, e->stream));
        off += n * ParticleSoA::res_es[k];
    }
    e->resume_on = e->snap_resume;
    if (e->snap_pid) e->have_pid = true;
    e->n = (long long)n;
    return PB_OK;
}

int64_t pb_particles_count(pb_engine* e) { return e ? e->n : -1; }

static bool uvw_windowed(const pb_engine* e) { return e->fwin[0] || e->fwin[1] || e->fwin[2]; }

// the time levels a FieldDev can read: its ring and the sample times the resident window covers, or every level
static void set_window_desc(const pb_engine* e, bool windowed, long long T, FieldDev& f) {
    f.ring = windowed ? e->ring : (int)T;
    f.windowed = windowed ? 1 : 0;
    f.win_t0 = 0.0; f.win_t1 = 0.0;
    if (windowed && e->win_n > 0 && !e->time_host.empty()) {
        f.win_t0 = e->time_host[e->win_first];
        f.win_t1 = e->time_host[e->win_first + e->win_n - 1];
    }
}

static void fill_field_desc(pb_engine* e, FieldDev& f) {
    const long long T = e->fshape[0][0], Z = e->fshape[0][1], Y = e->fshape[0][2], X = e->fshape[0][3];
    for (int c = 0; c < 3; ++c) f.p[c] = e->fptr[c];
    f.T = (int)T; f.Z = (int)Z; f.Y = (int)Y; f.X = (int)X;
    f.sX = X > 1 ? 1 : 0;
    f.sY = Y > 1 ? X : 0;
    f.sZ = Z > 1 ? X * Y : 0;
    f.sT = T > 1 ? X * Y * Z : 0;
    set_window_desc(e, uvw_windowed(e), T, f);
    f.il = (e->il_valid && !e->ring) ? e->il.p : nullptr;
}

// A sampling call on windowed slots: a finite sample time inside the time axis needs its levels resident (outside the axis is
// OutsideTimeInterval and reads nothing); otherwise its ring slot may hold another level
static int32_t check_resident_times(pb_engine* e, int64_t n, const double* t) {
    if (e->time_host.empty()) return PB_OK;
    const double ax0 = e->time_host.front(), ax1 = e->time_host.back();
    const double w0 = e->win_n > 0 ? e->time_host[e->win_first] : 0.0;
    const double w1 = e->win_n > 0 ? e->time_host[e->win_first + e->win_n - 1] : -1.0;
    double lo = HUGE_VAL, hi = -HUGE_VAL;
    for (int64_t k = 0; k < n; ++k)
        if (t[k] >= ax0 && t[k] <= ax1) { lo = t[k] < lo ? t[k] : lo; hi = t[k] > hi ? t[k] : hi; }
    if (lo <= hi && !(lo >= w0 && hi <= w1))
        return fail(PB_ERR_INVALID, "sample times [%.17g, %.17g] are not all inside the resident time levels [%.17g, %.17g]: "
                                    "pb_field_window_set first", lo, hi, w0, w1);
    return PB_OK;
}

// FieldDev of the field in one slot (p[0] only; every level resident, or the ring of a windowed slot), its shape validated
// against the grid
static int32_t field_slot_desc(pb_engine* e, int32_t slot, FieldDev& f) {
    const long long T = e->fshape[slot][0], Z = e->fshape[slot][1], Y = e->fshape[slot][2], X = e->fshape[slot][3];
    if ((X > 1 && X != e->g.nx) || (Y > 1 && Y != e->g.ny) || (Z > 1 && e->g.nz > 0 && Z != e->g.nz) || (T > 1 && T != e->g.nt))
        return fail(PB_ERR_INVALID, "field shape (%lld,%lld,%lld,%lld) does not match grid nodes (nt=%d nz=%d ny=%d nx=%d)", T, Z, Y, X,
                    e->g.nt, e->g.nz, e->g.ny, e->g.nx);
    if (Z > 1 && e->g.nz == 0) return fail(PB_ERR_INVALID, "field has a depth dimension but the grid has no Z axis");
    f = FieldDev{};
    f.p[0] = e->fptr[slot];
    f.T = (int)T; f.Z = (int)Z; f.Y = (int)Y; f.X = (int)X;
    f.sX = X > 1 ? 1 : 0; f.sY = Y > 1 ? X : 0; f.sZ = Z > 1 ? X * Y : 0; f.sT = T > 1 ? X * Y * Z : 0;
    set_window_desc(e, e->fwin[slot], T, f);
    return PB_OK;
}


// Column slabs (pb_decomp_set_columns): the grid is global, the fields hold a column slab.  Only the column-slab instantiations of
// the advection kernels (CurvPolicy with CURV_COLUMNS) shift the found global column into the slab and test the halo; the sampling
// kernels would read the slab at global columns, past its end, so sampling is refused on such an engine.
static bool on_columns(const pb_engine* e) { return e->g.curvilinear && e->g.decomposed; }
static const char* const COLUMNS_NO_SAMPLING =
    "field sampling is not available on a column slab of a curvilinear grid (mode D): sample the undecomposed FieldSet";

// validation shared by pb_advect and pb_sample_velocity; nc = 2 (UV) or 3 (UVW)
static int32_t check_fields(pb_engine* e, int nc) {
    if (!e->have_grid) return fail(PB_ERR_STATE, "grid not uploaded (pb_grid_upload_*)");
    if (!e->fptr[0] || !e->fptr[1]) return fail(PB_ERR_STATE, "U and V not uploaded");
    if (nc == 3 && !e->fptr[2]) return fail(PB_ERR_STATE, "3-D evaluation needs a W field (fieldset.UVW)");
    for (int c = 1; c < nc; ++c) {
        if (e->f_f64[c] != e->f_f64[0]) return fail(PB_ERR_INVALID, "U, V, W must share one dtype");
        for (int d = 0; d < 4; ++d)
            if (e->fshape[c][d] != e->fshape[0][d]) return fail(PB_ERR_INVALID, "U, V, W must share one shape");
    }
    const long long T = e->fshape[0][0], Z = e->fshape[0][1], Y = e->fshape[0][2], X = e->fshape[0][3];
    // column slabs (pb_decomp_set_columns): the fields hold node columns [xi_offset, xi_offset + X) of the global grid
    const bool columns = on_columns(e);
    if ((X > 1 && X != e->g.nx && !(columns && X >= 2 && e->g.xi_offset + X <= e->g.nx)) || (Y > 1 && Y != e->g.ny) || (Z > 1 && e->g.nz > 0 && Z != e->g.nz) ||
        (T > 1 && e->g.nt > 0 && T != e->g.nt))
        return fail(PB_ERR_INVALID, "field shape (%lld,%lld,%lld,%lld) does not match grid nodes (nt=%d nz=%d ny=%d nx=%d)", T, Z, Y, X,
                    e->g.nt, e->g.nz, e->g.ny, e->g.nx);
    if ((T > 1) != (e->g.nt > 0)) return fail(PB_ERR_INVALID, "field has %lld time levels but the grid time axis has %d", T, e->g.nt);
    if (Z > 1 && e->g.nz == 0) return fail(PB_ERR_INVALID, "field has a depth dimension but the grid has no Z axis");
    if (e->g.curvilinear && e->interp != PB_INTERP_CGRID_VELOCITY && e->interp != PB_INTERP_XLINEAR_VELOCITY)
        return fail(PB_ERR_INVALID, "curvilinear grids are supported with CGrid_Velocity and XLinear_Velocity interpolation");
    return PB_OK;
}

// pre-pass of a sampling call: the reference's batch-level lenT / lenZ into the device word `flags` (see sample_flags_kernel)
static constexpr int SAMPLE_FLAGS_BLOCK = 256;
static int32_t launch_sample_flags(pb_engine* e, SampleParams& sp, bool has_time, int* flags) {
    CK(cudaMemsetAsync(flags, 0, sizeof(int), e->stream));
    const unsigned grid = (unsigned)((sp.n + SAMPLE_FLAGS_BLOCK - 1) / SAMPLE_FLAGS_BLOCK);
    if (e->coord_f64) sample_flags_kernel<double><<<grid, SAMPLE_FLAGS_BLOCK, 0, e->stream>>>(sp, has_time ? 1 : 0, flags);
    else sample_flags_kernel<float><<<grid, SAMPLE_FLAGS_BLOCK, 0, e->stream>>>(sp, has_time ? 1 : 0, flags);
    CK(cudaGetLastError());
    sp.batch_flags = flags;
    return PB_OK;
}

int32_t pb_sample_velocity(pb_engine* e, int64_t n, const double* t, const double* z, const double* y, const double* x,
                           int32_t positions_are_f32, int32_t three_d, const int32_t* ei_hint, int32_t no_hint, double* u,
                           double* v, double* w, int32_t* ei_out, int32_t* state_out) {
    PB_RANGE("pb_sample_velocity");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (n < 0 || (n && (!t || !z || !y || !x || !u || !v || !w || !ei_out || !state_out))) return fail(PB_ERR_INVALID, "NULL argument");
    const int nc = three_d ? 3 : 2;
    if (on_columns(e)) return fail(PB_ERR_STATE, "%s", COLUMNS_NO_SAMPLING);
    int32_t rc = check_fields(e, nc);
    if (rc) return rc;
    if (n == 0) return PB_OK;
    if (uvw_windowed(e) && (rc = check_resident_times(e, n, t))) return rc;
    CK(cudaSetDevice(e->device));
    if ((rc = e->samp_d.ensure((size_t)n * 7 * sizeof(double)))) return rc;
    if ((rc = e->samp_i.ensure(((size_t)n * 3 + 1) * sizeof(int)))) return rc;
    double* d = (double*)e->samp_d.p;  // t z y x u v w
    int* di = (int*)e->samp_i.p;       // hint ei state, batch flags
    const double* src[4] = {t, z, y, x};
    for (int k = 0; k < 4; ++k) CK(cudaMemcpyAsync(d + k * n, src[k], n * 8, cudaMemcpyHostToDevice, e->stream));
    if (ei_hint) CK(cudaMemcpyAsync(di, ei_hint, n * 4, cudaMemcpyHostToDevice, e->stream));
    SampleParams sp{};
    sp.g = e->g;
    fill_field_desc(e, sp.f);
    sp.n = n;
    sp.t = d; sp.z = d + n; sp.y = d + 2 * n; sp.x = d + 3 * n;
    sp.u = d + 4 * n; sp.v = d + 5 * n; sp.w = d + 6 * n;
    sp.ei_hint = ei_hint ? di : nullptr;
    sp.ei_out = di + n; sp.state_out = di + 2 * n;
    sp.pos_f32 = positions_are_f32; sp.no_hint = no_hint;
    if ((rc = launch_sample_flags(e, sp, e->g.nt > 0, di + 3 * n))) return rc;
    const int alt = agrid_alt_mode(e->interp);
    cudaError_t ce = e->interp == PB_INTERP_CGRID_VELOCITY
                         ? launch_sample_cgrid(sp, e->coord_f64 != 0, e->f_f64[0] != 0, nc, e->stream)
                     : e->g.curvilinear ? launch_sample_curv_agrid(sp, e->coord_f64 != 0, e->f_f64[0] != 0, nc, e->stream)
                     : alt ? launch_sample_agrid_alt(sp, alt, e->coord_f64 != 0, e->f_f64[0] != 0, e->g.nt > 0, nc, e->stream)
                           : launch_sample_agrid(sp, e->coord_f64 != 0, e->f_f64[0] != 0, e->g.nt > 0, nc, e->stream);
    if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "sample_kernel launch failed: %s", cudaGetErrorString(ce));
    double* dst[3] = {u, v, w};
    for (int k = 0; k < 3; ++k) CK(cudaMemcpyAsync(dst[k], d + (4 + k) * n, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(ei_out, di + n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(state_out, di + 2 * n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_sample_scalar(pb_engine* e, int32_t slot, int32_t method, int64_t n, const double* t, const double* z, const double* y,
                         const double* x, int32_t positions_are_f32, const int32_t* ei_hint, double* value, int32_t* value_is_f32,
                         int32_t* ei_out, int32_t* state_out) {
    PB_RANGE("pb_sample_scalar");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (n < 0 || (n && (!t || !z || !y || !x || !value || !ei_out || !state_out))) return fail(PB_ERR_INVALID, "NULL argument");
    if (slot < 0 || slot >= PB_MAX_FIELDS || !e->fptr[slot]) return fail(PB_ERR_STATE, "no field in slot %d", slot);
    if (method < PB_SCALAR_XLINEAR || method > PB_SCALAR_XLINEAR_INVDIST_LAND) return fail(PB_ERR_INVALID, "unknown scalar interpolation %d", method);
    if (!e->have_grid) return fail(PB_ERR_STATE, "grid not uploaded (pb_grid_upload_*)");
    if (on_columns(e)) return fail(PB_ERR_STATE, "%s", COLUMNS_NO_SAMPLING);
    if (e->g.curvilinear && method == PB_SCALAR_XLINEAR_INVDIST_LAND)
        return fail(PB_ERR_INVALID, "on curvilinear grids scalar sampling is implemented for XLinear, CGrid_Tracer and XNearest");
    if (e->ring && slot < 3) return fail(PB_ERR_INVALID, "U, V, W are time-windowed: sample them through pb_sample_velocity");
    SampleParams sp{};
    int32_t rc = field_slot_desc(e, slot, sp.f);
    if (rc) return rc;
    if (n == 0) return PB_OK;
    if (e->fwin[slot] && (rc = check_resident_times(e, n, t))) return rc;
    CK(cudaSetDevice(e->device));
    if ((rc = e->samp_d.ensure((size_t)n * 5 * sizeof(double)))) return rc;
    if ((rc = e->samp_i.ensure(((size_t)n * 4 + 1) * sizeof(int)))) return rc;
    double* d = (double*)e->samp_d.p;  // t z y x value
    int* di = (int*)e->samp_i.p;       // hint ei state f32, batch flags
    const double* src[4] = {t, z, y, x};
    for (int k = 0; k < 4; ++k) CK(cudaMemcpyAsync(d + k * n, src[k], n * 8, cudaMemcpyHostToDevice, e->stream));
    if (ei_hint) CK(cudaMemcpyAsync(di, ei_hint, n * 4, cudaMemcpyHostToDevice, e->stream));
    sp.g = e->g;
    sp.n = n;
    sp.t = d; sp.z = d + n; sp.y = d + 2 * n; sp.x = d + 3 * n;
    sp.u = d + 4 * n; sp.v = nullptr; sp.w = nullptr;
    sp.ei_hint = ei_hint ? di : nullptr;
    sp.ei_out = di + n; sp.state_out = di + 2 * n; sp.f32_out = di + 3 * n;
    sp.pos_f32 = positions_are_f32; sp.no_hint = ei_hint ? 0 : 1;
    const bool has_time = sp.f.T > 1;
    if ((rc = launch_sample_flags(e, sp, has_time, di + 4 * n))) return rc;
    // a field without a time dimension has no time interval: no time search at all (field.py:112-117)
    cudaError_t ce = e->g.curvilinear ? launch_sample_scalar_curv(sp, 3 + method, e->coord_f64 != 0, e->f_f64[slot] != 0, has_time, e->stream)
                                      : launch_sample_scalar(sp, 3 + method, e->coord_f64 != 0, e->f_f64[slot] != 0, has_time, e->stream);
    if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "sample_kernel launch failed: %s", cudaGetErrorString(ce));
    CK(cudaMemcpyAsync(value, d + 4 * n, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(ei_out, di + n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(state_out, di + 2 * n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    if (value_is_f32) CK(cudaMemcpyAsync(value_is_f32, di + 3 * n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

// The specialised RK4 kernel (afast.cu) gathers from a node-interleaved {u, v, w, 0} copy of the float32 fields: built here, on
// the device, the first time an RK4 launch can use it (float64 rectilinear grid, XLinear_Velocity, every level resident).
#ifndef PB_FAST_DEFAULT_DIFFUSION
#define PB_FAST_DEFAULT_DIFFUSION 1
#endif
static bool fast_kernel_enabled() {
    const char* v = getenv("PB_DISABLE_FAST_KERNEL");  // A/B switch of the parity tests and variant sweeps
    return !(v && v[0] == '1');
}
// which schedule of the specialised RK4 kernel (afast.cu): 2 = a two-stage loop body with compile-time renew / reuse, 1 = one
// evaluation site in a four-trip loop.  Schedule 2 is the faster one for advection only; with the fused diffusion block the
// two-stage body overflows the instruction cache: lists with DiffusionUniformKh run schedule 1.  PB_FAST_KERNEL=1|2 forces one.
static int fast_kernel_version(bool diffusion) {
    const char* v = getenv("PB_FAST_KERNEL");
    if (v && v[0] == '1') return 1;
    if (v && v[0] == '2') return 2;
    return diffusion ? PB_FAST_DEFAULT_DIFFUSION : 2;
}
static int32_t ensure_interleaved(pb_engine* e, int scheme) {
    if (e->il_valid) return PB_OK;
    if (!(scheme == PB_ADVECTION_RK4 || scheme == PB_ADVECTION_RK4_3D) || !fast_kernel_enabled()) return PB_OK;
    if (e->interp != PB_INTERP_XLINEAR_VELOCITY || e->g.curvilinear || !e->coord_f64 || e->ring || e->f_f64[0] || e->g.nt < 2) return PB_OK;
    if (!e->fptr[0] || !e->fptr[1]) return PB_OK;
    const long long nodes = e->fshape[0][0] * e->fshape[0][1] * e->fshape[0][2] * e->fshape[0][3];
    const bool have_w = e->fptr[2] && !e->f_f64[2] && e->fshape[2][0] == e->fshape[0][0] && e->fshape[2][1] == e->fshape[0][1] &&
                        e->fshape[2][2] == e->fshape[0][2] && e->fshape[2][3] == e->fshape[0][3];
    if (e->fptr[2] && !have_w) return PB_OK;  // (a W of another dtype / shape: the generic kernel's own checks apply)
    int32_t rc = e->il.ensure((size_t)nodes * 16);
    if (rc) return rc;
    cudaError_t ce = launch_interleave((const float*)e->fptr[0], (const float*)e->fptr[1], have_w ? (const float*)e->fptr[2] : nullptr,
                                       nodes, e->il.p, e->stream);
    if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "interleave_kernel launch failed: %s", cudaGetErrorString(ce));
    e->il_valid = true;
    return PB_OK;
}

// kernel parameters every advect entry point takes from the engine and from its arguments (pb_advect_args, pb_rk45_args,
// pb_advdiff_args); each entry point sets its own on top
extern "C++" {
template <class Args>
static void fill_advect_params(pb_engine* e, const Args* a, AdvectParams& p) {
    p.g = e->g;
    fill_field_desc(e, p.f);
    p.P = e->cur.view(e->n);
    p.delete_on_error = a->delete_on_error;
    p.dt = a->dt; p.endtime = a->endtime; p.max_iters = a->max_iters;
    p.resume = a->resume; p.kernels_only = a->kernels_only;
    p.batch_levels = a->batch_levels;
    p.rep = e->d_rep;
    for (int k = 0; k < 4; ++k) p.cells[k] = e->cellp[k];
}
}

// AdvectParams::lone_particle: the resident set is the whole set and holds one particle.  (Under mode D a rank holds a shard:
// its count says nothing about the whole set, and a shard of one particle is no batch of one.)
static int lone_particle(const pb_engine* e) { return e->n == 1 && !e->g.decomposed; }

// in-kernel migration (connected over peer memory, mode D): where the kernels deliver a leaving particle
static int32_t fill_mig(pb_engine* e, AdvectParams& p) {
    if (e->mig_on && e->g.decomposed) {
        if (!e->have_pid) return fail(PB_ERR_STATE, "migration needs particle_id");
        for (int r = 0; r < e->nranks; ++r) p.mig.peer[r] = e->mig_peer[r];
        p.mig.bounds = (const double*)e->mbounds.p;
        p.mig.cap = e->mig_cap;
        p.mig.nranks = e->nranks; p.mig.rank = e->rank;
        p.mig.slot = e->mig_slot;
        p.mig.on = 1;
    }
    return PB_OK;
}

// validation + kernel parameters shared by pb_advect_async and pb_advect_host (pb_advect_host sets p.P per chunk)
static int32_t prepare_advect(pb_engine* e, const pb_advect_args* a, AdvectParams& p, int& nc) {
    if (!e || !a) return fail(PB_ERR_INVALID, "NULL argument");
    if (a->dt == 0.0 || a->dt != a->dt) return fail(PB_ERR_INVALID, "dt must be a non-zero number");
    switch (a->scheme) {
        case PB_ADVECTION_NONE: case PB_ADVECTION_EE: case PB_ADVECTION_RK2: case PB_ADVECTION_RK4: nc = 2; break;
        case PB_ADVECTION_RK2_3D: case PB_ADVECTION_RK4_3D: nc = 3; break;
        default: return fail(PB_ERR_INVALID, "unknown scheme %d", a->scheme);
    }
    int32_t rc = check_fields(e, nc);
    if (rc) return rc;
    if ((rc = ensure_interleaved(e, a->scheme))) return rc;  // (before the field descriptor: it may now point at the copy)
    fill_advect_params(e, a, p);
    p.scheme = a->scheme; p.diffusion = a->diffusion;
    p.kh_spherical = a->kh_spherical;
    p.kh_zonal = a->kh_zonal; p.kh_meridional = a->kh_meridional; p.kh_deg2m = a->kh_deg2m;
    p.seed = a->seed; p.rng_call = a->rng_call;
    p.hint_all_zero = a->hint_all_zero;
    return fill_mig(e, p);
}

static cudaError_t launch_advect_kernel(pb_engine* e, const AdvectParams& p, int nc, cudaStream_t stream) {
    const int alt = agrid_alt_mode(e->interp);
    if (e->interp == PB_INTERP_XLINEAR_VELOCITY && fast_kernel_enabled() &&
        agrid_fast_applies(p, e->coord_f64 != 0, e->f_f64[0] != 0, e->g.nt > 0, nc)) {
        e->last_variant = fast_kernel_version(p.diffusion != 0);
        return launch_agrid_fast(p, nc, e->last_variant, stream);
    }
    e->last_variant = 0;
    return e->interp == PB_INTERP_CGRID_VELOCITY ? launch_cgrid(p, e->coord_f64 != 0, e->f_f64[0] != 0, nc, stream)
           : e->g.curvilinear ? launch_curv_agrid(p, e->coord_f64 != 0, e->f_f64[0] != 0, nc, stream)
           : alt ? launch_agrid_alt(p, alt, e->coord_f64 != 0, e->f_f64[0] != 0, e->g.nt > 0, nc, stream)
                 : launch_agrid(p, e->coord_f64 != 0, e->f_f64[0] != 0, e->g.nt > 0, nc, stream);
}

int32_t pb_advect_async(pb_engine* e, const pb_advect_args* a) {
    PB_RANGE("pb_advect_async");
    AdvectParams p{};
    int nc = 2;
    int32_t rc = prepare_advect(e, a, p, nc);
    if (rc) return rc;
    if (a->diffusion && !e->have_pid) return fail(PB_ERR_STATE, "diffusion needs particle_id (RNG counter)");
    CK(cudaSetDevice(e->device));
    p.lone_particle = lone_particle(e);
    if ((rc = begin_launch(e))) return rc;
    if (e->n > 0) {
        cudaError_t ce = launch_advect_kernel(e, p, nc, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "advect_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    return end_launch(e);
}

// Kernel.execute on HOST particle arrays, software-pipelined: the set is cut into chunks, each chunk goes H2D -> start-of-interval
// snapshot (D2D) -> advect kernel (-> D2H) in ONE in-order stream, and consecutive chunks use different streams, so the copies of
// one chunk run under the kernels of the others (separate DMA engines per direction) and the kernels of neighbouring chunks fill
// each other's tails.  No data-path dependency exists between particles, hence none between chunks; the report is accumulated
// with the same atomics.  Equivalent to pb_particles_upload + pb_particles_snapshot + pb_advect (+ pb_particles_download).
int32_t pb_advect_host(pb_engine* e, const pb_advect_args* a, int64_t n, const pb_particle_arrays* h, int32_t download,
                       int32_t n_chunks, pb_report* rep) {
    PB_RANGE("pb_advect_host");
    if (!e || !a || !h) return fail(PB_ERR_INVALID, "NULL argument");
    if (n < 0) return fail(PB_ERR_INVALID, "n < 0");
    if (n && (!h->x || !h->y || !h->z || !h->t || !h->state || !h->ei)) return fail(PB_ERR_INVALID, "NULL particle array");
    if (e->ring) return fail(PB_ERR_STATE, "pb_advect_host does not drive time-slab streaming: use pb_particles_upload + pb_advect");
    AdvectParams p{};
    int nc = 2;
    int32_t rc = prepare_advect(e, a, p, nc);
    if (rc) return rc;
    if (a->diffusion && !h->particle_id) return fail(PB_ERR_STATE, "diffusion needs particle_id (RNG counter)");
    CK(cudaSetDevice(e->device));
    if (!e->pipe_fork) {
        CK(cudaEventCreateWithFlags(&e->pipe_fork, cudaEventDisableTiming));
        for (int k = 0; k < pb_engine::PIPE; ++k) {
            CK(cudaStreamCreateWithFlags(&e->pipe_stream[k], cudaStreamNonBlocking));
            CK(cudaEventCreateWithFlags(&e->pipe_done[k], cudaEventDisableTiming));
        }
    }
    CK(cudaStreamSynchronize(e->stream));  // the buffers may be re-allocated below: nothing of an earlier call may be in flight
    const void* src[ParticleSoA::NCOL] = {h->x, h->y, h->z, h->dx, h->dy, h->dz, h->t, h->state, h->ei, h->particle_id};
    // the columns this call makes resident and snapshots: all but the ids when none are given
    auto resident = [&](int k) { return !ParticleSoA::cols[k].optional || src[k]; };
    for (int k = 0; k < ParticleSoA::NCOL; ++k)
        if (resident(k) && (rc = e->cur.col[k].ensure(n ? (size_t)n * ParticleSoA::cols[k].es : 1))) return rc;
    if ((rc = e->snap.ensure(n ? (size_t)n * ParticleSoA::row_bytes(true) : 1))) return rc;
    e->have_pid = h->particle_id != nullptr;
    e->snap_pid = e->have_pid;
    e->resume_on = e->snap_resume = false;
    e->n = n;
    e->snap_n = n;  // the chunks below write the start-of-interval copy
    p.lone_particle = n == 1;

    if ((rc = begin_launch(e))) return rc;
    CK(cudaEventRecord(e->pipe_fork, e->stream));
    // chunks of whole waves of 256-thread blocks over the H100's 132 SMs; small sets are not cut
    const long long align = 256 * 132;
    long long chunks = n_chunks < 1 ? 1 : n_chunks;
    long long per = n > 0 ? ((n + chunks - 1) / chunks + align - 1) / align * align : 0;
    if (per <= 0) per = align;
    const long long nchunk = n > 0 ? (n + per - 1) / per : 0;
    const int nstream = (int)(nchunk < pb_engine::PIPE ? nchunk : pb_engine::PIPE);
    for (int k = 0; k < nstream; ++k) CK(cudaStreamWaitEvent(e->pipe_stream[k], e->pipe_fork, 0));
    for (long long c = 0; c < nchunk; ++c) {
        cudaStream_t st = e->pipe_stream[c % pb_engine::PIPE];
        const long long lo = c * per, m = (n - lo < per ? n - lo : per);
        size_t snap_off = 0;
        for (int k = 0; k < ParticleSoA::NCOL; ++k) {
            if (!resident(k)) continue;
            const ParticleSoA::Column& col = ParticleSoA::cols[k];
            char* dev = (char*)e->cur.col[k].p + (size_t)lo * col.es;
            if (src[k]) CK(cudaMemcpyAsync(dev, (const char*)src[k] + (size_t)lo * col.es, (size_t)m * col.es, cudaMemcpyHostToDevice, st));
            else if (col.zero_if_absent) CK(cudaMemsetAsync(dev, 0, (size_t)m * col.es, st));
            // start-of-interval copy in pb_particles_snapshot's layout
            CK(cudaMemcpyAsync((char*)e->snap.p + snap_off + (size_t)lo * col.es, dev, (size_t)m * col.es, cudaMemcpyDeviceToDevice, st));
            snap_off += (size_t)n * col.es;
        }
        p.P = e->cur.view(m, lo);
        cudaError_t ce = launch_advect_kernel(e, p, nc, st);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "advect_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    if (download)  // issued after every launch: a copy into pageable memory blocks the host until it is done
        for (long long c = 0; c < nchunk; ++c) {
            cudaStream_t st = e->pipe_stream[c % pb_engine::PIPE];
            const long long lo = c * per, m = (n - lo < per ? n - lo : per);
            for (int k = 0; k < ParticleSoA::PID; ++k) {  // (the ids are not written back)
                const size_t es = ParticleSoA::cols[k].es;
                if (src[k])
                    CK(cudaMemcpyAsync((char*)const_cast<void*>(src[k]) + (size_t)lo * es, (char*)e->cur.col[k].p + (size_t)lo * es,
                                       (size_t)m * es, cudaMemcpyDeviceToHost, st));
            }
        }
    for (int k = 0; k < nstream; ++k) {
        CK(cudaEventRecord(e->pipe_done[k], e->pipe_stream[k]));
        CK(cudaStreamWaitEvent(e->stream, e->pipe_done[k], 0));
    }
    if ((rc = end_launch(e))) return rc;
    pb_report tmp;
    rc = pb_last_report(e, &tmp);
    if (rc) return rc;
    if (rep) *rep = tmp;
    return PB_OK;
}

int32_t pb_last_report(pb_engine* e, pb_report* rep) {
    PB_RANGE("pb_last_report");
    if (!e || !rep) return fail(PB_ERR_INVALID, "NULL argument");
    if (e->pending) {
        CK(cudaSetDevice(e->device));
        CK(cudaStreamSynchronize(e->stream));
        const ReportDev& r = *e->h_rep;
        pb_report o{};
        o.particle_steps = (int64_t)r.particle_steps;
        o.n_error = (int64_t)r.n_error;
        o.n_deleted = (int64_t)r.n_deleted;
        o.first_error_iter = r.first_error_iter == LLONG_MAX ? -1 : r.first_error_iter;
        o.n_out_of_time = (int64_t)r.n_out_of_time;
        o.max_iters_done = r.max_iters_done;
        o.cache_refills = (int64_t)r.cache_refills;
        o.n_migrate = (int64_t)r.n_migrate;
        o.n_wait_window = (int64_t)r.n_wait_window;
        if (r.n_wait_window) {
            long long lo = (long long)r.wait_t_min_bits, hi = (long long)r.wait_t_max_bits;
            memcpy(&o.wait_t_min, &lo, 8);
            memcpy(&o.wait_t_max, &hi, 8);
        }
        o.max_state = r.max_state;
        o.kernel_variant = e->last_variant;
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e->ev0, e->ev1));
        o.kernel_ms = ms;
        e->last = o;
        e->pending = false;
    }
    *rep = e->last;
    return PB_OK;
}

int32_t pb_advect(pb_engine* e, const pb_advect_args* a, pb_report* rep) {
    int32_t rc = pb_advect_async(e, a);
    if (rc) return rc;
    pb_report tmp;
    rc = pb_last_report(e, &tmp);
    if (rc) return rc;
    if (rep) *rep = tmp;
    return PB_OK;
}

// rk45_kernel for the engine's velocity interpolator: CGrid_Velocity, XFreeslip / XPartialslip or XLinear_Velocity
static cudaError_t launch_rk45_kernel(const pb_engine* e, const AdvectParams& p, const pb_rk45_args* a, double* dt, double* next_dt,
                                      int* iters) {
    const bool coord_f64 = e->coord_f64 != 0, data_f64 = e->f_f64[0] != 0;
    if (e->interp == PB_INTERP_CGRID_VELOCITY)
        return launch_rk45_cgrid(p, dt, next_dt, iters, a->next_dt_is_f32, a->tol, a->min_dt, a->max_dt, coord_f64, data_f64, e->stream);
    if (agrid_alt_mode(e->interp) == 1)
        return launch_rk45_slip(p, dt, next_dt, iters, a->next_dt_is_f32, a->tol, a->min_dt, a->max_dt, coord_f64, data_f64, e->g.nt > 0,
                                e->stream);
    return launch_rk45(p, dt, next_dt, iters, a->next_dt_is_f32, a->tol, a->min_dt, a->max_dt, coord_f64, data_f64, e->g.nt > 0, e->stream);
}

int32_t pb_advect_rk45(pb_engine* e, const pb_rk45_args* a, double* dt_inout, double* next_dt_inout, pb_report* rep) {
    PB_RANGE("pb_advect_rk45");
    if (!e || !a || !rep) return fail(PB_ERR_INVALID, "NULL argument");
    if (a->dt == 0.0 || a->dt != a->dt) return fail(PB_ERR_INVALID, "dt must be a non-zero number");
    if (e->n && (!dt_inout || !next_dt_inout)) return fail(PB_ERR_INVALID, "NULL dt / next_dt array");
    int32_t rc = check_fields(e, 2);
    if (rc) return rc;
    const bool cgrid = e->interp == PB_INTERP_CGRID_VELOCITY;
    const bool slip = agrid_alt_mode(e->interp) == 1;
    if (!(cgrid || ((e->interp == PB_INTERP_XLINEAR_VELOCITY || slip) && !e->g.curvilinear)) || e->g.decomposed)
        return fail(PB_ERR_INVALID, "AdvectionRK45 runs on XLinear_Velocity / XFreeslip / XPartialslip (rectilinear A-grid) "
                                    "or CGrid_Velocity fields, not under domain decomposition");
    CK(cudaSetDevice(e->device));
    const size_t n = (size_t)e->n;
    DevBuf& buf = e->sout;  // dt, next_dt (f64), iters (i32)
    if ((rc = buf.ensure(n ? n * 20 : 1))) return rc;  // (kept as it is across resumed launches: the iteration counts live here)
    double* d_dt = (double*)buf.p;
    double* d_ndt = d_dt + n;
    int* d_it = (int*)(d_ndt + n);
    if (n) {
        CK(cudaMemcpyAsync(d_dt, dt_inout, n * 8, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(d_ndt, next_dt_inout, n * 8, cudaMemcpyHostToDevice, e->stream));
    }
    AdvectParams p{};
    fill_advect_params(e, a, p);
    p.scheme = PB_ADVECTION_RK45;
    p.hint_all_zero = a->hint_all_zero;
    p.lone_particle = e->n == 1;
    if ((rc = begin_launch(e))) return rc;
    if (n) {
        cudaError_t ce = launch_rk45_kernel(e, p, a, d_dt, d_ndt, d_it);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "rk45_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    if ((rc = end_launch(e))) return rc;
    if ((rc = pb_last_report(e, rep))) return rc;
    if (n) {
        // once, after the last launch of the call: a launch that left lanes waiting for the time window is resumed, and the
        // counts it left in d_it are continued.  (In a mixed list the host clamps every particle's dt at the top of each iteration.)
        if (!a->kernels_only && rep->n_wait_window == 0) {
            cudaError_t ce = launch_rk45_finalize(p.P, d_dt, d_it, rep->max_iters_done, a->endtime, a->dt > 0 ? 1 : -1, e->stream);
            if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "rk45_finalize launch failed: %s", cudaGetErrorString(ce));
        }
        CK(cudaMemcpyAsync(dt_inout, d_dt, n * 8, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(next_dt_inout, d_ndt, n * 8, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
    }
    return PB_OK;
}

// AdvectionRK45 on the RESIDENT dt / next_dt / iteration columns (pb_particles_upload_resume): the route of a domain-decomposed
// engine, where these travel with the particles.  No finalize clamp: pb_rk45_finalize_resident once the whole call is done.
int32_t pb_advect_rk45_resident_async(pb_engine* e, const pb_rk45_args* a) {
    PB_RANGE("pb_advect_rk45_resident");
    if (!e || !a) return fail(PB_ERR_INVALID, "NULL argument");
    if (a->dt == 0.0 || a->dt != a->dt) return fail(PB_ERR_INVALID, "dt must be a non-zero number");
    if (a->kernels_only) return fail(PB_ERR_INVALID, "pb_advect_rk45_resident runs whole loop iterations (kernels_only = 0)");
    if (!e->resume_on) return fail(PB_ERR_STATE, "dt / next_dt / iteration columns not resident (pb_particles_upload_resume)");
    int32_t rc = check_fields(e, 2);
    if (rc) return rc;
    const bool cgrid = e->interp == PB_INTERP_CGRID_VELOCITY;
    const bool slip = agrid_alt_mode(e->interp) == 1;
    if (!(cgrid || ((e->interp == PB_INTERP_XLINEAR_VELOCITY || slip) && !e->g.curvilinear)))
        return fail(PB_ERR_INVALID, "pb_advect_rk45_resident runs on rectilinear grids with XLinear_Velocity, XFreeslip, XPartialslip "
                                    "or on rectilinear and curvilinear grids with CGrid_Velocity");
    CK(cudaSetDevice(e->device));
    AdvectParams p{};
    fill_advect_params(e, a, p);
    p.scheme = PB_ADVECTION_RK45;
    p.hint_all_zero = a->hint_all_zero;
    p.lone_particle = lone_particle(e);
    if ((rc = fill_mig(e, p))) return rc;
    if ((rc = begin_launch(e))) return rc;
    if (e->n > 0) {
        const ResumeDev r = e->cur.resume();
        cudaError_t ce = launch_rk45_kernel(e, p, a, r.dt, r.next_dt, r.iters);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "rk45_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    return end_launch(e);
}

int32_t pb_rk45_finalize_resident(pb_engine* e, double dt, double endtime, int64_t total_iters) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!e->resume_on) return fail(PB_ERR_STATE, "dt / next_dt / iteration columns not resident (pb_particles_upload_resume)");
    if (e->pending) return fail(PB_ERR_STATE, "an advect call is pending: call pb_last_report first");
    CK(cudaSetDevice(e->device));
    const ResumeDev r = e->cur.resume();
    cudaError_t ce = launch_rk45_finalize(e->cur.view(e->n), r.dt, r.iters, total_iters, endtime, dt > 0 ? 1 : -1, e->stream);
    if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "rk45_finalize launch failed: %s", cudaGetErrorString(ce));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

// FieldDev of a scalar field slot (slots 3.. hold the scalar fields)
static int32_t scalar_field_desc(pb_engine* e, int32_t slot, FieldDev& f) {
    if (slot < 3 || slot >= PB_MAX_FIELDS || !e->fptr[slot]) return fail(PB_ERR_STATE, "no scalar field in slot %d", slot);
    return field_slot_desc(e, slot, f);
}

int32_t pb_advect_diffusion_async(pb_engine* e, const pb_advdiff_args* a) {
    PB_RANGE("pb_advect_diffusion");
    if (!e || !a) return fail(PB_ERR_INVALID, "NULL argument");
    if (a->dt == 0.0 || a->dt != a->dt) return fail(PB_ERR_INVALID, "dt must be a non-zero number");
    if (a->scheme != PB_ADVDIFF_M1 && a->scheme != PB_ADVDIFF_EM) return fail(PB_ERR_INVALID, "unknown advection-diffusion scheme %d", a->scheme);
    if (!(a->dres == a->dres) || a->dres == 0.0) return fail(PB_ERR_INVALID, "dres must be a non-zero number");
    int32_t rc = check_fields(e, 2);
    if (rc) return rc;
    if ((e->interp != PB_INTERP_XLINEAR_VELOCITY && e->interp != PB_INTERP_CGRID_VELOCITY) || e->g.curvilinear)
        return fail(PB_ERR_INVALID, "AdvectionDiffusionM1/EM run on rectilinear fields with XLinear_Velocity or CGrid_Velocity");
    // under domain decomposition every lane's iteration count travels with its particle: a resident column
    if (e->g.decomposed && !e->resume_on)
        return fail(PB_ERR_INVALID, "AdvectionDiffusionM1/EM under domain decomposition run on the resident iteration columns "
                                    "(pb_particles_upload_resume)");
    if (!e->have_pid) return fail(PB_ERR_STATE, "diffusion needs particle_id (RNG counter)");
    FieldDev fkz, fkm;
    if ((rc = scalar_field_desc(e, a->kh_zonal_slot, fkz))) return rc;
    if ((rc = scalar_field_desc(e, a->kh_meridional_slot, fkm))) return rc;
    if (e->f_f64[a->kh_zonal_slot] != e->f_f64[a->kh_meridional_slot] || (fkz.T > 1) != (fkm.T > 1))
        return fail(PB_ERR_INVALID, "Kh_zonal and Kh_meridional must share dtype and time dimension");
    // a windowed Kh reads the levels of the one engine window, which the kernel's wait test checks through U, V
    if ((fkz.windowed || fkm.windowed) && !uvw_windowed(e))
        return fail(PB_ERR_INVALID, "time-windowed Kh_zonal / Kh_meridional need time-windowed U and V");
    CK(cudaSetDevice(e->device));
    AdvectParams p{};
    fill_advect_params(e, a, p);
    p.seed = a->seed; p.rng_call = a->rng_call;
    if ((rc = fill_mig(e, p))) return rc;
    // time-windowed fields: the lanes' iteration counts survive into the resumed launches (resident fields need none); with the
    // resumable-state columns resident (mode D) they live there
    int* iters = nullptr;
    if (e->resume_on) {
        iters = e->cur.resume().iters;
    } else if (e->ring) {
        if ((rc = e->ad_iters.ensure(e->n ? (size_t)e->n * sizeof(int) : 1))) return rc;
        iters = (int*)e->ad_iters.p;
    }
    if ((rc = begin_launch(e))) return rc;
    if (e->n > 0) {
        cudaError_t ce = launch_advdiff(p, fkz, fkm, a->scheme == PB_ADVDIFF_EM, a->dres, a->deg2m_sq, e->coord_f64 != 0, e->f_f64[0] != 0,
                                        e->f_f64[a->kh_zonal_slot] != 0, e->g.nt > 0, fkz.T > 1, e->interp == PB_INTERP_CGRID_VELOCITY,
                                        iters, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "advdiff_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    return end_launch(e);
}

int32_t pb_advect_diffusion(pb_engine* e, const pb_advdiff_args* a, pb_report* rep) {
    if (!rep) return fail(PB_ERR_INVALID, "NULL argument");
    int32_t rc = pb_advect_diffusion_async(e, a);
    if (rc) return rc;
    return pb_last_report(e, rep);
}

static int32_t flag_view(pb_engine* e, double dt, double endtime, int new_state) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    CK(cudaSetDevice(e->device));
    if (e->n > 0) {
        flag_view_kernel<<<(unsigned)((e->n + 255) / 256), 256, 0, e->stream>>>(e->cur.view(e->n), dt, endtime, new_state);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_flag_view_outside_time(pb_engine* e, double dt, double endtime) {
    return flag_view(e, dt, endtime, PB_ERROR_OUTSIDE_TIME_INTERVAL);
}

int32_t pb_delete_view_outside_time(pb_engine* e, double dt, double endtime) { return flag_view(e, dt, endtime, PB_DELETE); }

int32_t pb_debug_normals(pb_engine* e, uint64_t seed, uint64_t rng_call, int64_t iter, int64_t n,
                         const int64_t* particle_id, double* out) {
    if (!e || (n && (!particle_id || !out))) return fail(PB_ERR_INVALID, "NULL argument");
    CK(cudaSetDevice(e->device));
    if (n == 0) return PB_OK;
    long long* d_pid = nullptr;
    double* d_out = nullptr;
    CK(cudaMalloc(&d_pid, n * 8));
    CK(cudaMalloc(&d_out, n * 16));
    CK(cudaMemcpyAsync(d_pid, particle_id, n * 8, cudaMemcpyHostToDevice, e->stream));
    normals_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(seed, rng_call, iter, n, d_pid, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d_out, n * 16, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    cudaFree(d_pid);
    cudaFree(d_out);
    return PB_OK;
}

int32_t pb_debug_axis_cells(pb_engine* e, int32_t axis, int64_t cells, double* out) {
    if (!e || !out || axis < 0 || axis > 3) return fail(PB_ERR_INVALID, "NULL argument or unknown axis");
    const int n[4] = {e->g.nx, e->g.ny, e->g.nz, e->g.nt};
    if (!e->cellp[axis] || cells != (int64_t)n[axis] - 1) return fail(PB_ERR_INVALID, "no cell table of %lld cells for axis %d", (long long)cells, axis);
    CK(cudaSetDevice(e->device));
    CK(cudaMemcpyAsync(out, e->cellp[axis], (size_t)cells * sizeof(AxisCellRec), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

int32_t pb_debug_math(pb_engine* e, int32_t op, int64_t n, const double* a, const double* b, double* out) {
    if (!e || n < 0 || (n && (!a || !out))) return fail(PB_ERR_INVALID, "NULL argument");
    if (op < PB_MATH_COS_NP || op > PB_MATH_SIN) return fail(PB_ERR_INVALID, "unknown math op %d", op);
    const bool binary = op == PB_MATH_DIV_BY_CACHED || op == PB_MATH_DIV_BY_CACHED_GUARDED || op == PB_MATH_BOX_MULLER_F32;
    if (n && binary && !b) return fail(PB_ERR_INVALID, "math op %d needs a second operand", op);
    CK(cudaSetDevice(e->device));
    if (n == 0) return PB_OK;
    double *d_a = nullptr, *d_b = nullptr, *d_out = nullptr;
    CK(cudaMalloc(&d_a, n * 8));
    CK(cudaMalloc(&d_out, n * 16));
    if (binary) CK(cudaMalloc(&d_b, n * 8));
    CK(cudaMemcpyAsync(d_a, a, n * 8, cudaMemcpyHostToDevice, e->stream));
    if (binary) CK(cudaMemcpyAsync(d_b, b, n * 8, cudaMemcpyHostToDevice, e->stream));
    CK(launch_debug_math(op, n, d_a, d_b, d_out, e->stream));
    CK(cudaMemcpyAsync(out, d_out, n * 16, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    cudaFree(d_a);
    cudaFree(d_b);
    cudaFree(d_out);
    return PB_OK;
}

int32_t pb_debug_launch_block(int32_t family) {
    switch (family) {
        case PB_BLOCK_AGRID_FAST: return afast_launch_block();
        case PB_BLOCK_AGRID: return agrid_launch_block();
        case PB_BLOCK_CGRID: return cgrid_launch_block();
        case PB_BLOCK_CURV_AGRID: return curva_launch_block();
        case PB_BLOCK_SAMPLE_FLAGS: return SAMPLE_FLAGS_BLOCK;
        default: return fail(PB_ERR_INVALID, "unknown kernel family %d", family);
    }
}


// ------------------------------------------------------------------------------------------------
// mode D: X-slab domain decomposition + particle migration (SURVEY.md 8e).  The exchange itself is an
// all-to-all-v done by the caller over NCCL (torch.distributed) on the device buffers packed here.
// ------------------------------------------------------------------------------------------------
int32_t pb_decomp_set(pb_engine* e, int32_t nranks, int32_t rank, const double* bounds, int64_t xi_offset,
                      int32_t left_is_global, int32_t right_is_global) {
    if (!e || !bounds) return fail(PB_ERR_INVALID, "NULL argument");
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(PB_ERR_INVALID, "bad rank %d of %d", rank, nranks);
    if (!e->have_grid || e->g.curvilinear) return fail(PB_ERR_STATE, "domain decomposition needs an uploaded rectilinear grid");
    for (int r = 0; r < nranks; ++r)
        if (!(bounds[r] < bounds[r + 1])) return fail(PB_ERR_INVALID, "slab bounds must be strictly increasing");
    CK(cudaSetDevice(e->device));
    int32_t rc = upload(e, e->mbounds, bounds, (size_t)(nranks + 1) * sizeof(double));
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->stream));
    e->nranks = nranks; e->rank = rank;
    e->g.decomposed = nranks > 1 ? 1 : 0;
    e->g.xi_offset = (int)xi_offset;
    e->g.left_global = left_is_global ? 1 : 0;
    e->g.right_global = right_is_global ? 1 : 0;
    // rank 0 also owns everything left of the domain, the last rank everything right of it (there the
    // reference's own out-of-bounds semantics apply: index -2 / -1 at a GLOBAL edge)
    e->g.own_lo = rank == 0 ? -HUGE_VAL : bounds[rank];
    e->g.own_hi = rank == nranks - 1 ? HUGE_VAL : bounds[rank + 1];
    e->send_counts.assign(nranks, 0);
    return PB_OK;
}

// Column slabs of a curvilinear grid: the engine holds the WHOLE horizontal grid (lon / lat, cell projections, spatial hash) and
// the node columns [xi_offset, xi_offset + X) of the fields; rank r owns the cells whose global column i has
// col_edges[r] <= i < col_edges[r + 1].  The edges are kept as doubles in the slab-bounds buffer: the kernels' routing loop
// compares the found column with them as the rectilinear one compares x with longitudes.
int32_t pb_decomp_set_columns(pb_engine* e, int32_t nranks, int32_t rank, const int64_t* col_edges, int64_t xi_offset,
                              int32_t left_is_global, int32_t right_is_global) {
    if (!e || !col_edges) return fail(PB_ERR_INVALID, "NULL argument");
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(PB_ERR_INVALID, "bad rank %d of %d", rank, nranks);
    if (!e->have_grid || !e->g.curvilinear) return fail(PB_ERR_STATE, "column slabs need an uploaded curvilinear grid");
    if (col_edges[0] != 0 || col_edges[nranks] != e->g.nx - 1) return fail(PB_ERR_INVALID, "column edges must span cells 0 .. nx - 1");
    for (int r = 0; r < nranks; ++r)
        if (!(col_edges[r] < col_edges[r + 1])) return fail(PB_ERR_INVALID, "column edges must be strictly increasing");
    if (xi_offset < 0 || xi_offset > col_edges[rank] || (left_is_global != 0) != (xi_offset == 0))
        return fail(PB_ERR_INVALID, "bad column offset %lld for the cells of rank %d", (long long)xi_offset, rank);
    std::vector<double> edges(nranks + 1);
    for (int r = 0; r <= nranks; ++r) edges[r] = (double)col_edges[r];
    CK(cudaSetDevice(e->device));
    int32_t rc = upload(e, e->mbounds, edges.data(), edges.size() * sizeof(double));
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->stream));
    e->nranks = nranks; e->rank = rank;
    e->g.decomposed = nranks > 1 ? 1 : 0;
    e->g.xi_offset = (int)xi_offset;
    e->g.left_global = left_is_global ? 1 : 0;
    e->g.right_global = right_is_global ? 1 : 0;
    e->g.own_lo = edges[rank];
    e->g.own_hi = edges[rank + 1];
    e->send_counts.assign(nranks, 0);
    return PB_OK;
}

int32_t pb_migrate_classify_columns(pb_engine* e, int32_t no_hint, int64_t* counts) {
    PB_RANGE("pb_migrate_classify_columns");
    if (!e || !counts) return fail(PB_ERR_INVALID, "NULL argument");
    if (!e->g.curvilinear || e->nranks < 1 || e->mbounds.bytes == 0) return fail(PB_ERR_STATE, "pb_decomp_set_columns not called");
    if (!e->have_pid && e->n) return fail(PB_ERR_STATE, "migration needs particle_id");
    CK(cudaSetDevice(e->device));
    const int nr = e->nranks;
    int32_t rc;
    if ((rc = e->mdest.ensure(e->n ? e->n * 4 : 4))) return rc;
    if ((rc = e->mcount.ensure((size_t)(nr + 1) * 8))) return rc;
    CK(cudaMemsetAsync(e->mcount.p, 0, (size_t)(nr + 1) * 8, e->stream));
    if (e->n > 0) {
        AdvectParams p{};
        p.g = e->g;
        p.P = e->cur.view(e->n);
        p.hint_all_zero = no_hint;
        // the kernels that count their iterations across ranks (resumable state resident) skip the hint at a lane's first only
        const int* iters = e->resume_on ? e->cur.resume().iters : nullptr;
        cudaError_t ce = launch_classify_columns(p, e->coord_f64 != 0, iters, no_hint, (const double*)e->mbounds.p, nr, e->rank,
                                                 (int*)e->mdest.p, (unsigned long long*)e->mcount.p, e->stream);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "classify_columns_kernel launch failed: %s", cudaGetErrorString(ce));
    }
    std::vector<unsigned long long> h(nr + 1);
    CK(cudaMemcpyAsync(h.data(), e->mcount.p, (size_t)(nr + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->n_send = 0;
    for (int r = 0; r < nr; ++r) { counts[r] = (int64_t)h[r]; e->send_counts[r] = (long long)h[r]; e->n_send += (long long)h[r]; }
    e->n_keep = (long long)h[nr];
    return PB_OK;
}

int32_t pb_memory_bytes(pb_engine* e, int64_t* grid_bytes, int64_t* field_bytes) {
    if (!e || !grid_bytes || !field_bytes) return fail(PB_ERR_INVALID, "NULL argument");
    int64_t g = 0, f = 0;
    for (const DevBuf* b : {&e->lon, &e->lat, &e->depth, &e->time, &e->hkeys, &e->hstarts, &e->hcounts, &e->hfaces, &e->hbucket,
                            &e->cellproj, &e->hqbox, &e->cells})
        g += (int64_t)b->bytes;
    for (const DevBuf& b : e->fbuf) f += (int64_t)b.bytes;
    f += (int64_t)e->il.bytes;
    *grid_bytes = g;
    *field_bytes = f;
    return PB_OK;
}

// ordered selection of the resident particles: indices to e->sidx, count returned
static int32_t run_select(pb_engine* e, const SelectRule& r, long long* n_sel) {
    CK(cudaSetDevice(e->device));
    *n_sel = 0;
    if (e->n == 0) return PB_OK;
    const long long nb = (e->n + SEL_BLOCK - 1) / SEL_BLOCK;
    int32_t rc;
    if ((rc = e->sblock.ensure((size_t)nb * 4))) return rc;
    if ((rc = e->soffs.ensure((size_t)(nb + 1) * 8))) return rc;
    if ((rc = e->sidx.ensure((size_t)e->n * 8))) return rc;
    const ParticlesDev P = e->cur.view(e->n);
    sel_count<<<(unsigned)nb, SEL_BLOCK, 0, e->stream>>>(P, r, (unsigned int*)e->sblock.p);
    CK(cudaGetLastError());
    long long* offs = (long long*)e->soffs.p;
    sel_scan<<<1, 1024, 0, e->stream>>>((const unsigned int*)e->sblock.p, offs, nb, offs + nb);
    CK(cudaGetLastError());
    sel_scatter<<<(unsigned)nb, SEL_BLOCK, 0, e->stream>>>(P, r, offs, (long long*)e->sidx.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_sel_total, offs + nb, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    *n_sel = *e->h_sel_total;
    return PB_OK;
}

int32_t pb_output_select(pb_engine* e, double t_out, double dt, int64_t* n_selected) {
    PB_RANGE("pb_output_select");
    if (!e || !n_selected) return fail(PB_ERR_INVALID, "NULL argument");
    if (e->pending) return fail(PB_ERR_STATE, "an advect call is pending: call pb_last_report first");
    const double half = fabs(dt / 2);
    long long m = 0;
    int32_t rc = run_select(e, SelectRule{SEL_OUTPUT, t_out - half, t_out + half}, &m);
    if (rc) return rc;
    e->n_selected = m;
    *n_selected = m;
    return PB_OK;
}

int32_t pb_output_gather(pb_engine* e, int64_t n_selected, int64_t* index, float* x, float* y, float* z, double* t,
                         int64_t* particle_id) {
    PB_RANGE("pb_output_gather");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (e->n_selected < 0 || n_selected != e->n_selected)
        return fail(PB_ERR_STATE, "gather of %lld rows but the last pb_output_select chose %lld", (long long)n_selected, e->n_selected);
    if (particle_id && !e->have_pid && n_selected) return fail(PB_ERR_STATE, "no particle ids resident");
    if (n_selected == 0) return PB_OK;
    CK(cudaSetDevice(e->device));
    const size_t m = (size_t)n_selected;
    int32_t rc = e->sout.ensure(m * 28);  // x, y, z (4 B) + t, particle_id (8 B)
    if (rc) return rc;
    char* o = (char*)e->sout.p;
    double* dt_ = (double*)o;                 // 8-byte columns first: keeps every column aligned
    long long* dpid = (long long*)(o + m * 8);
    float* dx = (float*)(o + m * 16);
    float* dy = dx + m;
    float* dz = dy + m;
    out_gather<<<(unsigned)((m + 255) / 256), 256, 0, e->stream>>>(e->cur.view(e->n), (const long long*)e->sidx.p, (long long)m,
                                                                  x ? dx : nullptr, y ? dy : nullptr, z ? dz : nullptr,
                                                                  t ? dt_ : nullptr, particle_id ? dpid : nullptr);
    CK(cudaGetLastError());
    if (x) CK(cudaMemcpyAsync(x, dx, m * 4, cudaMemcpyDeviceToHost, e->stream));
    if (y) CK(cudaMemcpyAsync(y, dy, m * 4, cudaMemcpyDeviceToHost, e->stream));
    if (z) CK(cudaMemcpyAsync(z, dz, m * 4, cudaMemcpyDeviceToHost, e->stream));
    if (t) CK(cudaMemcpyAsync(t, dt_, m * 8, cudaMemcpyDeviceToHost, e->stream));
    if (particle_id) CK(cudaMemcpyAsync(particle_id, dpid, m * 8, cudaMemcpyDeviceToHost, e->stream));
    if (index) CK(cudaMemcpyAsync(index, e->sidx.p, m * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return PB_OK;
}

// The new resident set, built in the alternate columns: the current rows keep_idx[0..n_keep), then n_in arrival records; the
// alternates then become current.  headroom: allocate 25 % more than needed (fewer reallocations when the count drifts).
// With the resumable-state columns resident they are carried too (arrivals_resume: the arrivals' MigResume at the same index).
static int32_t rebuild_resident(pb_engine* e, const long long* keep_idx, long long n_keep, const MigRecord* arrivals,
                                const MigResume* arrivals_resume, long long n_in, bool headroom) {
    const long long n_new = n_keep + n_in;
    const size_t cap = n_new ? (size_t)n_new : 1;
    for (int k = 0; k < ParticleSoA::NCOL; ++k) {
        const size_t bytes = cap * ParticleSoA::cols[k].es;
        int32_t rc = e->alt.col[k].ensure(headroom ? bytes + bytes / 4 : bytes);
        if (rc) return rc;
    }
    for (int k = 0; e->resume_on && k < ParticleSoA::NRES; ++k) {
        const size_t bytes = cap * ParticleSoA::res_es[k];
        int32_t rc = e->alt.res[k].ensure(headroom ? bytes + bytes / 4 : bytes);
        if (rc) return rc;
    }
    if (e->resume_on && n_in > 0 && !arrivals_resume) return fail(PB_ERR_INVALID, "arrivals without their resumable state");
    const ParticlesDev dst = e->alt.view(n_new);
    const ResumeDev rsrc = e->resume_on ? e->cur.resume() : ResumeDev{}, rdst = e->resume_on ? e->alt.resume() : ResumeDev{};
    if (n_keep > 0) {
        mig_compact<<<(unsigned)((n_keep + 255) / 256), 256, 0, e->stream>>>(e->cur.view(e->n), dst, rsrc, rdst, keep_idx, n_keep);
        CK(cudaGetLastError());
    }
    if (n_in > 0) {
        mig_unpack<<<(unsigned)((n_in + 255) / 256), 256, 0, e->stream>>>(dst, rdst, n_keep, arrivals, arrivals_resume, n_in);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(e->stream));
    std::swap(e->cur, e->alt);
    e->n = n_new;
    if (!e->snap_pid) e->snap_n = -1;  // (a snapshot with ids restores the whole earlier set, count included)
    e->n_keep = n_new;
    return PB_OK;
}

int32_t pb_particles_remove_deleted(pb_engine* e, int64_t* n_left) {
    PB_RANGE("pb_particles_remove_deleted");
    if (!e || !n_left) return fail(PB_ERR_INVALID, "NULL argument");
    if (e->pending) return fail(PB_ERR_STATE, "an advect call is pending: call pb_last_report first");
    if (!e->have_pid && e->n) return fail(PB_ERR_STATE, "compaction needs particle_id resident");
    long long keep = 0;
    int32_t rc = run_select(e, SelectRule{SEL_ALIVE, 0.0, 0.0}, &keep);
    if (rc) return rc;
    e->n_selected = -1;
    if (keep == e->n) { *n_left = keep; return PB_OK; }
    if ((rc = rebuild_resident(e, (const long long*)e->sidx.p, keep, nullptr, nullptr, 0, false))) return rc;
    *n_left = keep;
    return PB_OK;
}

int32_t pb_migrate_count(pb_engine* e, int64_t* counts) {
    PB_RANGE("pb_migrate_count");
    if (!e || !counts) return fail(PB_ERR_INVALID, "NULL argument");
    if (e->nranks < 1 || e->mbounds.bytes == 0) return fail(PB_ERR_STATE, "pb_decomp_set not called");
    if (!e->have_pid && e->n) return fail(PB_ERR_STATE, "migration needs particle_id");
    CK(cudaSetDevice(e->device));
    const int nr = e->nranks;
    int32_t rc;
    if ((rc = e->mdest.ensure(e->n ? e->n * 4 : 4))) return rc;
    if ((rc = e->mcount.ensure((size_t)(nr + 1) * 8))) return rc;
    CK(cudaMemsetAsync(e->mcount.p, 0, (size_t)(nr + 1) * 8, e->stream));
    if (e->n > 0) {
        mig_classify<<<(unsigned)((e->n + 255) / 256), 256, 0, e->stream>>>(e->cur.view(e->n), (const double*)e->mbounds.p, nr, e->rank,
                                                                            (int*)e->mdest.p, (unsigned long long*)e->mcount.p);
        CK(cudaGetLastError());
    }
    std::vector<unsigned long long> h(nr + 1);
    CK(cudaMemcpyAsync(h.data(), e->mcount.p, (size_t)(nr + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->n_send = 0;
    for (int r = 0; r < nr; ++r) { counts[r] = (int64_t)h[r]; e->send_counts[r] = (long long)h[r]; e->n_send += (long long)h[r]; }
    e->n_keep = (long long)h[nr];
    return PB_OK;
}

static int32_t migrate_pack(pb_engine* e, void* sendbuf_dev, void* resume_sendbuf_dev, int64_t capacity_records) {
    if (e->n_send > capacity_records) return fail(PB_ERR_INVALID, "send buffer holds %lld records, %lld needed", (long long)capacity_records, e->n_send);
    if (e->n_send && (!sendbuf_dev || (e->resume_on && !resume_sendbuf_dev))) return fail(PB_ERR_INVALID, "NULL send buffer");
    CK(cudaSetDevice(e->device));
    const int nr = e->nranks;
    // cursors: [0..nr-1] = exclusive prefix of the per-destination counts, [nr] = 0 (keep cursor)
    std::vector<unsigned long long> cur(nr + 1, 0);
    for (int r = 1; r < nr; ++r) cur[r] = cur[r - 1] + (unsigned long long)e->send_counts[r - 1];
    CK(cudaMemcpyAsync(e->mcount.p, cur.data(), (size_t)(nr + 1) * 8, cudaMemcpyHostToDevice, e->stream));
    int32_t rc;
    if ((rc = e->mkeep.ensure(e->n_keep ? e->n_keep * 8 : 8))) return rc;
    if (e->n > 0) {
        mig_pack<<<(unsigned)((e->n + 255) / 256), 256, 0, e->stream>>>(
            e->cur.view(e->n), e->resume_on ? e->cur.resume() : ResumeDev{}, (const int*)e->mdest.p, nr, (unsigned long long*)e->mcount.p,
            (MigRecord*)sendbuf_dev, e->resume_on ? (MigResume*)resume_sendbuf_dev : nullptr, (long long*)e->mkeep.p);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(e->stream));  // cur goes out of scope; the caller hands sendbuf to NCCL next
    return PB_OK;
}

int32_t pb_migrate_pack(pb_engine* e, void* sendbuf_dev, int64_t capacity_records) {
    PB_RANGE("pb_migrate_pack");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (e->resume_on) return fail(PB_ERR_STATE, "resumable state resident: pb_migrate_pack_resume carries it");
    return migrate_pack(e, sendbuf_dev, nullptr, capacity_records);
}

int32_t pb_migrate_pack_resume(pb_engine* e, void* sendbuf_dev, void* resume_sendbuf_dev, int64_t capacity_records) {
    PB_RANGE("pb_migrate_pack_resume");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!e->resume_on) return fail(PB_ERR_STATE, "no resumable state resident (pb_particles_upload_resume)");
    return migrate_pack(e, sendbuf_dev, resume_sendbuf_dev, capacity_records);
}

int32_t pb_migrate_unpack(pb_engine* e, const void* recvbuf_dev, int64_t n_in) {
    PB_RANGE("pb_migrate_unpack");
    if (!e || n_in < 0 || (n_in && !recvbuf_dev)) return fail(PB_ERR_INVALID, "bad argument");
    if (e->resume_on) return fail(PB_ERR_STATE, "resumable state resident: pb_migrate_unpack_resume carries it");
    CK(cudaSetDevice(e->device));
    int32_t rc = rebuild_resident(e, (const long long*)e->mkeep.p, e->n_keep, (const MigRecord*)recvbuf_dev, nullptr, n_in, true);
    if (rc) return rc;
    e->n_send = 0;
    return PB_OK;
}

int32_t pb_migrate_unpack_resume(pb_engine* e, const void* recvbuf_dev, const void* resume_recvbuf_dev, int64_t n_in) {
    PB_RANGE("pb_migrate_unpack_resume");
    if (!e || n_in < 0 || (n_in && (!recvbuf_dev || !resume_recvbuf_dev))) return fail(PB_ERR_INVALID, "bad argument");
    if (!e->resume_on) return fail(PB_ERR_STATE, "no resumable state resident (pb_particles_upload_resume)");
    CK(cudaSetDevice(e->device));
    int32_t rc = rebuild_resident(e, (const long long*)e->mkeep.p, e->n_keep, (const MigRecord*)recvbuf_dev,
                                  (const MigResume*)resume_recvbuf_dev, n_in, true);
    if (rc) return rc;
    e->n_send = 0;
    return PB_OK;
}


// ---- in-kernel migration over peer memory (NVLink / NVSwitch) ----
// The advection kernel itself stores a leaving particle's record into the new owner's inbox (common.cuh, MigDev); the host side
// is the set-up (allocate the inbox, exchange CUDA-IPC handles, map the peers) and, once per round and AFTER a barrier that
// orders every rank's kernel before it, pb_migrate_p2p_finish: drop the records that left, append the arrivals, flip the slot.
int32_t pb_migrate_p2p_init(pb_engine* e, int64_t capacity_records, uint8_t* ipc_handle, uint64_t* local_base) {
    if (!e || capacity_records < 1) return fail(PB_ERR_INVALID, "bad argument");
    if (e->nranks < 2 || !e->g.decomposed) return fail(PB_ERR_STATE, "pb_decomp_set (>= 2 ranks) not called");
    if (e->nranks > PB_MIG_MAX_RANKS) return fail(PB_ERR_INVALID, "in-kernel migration supports <= %d ranks", PB_MIG_MAX_RANKS);
    if (e->mig_base) return fail(PB_ERR_STATE, "pb_migrate_p2p_init called twice");
    CK(cudaSetDevice(e->device));
    // [header 0][header 1][records of slot 0][records of slot 1][MigResume of slot 0][MigResume of slot 1] (common.cuh)
    const size_t bytes = 2 * (size_t)PB_MIG_HEADER_BYTES + 2 * (size_t)capacity_records * (sizeof(MigRecord) + sizeof(MigResume));
    void* p = nullptr;
    CK(cudaMalloc(&p, bytes));  // (its own allocation: IPC handles export whole allocations)
    e->mig_base = (unsigned char*)p;
    CK(cudaMemsetAsync(p, 0, 2 * (size_t)PB_MIG_HEADER_BYTES, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->mig_cap = capacity_records;
    e->mig_slot = 0;
    if (!e->h_mig_count) CK(cudaMallocHost((void**)&e->h_mig_count, 8));
    if (ipc_handle) {
        cudaIpcMemHandle_t h;
        CK(cudaIpcGetMemHandle(&h, p));
        static_assert(sizeof(h) == PB_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t size");
        memcpy(ipc_handle, &h, sizeof(h));
    }
    if (local_base) *local_base = (uint64_t)(uintptr_t)p;
    return PB_OK;
}

int32_t pb_migrate_p2p_connect(pb_engine* e, const uint8_t* ipc_handles, const uint64_t* local_bases) {
    if (!e || (!ipc_handles && !local_bases)) return fail(PB_ERR_INVALID, "NULL argument");
    if (!e->mig_base) return fail(PB_ERR_STATE, "pb_migrate_p2p_init not called");
    CK(cudaSetDevice(e->device));
    for (int r = 0; r < e->nranks; ++r) {
        if (r == e->rank) { e->mig_peer[r] = e->mig_base; continue; }
        if (local_bases && local_bases[r]) {  // a peer engine of THIS process: its pointer is valid here as it is
            e->mig_peer[r] = (unsigned char*)(uintptr_t)local_bases[r];
            continue;
        }
        if (!ipc_handles) return fail(PB_ERR_INVALID, "no handle for rank %d", r);
        cudaIpcMemHandle_t h;
        memcpy(&h, ipc_handles + (size_t)r * PB_IPC_HANDLE_BYTES, sizeof(h));
        void* q = nullptr;
        cudaError_t ce = cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
        if (ce != cudaSuccess) return fail(PB_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(ce));
        e->mig_peer[r] = (unsigned char*)q;
        e->mig_ipc_opened[r] = true;
    }
    e->mig_on = true;
    return PB_OK;
}

int32_t pb_migrate_p2p_disable(pb_engine* e) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    e->mig_on = false;
    return PB_OK;
}

int32_t pb_migrate_p2p_finish(pb_engine* e, int64_t* n_in_out, int64_t* n_now) {
    PB_RANGE("pb_migrate_p2p_finish");
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!e->mig_on) return fail(PB_ERR_STATE, "pb_migrate_p2p_connect not called");
    if (e->pending) return fail(PB_ERR_STATE, "an advect call is pending: call pb_last_report first");
    CK(cudaSetDevice(e->device));
    const int slot = e->mig_slot;
    CK(cudaMemcpyAsync(e->h_mig_count, mig_counter(e->mig_base, slot), 8, cudaMemcpyDeviceToHost, e->stream));
    long long keep = 0;
    int32_t rc = run_select(e, SelectRule{SEL_RESIDENT, 0.0, 0.0}, &keep);  // (synchronises the stream: the count above is in)
    if (rc) return rc;
    if (e->n == 0) CK(cudaStreamSynchronize(e->stream));
    e->n_selected = -1;
    const unsigned long long arrived = *e->h_mig_count;
    const long long n_in = (long long)(arrived < (unsigned long long)e->mig_cap ? arrived : (unsigned long long)e->mig_cap);
    if (keep != e->n || n_in > 0)
        if ((rc = rebuild_resident(e, (const long long*)e->sidx.p, keep, mig_records(e->mig_base, slot, e->mig_cap),
                                   mig_resume(e->mig_base, slot, e->mig_cap), n_in, true)))
            return rc;
    // this slot is written again two rounds from now, after at least one more barrier: reset its counter now
    CK(cudaMemsetAsync(mig_counter(e->mig_base, slot), 0, 8, e->stream));
    e->mig_slot ^= 1;
    if (n_in_out) *n_in_out = n_in;
    if (n_now) *n_now = e->n;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// time-slab streaming (SURVEY.md 8f-1): GPU analogue of the reference's WindowedArray
// (_core/_windowed_array.py:25-97, _core/model.py:79-113): only `window_levels` consecutive time levels of
// U, V, W are resident; one extra ring slot receives the next level on a copy stream while the advection
// kernel runs on the levels it needs.
// ------------------------------------------------------------------------------------------------
int32_t pb_field_window_create(pb_engine* e, int32_t slot, int32_t data_is_f64, int64_t T_total, int64_t Z, int64_t Y, int64_t X,
                               int32_t window_levels) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (slot < 0 || slot >= PB_MAX_FIELDS) return fail(PB_ERR_INVALID, "bad field slot %d", slot);
    if (T_total < 2 || Z < 1 || Y < 1 || X < 1 || window_levels < 2) return fail(PB_ERR_INVALID, "a time window needs >= 2 levels of a time-varying field");
    if (window_levels + 1 > T_total) return fail(PB_ERR_INVALID, "window (%d levels) + 1 prefetch slot exceeds the %lld levels of the field: upload it whole", window_levels, (long long)T_total);
    if (e->ring && e->ring != window_levels + 1) return fail(PB_ERR_INVALID, "all components must use the same window");
    CK(cudaSetDevice(e->device));
    const size_t level_bytes = (size_t)Z * Y * X * (data_is_f64 ? 8 : 4);
    int32_t rc = e->fbuf[slot].ensure(level_bytes * (size_t)(window_levels + 1));
    if (rc) return rc;
    // A sample exactly on a time level t == time[k] has ti = k - 1, tau = 1 (side="left" search): level k - 1 is gathered and
    // multiplied by (1 - tau) = 0.  It need not be resident for the result -- but its ring slot must hold FINITE values, or
    // 0 * garbage = NaN flags the particle (found by oracle/hostsim, where "device" memory is malloc'ed, not zero pages)
    CK(cudaMemsetAsync(e->fbuf[slot].p, 0, level_bytes * (size_t)(window_levels + 1), e->stream));
    CK(cudaStreamSynchronize(e->stream));  // the level loads run on the copy stream: the zeros must be in place first
    e->ring = window_levels + 1;
    e->win_first = 0; e->win_n = 0;
    rc = set_field(e, slot, e->fbuf[slot].p, data_is_f64, T_total, Z, Y, X);
    e->fwin[slot] = true;
    return rc;
}

int32_t pb_field_window_load(pb_engine* e, int32_t slot, int64_t level, const void* host_level_data) {
    PB_RANGE("pb_field_window_load");
    if (!e || !host_level_data) return fail(PB_ERR_INVALID, "NULL argument");
    if (slot < 0 || slot >= PB_MAX_FIELDS || !e->fwin[slot]) return fail(PB_ERR_STATE, "pb_field_window_create first");
    if (level < 0 || level >= e->fshape[slot][0]) return fail(PB_ERR_INVALID, "time level %lld out of range", (long long)level);
    CK(cudaSetDevice(e->device));
    const size_t level_bytes = (size_t)e->fshape[slot][1] * e->fshape[slot][2] * e->fshape[slot][3] * (e->f_f64[slot] ? 8 : 4);
    char* dst = (char*)e->fbuf[slot].p + (size_t)(level % e->ring) * level_bytes;
    CK(cudaMemcpyAsync(dst, host_level_data, level_bytes, cudaMemcpyHostToDevice, e->copy_stream));
    return PB_OK;
}

int32_t pb_field_window_set(pb_engine* e, int64_t first_level, int64_t n_levels) {
    if (!e) return fail(PB_ERR_INVALID, "engine is NULL");
    if (!e->ring) return fail(PB_ERR_STATE, "pb_field_window_create first");
    if (first_level < 0 || n_levels < 2 || n_levels > e->ring || first_level + n_levels > e->g.nt)
        return fail(PB_ERR_INVALID, "bad window [%lld, +%lld)", (long long)first_level, (long long)n_levels);
    CK(cudaSetDevice(e->device));
    // the advection stream must not start before the pending level loads have landed
    CK(cudaEventRecord(e->copy_done, e->copy_stream));
    CK(cudaStreamWaitEvent(e->stream, e->copy_done, 0));
    e->win_first = first_level; e->win_n = n_levels;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------------
// host-side column passes (see include/parcels_b200.h): plain C++ threads, no device
// ------------------------------------------------------------------------------------------------
int32_t pb_host_fill_f64(double* p, int64_t n, double value) {
    if (n < 0 || (n && !p)) return fail(PB_ERR_INVALID, "bad argument");
    host_parallel(n, [=](int, int64_t lo, int64_t hi) { for (int64_t i = lo; i < hi; ++i) p[i] = value; });
    return PB_OK;
}

int32_t pb_host_fill_i32(int32_t* p, int64_t n, int32_t value) {
    if (n < 0 || (n && !p)) return fail(PB_ERR_INVALID, "bad argument");
    host_parallel(n, [=](int, int64_t lo, int64_t hi) { for (int64_t i = lo; i < hi; ++i) p[i] = value; });
    return PB_OK;
}

// dst[i * dst_stride] = src[i * src_stride] (strides in elements): the last column of a FieldSet with several grids' `ei` (N, ngrids)
// to / from the contiguous column the device transfers use
int32_t pb_host_copy_strided_i32(int32_t* dst, int64_t dst_stride, const int32_t* src, int64_t src_stride, int64_t n) {
    if (n < 0 || (n && (!dst || !src)) || dst_stride < 1 || src_stride < 1) return fail(PB_ERR_INVALID, "bad argument");
    host_parallel(n, [=](int, int64_t lo, int64_t hi) { for (int64_t i = lo; i < hi; ++i) dst[i * dst_stride] = src[i * src_stride]; });
    return PB_OK;
}

int32_t pb_host_min_max_f64(const double* p, int64_t n, double* mn, double* mx, int32_t* has_nan) {
    if (n < 0 || (n && !p) || !mn || !mx || !has_nan) return fail(PB_ERR_INVALID, "bad argument");
    double lo_[8], hi_[8];
    int nan_[8];
    for (int k = 0; k < 8; ++k) { lo_[k] = HUGE_VAL; hi_[k] = -HUGE_VAL; nan_[k] = 0; }
    host_parallel(n, [&](int k, int64_t lo, int64_t hi) {
        double a = HUGE_VAL, b = -HUGE_VAL;
        int any = 0;
        for (int64_t i = lo; i < hi; ++i) {
            const double v = p[i];
            any |= (v != v);
            a = v < a ? v : a;  // (comparisons with NaN are false: NaNs are skipped)
            b = v > b ? v : b;
        }
        lo_[k] = a; hi_[k] = b; nan_[k] = any;
    });
    double a = HUGE_VAL, b = -HUGE_VAL;
    int any = 0;
    for (int k = 0; k < 8; ++k) { a = lo_[k] < a ? lo_[k] : a; b = hi_[k] > b ? hi_[k] : b; any |= nan_[k]; }
    *mn = a; *mx = b; *has_nan = any;
    return PB_OK;
}

int64_t pb_host_count_keep(const int32_t* state, int64_t n, int32_t delete_state) {
    if (n < 0 || (n && !state)) return -1;
    long long part[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    host_parallel(n, [&](int k, int64_t lo, int64_t hi) {
        long long c = 0;
        for (int64_t i = lo; i < hi; ++i) c += state[i] != delete_state;
        part[k] = c;
    });
    long long tot = 0;
    for (int k = 0; k < 8; ++k) tot += part[k];
    return tot;
}

int32_t pb_host_compact(const int32_t* state, int64_t n, int32_t delete_state, int32_t ncols, const void* const* src,
                        void* const* dst, const int64_t* row_bytes) {
    if (n < 0 || ncols < 0 || (n && !state) || (ncols && (!src || !dst || !row_bytes))) return fail(PB_ERR_INVALID, "bad argument");
    // pass 1: kept rows per thread segment (the segments of pass 2 are the same: host_parallel is deterministic in n)
    int64_t seg_lo[8], seg_keep[8];
    for (int k = 0; k < 8; ++k) { seg_lo[k] = -1; seg_keep[k] = 0; }
    host_parallel(n, [&](int k, int64_t lo, int64_t hi) {
        int64_t c = 0;
        for (int64_t i = lo; i < hi; ++i) c += state[i] != delete_state;
        seg_lo[k] = lo; seg_keep[k] = c;
    });
    int64_t offs[8], acc = 0;
    for (int k = 0; k < 8; ++k) { offs[k] = acc; acc += seg_keep[k]; }
    // pass 2: every thread copies the kept RUNS of its segment (deletions are sparse: long memcpy runs)
    host_parallel(n, [&](int k, int64_t lo, int64_t hi) {
        int64_t out = offs[k], i = lo;
        while (i < hi) {
            while (i < hi && state[i] == delete_state) ++i;
            int64_t j = i;
            while (j < hi && state[j] != delete_state) ++j;
            if (j > i) {
                for (int c = 0; c < ncols; ++c) {
                    const int64_t rb = row_bytes[c];
                    memcpy((char*)dst[c] + out * rb, (const char*)src[c] + i * rb, (size_t)((j - i) * rb));
                }
                out += j - i;
            }
            i = j;
        }
    });
    return PB_OK;
}

}  // extern "C"
