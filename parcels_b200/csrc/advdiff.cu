// advdiff.cu -- AdvectionDiffusionM1 / AdvectionDiffusionEM (reference kernels/_advectiondiffusion.py:11-18,21-117)
// inside Kernel.execute's loop (reference _core/kernel.py:174-247), one lane per particle, on rectilinear grids:
// fieldset.UV with XLinear_Velocity (AGridPolicy MODE 0) or -- the kernels are grid-agnostic in the reference -- with
// CGrid_Velocity (CGridPolicy, cgrid.cuh), and the scalar diffusivity fields Kh_zonal / Kh_meridional with XLinear (MODE 3)
// on the same grid.
//
// Per particle and loop iteration the reference evaluates, at float32 positions (particles.x + fieldset.dres is a
// float32 array plus a weak Python float):
//   M1:  Kh_zonal(x+dres), Kh_zonal(x-dres), UV(x), Kh_zonal(x), Kh_meridional(y+dres), Kh_meridional(y-dres), Kh_meridional(y)
//   EM:  UV(x) first, then the same six scalar evaluations
// Every evaluation raises particles.state like any Field.eval (numeric max, field.py:327-378) and overwrites
// particles.ei; the LAST one is Kh_meridional at the particle's own position, so that is the cell `ei` ends up with.
// The six scalar samples sit in up to five different cells, so the one-block corner cache of the scalar context is
// simply refilled for every sample (16 scattered loads); only the UV block is kept across steps.
#ifndef PB_SMEM_CACHE
#define PB_SMEM_CACHE
#endif
#include "agrid.cuh"
#include "cgrid.cuh"

struct AdvDiffParams {
    AdvectParams base;  // grid, UV field, particles, dt, endtime, seed, rng_call, max_iters, delete_on_error, report
    FieldDev fkz, fkm;  // Kh_zonal, Kh_meridional (p[0] only)
    int em;             // 0: Milstein (M1), 1: Euler-Maruyama (EM)
    int spherical;      // Kh_zonal.grid._mesh.is_spherical(): same grid as UV
    float dres_f32;     // fieldset.dres as the float32 it becomes in `particles.x + fieldset.dres`
    float pad_;
    double two_dres;    // 2 * fieldset.dres (Python float arithmetic)
    double deg2m;       // Kh_zonal.grid.deg2m
    double deg2m_sq;    // pow(deg2m, 2) as Python computes it
    int* iters;         // time-windowed fields: each lane's iteration count, kept across the resumed launches of one call (else NULL)
};

// NumPy-typed scalar helpers on tagged values: Python scalars are weak (cast to the array dtype first)
__device__ __forceinline__ Val v_sub(const Val& a, const Val& b) {
    if (a.f32 && b.f32) return Val{(double)((float)a.v - (float)b.v), true};
    return Val{a.v - b.v, false};
}
__device__ __forceinline__ Val v_add(const Val& a, const Val& b) {
    if (a.f32 && b.f32) return Val{(double)((float)a.v + (float)b.v), true};
    return Val{a.v + b.v, false};
}
__device__ __forceinline__ Val v_div_weak(const Val& a, double c) { return a.f32 ? Val{(double)((float)a.v / (float)c), true} : Val{a.v / c, false}; }
__device__ __forceinline__ Val v_div_f32(const Val& a, float c) { return a.f32 ? Val{(double)((float)a.v / c), true} : Val{a.v / (double)c, false}; }
__device__ __forceinline__ Val v_mul_weak(double c, const Val& a) { return a.f32 ? Val{(double)((float)c * (float)a.v), true} : Val{c * a.v, false}; }
__device__ __forceinline__ Val v_sqrt(const Val& a) { return a.f32 ? Val{(double)sqrtf((float)a.v), true} : Val{sqrt(a.v), false}; }

// CG: fieldset.UV is a CGrid_Velocity field (its two-face cache lives in registers: no shared-memory UV block)
template <class A, class D, class DK, bool HT, bool KHT, bool CG>
__global__ void __launch_bounds__(PB_BLOCK_THREADS, 2) advdiff_kernel(const AdvDiffParams q) {
    const AdvectParams& p = q.base;
    using PolUV = typename std::conditional<CG, CGridPolicy<A, D, 2>, AGridPolicy<A, D, HT, 2, 0>>::type;
    using PolK = AGridPolicy<A, DK, KHT, 1, 3>;
    using SU = typename decltype(EvalCtx<A, D, 2>::cor)::S;
    using SK = typename decltype(EvalCtx<A, DK, 1>::cor)::S;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long my_steps = 0, my_refills = 0;
    int final_state = 0;
    long long my_iters = 0;
    bool errored = false, deleted = false, oot = false, wait_window = false, migrate = false;
    long long err_iter = LLONG_MAX;

    if (i < p.P.n) {
        float x = p.P.x[i], y = p.P.y[i], z = p.P.z[i];
        float dx = p.P.dx[i], dy = p.P.dy[i], dz = p.P.dz[i];
        double t = p.P.t[i];
        const long long pid = p.P.pid[i];

        typename PolUV::Ctx eu;
        typename PolK::Ctx ek;
        PolUV::init(eu, p, p.P.ei[i]);
        PolK::init(ek, p, p.P.ei[i]);
        {   // the scalar context's corner block lives behind the UV blocks of the whole thread block
            extern __shared__ __align__(16) unsigned char pb_smem[];
            ek.cor.sm = reinterpret_cast<SK*>(pb_smem + (CG ? (size_t)0 : (size_t)2 * 16 * sizeof(SU) * PB_BLOCK)) + threadIdx.x;
        }
        int state = p.resume ? p.P.state[i] : (int)PB_EVALUATE;  // kernel.py:188
        eu.refills = 0; ek.refills = 0;
        eu.out_of_time = false; ek.out_of_time = false;
        const int sign = p.dt > 0 ? 1 : -1;

        // one Field.eval of a diffusivity field at float32 positions (field.py:144-191)
        auto evalK = [&](const FieldDev& fk, float zs, float ys, float xs) -> Val {
            Val val, d0, d1;
            ek.state = state;
            ek.cor.ti = INT_MIN;  // other field / other cell: always gather
            eval_uvw<A, DK, KHT, 1, 3, float, float, float>(p.g, fk, ek, t, zs, ys, xs, val, d0, d1);
            state = ek.state;
            return val;
        };

        // a resumed launch of the same Kernel.execute call (time-slab streaming) continues the lane's iteration count: the
        // Wiener increments (keyed by it), the first-iteration batch rule and max_iters are those of the resident run
        long long it = (q.iters && p.resume && !p.kernels_only) ? (long long)q.iters[i] : 0;
        for (;; ++it) {
            if (p.max_iters >= 0 && it >= p.max_iters) break;
            const double tte = sign * (p.endtime - t);                                    // kernel.py:191
            if (!((state == PB_SUCCESS || state == PB_EVALUATE) && tte >= 0)) break;      // :193-195
            // mode D: not ours (any more) -- before the window wait, as in advect_kernel
            if (p.g.decomposed && !((double)x >= p.g.own_lo && (double)x < p.g.own_hi)) {
                migrate = true;
                break;
            }
            const double dtp = (sign == 1) ? fmax(fmin(p.dt, tte), 0.0) : fmin(fmax(p.dt, -tte), 0.0);  // :199-203
            // every sample of M1 / EM is taken at the particle's own time (_advectiondiffusion.py:40-60,87-110): t must lie
            // within the resident time levels; outside the field's whole time interval is OutsideTimeInterval, not a wait
            if (p.f.windowed && !(t >= p.f.win_t0 && t <= p.f.win_t1) && t >= 0 && t <= p.g.time_len) {
                wait_window = true;
                atomicMin(&p.rep->wait_t_min_bits, (unsigned long long)__double_as_longlong(t));
                atomicMax(&p.rep->wait_t_max_bits, (unsigned long long)__double_as_longlong(t));
                break;
            }
            my_steps++;
            if constexpr (std::is_same<A, float>::value) {
                // float32 grids: every sample of this kernel is taken at the particle's own time with float32 positions; in the
                // call's first iteration the batch may mix tau == 0 (first time level) with tau > 0: lenT = 2 for all of it
                const signed char lt = (it == 0 && (p.batch_levels & 1)) ? 1 : -1;
                eu.len_t = lt; ek.len_t = lt;
            }

            // Wiener increments: N(0, sqrt(|dt|))
            double zx, zy;
            wiener_normals(p.seed, p.rng_call, it, pid, zx, zy);
            const double sq = sqrt(fabs(dtp));
            const double dWx = zx * sq, dWy = zy * sq;

            Val u = Val{0.0, false}, v = u, wdummy = u;
            auto evalUV = [&]() {
                eu.state = state;
                PolUV::template eval<float, float, float>(p, eu, false, t, z, y, x, u, v, wdummy);
                state = eu.state;
            };
            float m2 = 1.f;  // pow(deg2m * cos(lat * pi / 180), 2) in float32 (meters_to_degrees_zonal, :11-13)
            if (q.spherical) {
                const float ang = (y * (float)3.14159265358979323846) / 180.0f;
                const float m = (float)q.deg2m * cosf(ang);
                m2 = m * m;
            }
            if (q.em) evalUV();
            Val Kxp1 = evalK(q.fkz, z, y, x + q.dres_f32);
            Val Kxm1 = evalK(q.fkz, z, y, x - q.dres_f32);
            if (q.spherical) { Kxp1 = v_div_f32(Kxp1, m2); Kxm1 = v_div_f32(Kxm1, m2); }
            const Val dKdx = v_div_weak(v_sub(Kxp1, Kxm1), q.two_dres);
            if (!q.em) evalUV();
            Val khz = evalK(q.fkz, z, y, x);
            if (q.spherical) khz = v_div_f32(khz, m2);
            const Val bx = v_sqrt(v_mul_weak(2.0, khz));
            Val Kyp1 = evalK(q.fkm, z, y + q.dres_f32, x);
            Val Kym1 = evalK(q.fkm, z, y - q.dres_f32, x);
            if (q.spherical) { Kyp1 = v_div_weak(Kyp1, q.deg2m_sq); Kym1 = v_div_weak(Kym1, q.deg2m_sq); }
            const Val dKdy = v_div_weak(v_sub(Kyp1, Kym1), q.two_dres);
            Val khm = evalK(q.fkm, z, y, x);
            if (q.spherical) khm = v_div_weak(khm, q.deg2m_sq);
            const Val by = v_sqrt(v_mul_weak(2.0, khm));
            // mode D: a sample (UV, or Kh at x +- dres) left the owned + halo columns: the lane stops with state 99 before the
            // delete handler below could turn it into a deletion
            if (p.g.decomposed && state == 99) break;

            double sx, sy;  // the right-hand sides of `particles.dx += ...`, float64 (particles.dt is float64)
            if (q.em) {     // ax * dt + bx * dWx   (:85,101,115-117)
                const Val ax = v_add(u, dKdx), ay = v_add(v, dKdy);
                sx = ax.v * dtp + bx.v * dWx;
                sy = ay.v * dtp + by.v * dWy;
            } else {        // u * dt + 0.5 * dKdx * (dWx**2 + dt) + bx * dWx   (:64-66)
                sx = (u.v * dtp + v_mul_weak(0.5, dKdx).v * (dWx * dWx + dtp)) + bx.v * dWx;
                sy = (v.v * dtp + v_mul_weak(0.5, dKdy).v * (dWy * dWy + dtp)) + by.v * dWy;
            }
            dx = (float)((double)dx + sx);
            dy = (float)((double)dy + sy);

            if (p.kernels_only) { ++it; break; }  // mixed lists: the host finishes the iteration (stepwise.py)
            if (p.delete_on_error && state >= 50) state = PB_DELETE;
            if (state == PB_EVALUATE || state == PB_SUCCESS) {  // kernel.py:108-116,220-222
                x = x + dx; y = y + dy; z = z + dz;
                t = t + dtp;
                dx = 0.f; dy = 0.f; dz = 0.f;
            }
            if (state == PB_EVALUATE && t == p.endtime) state = PB_END_OF_LOOP;  // :229-230
            if (state == PB_DELETE) { deleted = true; ++it; break; }
            if (state >= 50) { errored = true; err_iter = it; ++it; break; }
        }
        PolK::finish(ek, p);   // ei of the last evaluation (Kh_meridional at the particle's position)
        my_iters = it;
        my_refills = (unsigned long long)eu.refills + ek.refills;
        oot = eu.out_of_time || ek.out_of_time;
        final_state = state;
        p.P.x[i] = x; p.P.y[i] = y; p.P.z[i] = z;
        p.P.dx[i] = dx; p.P.dy[i] = dy; p.P.dz[i] = dz;
        p.P.t[i] = t;
        p.P.state[i] = state;
        p.P.ei[i] = ek.ei;
        if (q.iters) q.iters[i] = (int)it;
        if (migrate && p.mig.on) {
            MigRecord rec;
            rec.t = t; rec.pid = pid;
            rec.x = x; rec.y = y; rec.z = z; rec.dx = dx; rec.dy = dy; rec.dz = dz;
            rec.state = state; rec.ei = ek.ei;
            migrate = mig_deliver(p, i, rec, MigResume{0.0, 0.0, (int)it, 0});
        }
    }

    const unsigned full = 0xffffffffu;
    unsigned long long s_steps = my_steps, s_ref = my_refills;
    unsigned n_err = errored, n_del = deleted, n_oot = oot, n_ww = wait_window, n_mig = migrate;
    // with the delete handler an out-of-interval sample is not an error of the lane, but the host still needs the iteration
    // it happened in (the reference deletes the WHOLE evaluated view of that iteration, field.py:31-44)
    long long mx_it = my_iters, mn_err = (oot && deleted) ? my_iters - 1 : err_iter;
    int mx_state = final_state;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s_steps += __shfl_xor_sync(full, s_steps, o);
        s_ref += __shfl_xor_sync(full, s_ref, o);
        n_err += __shfl_xor_sync(full, n_err, o);
        n_del += __shfl_xor_sync(full, n_del, o);
        n_oot += __shfl_xor_sync(full, n_oot, o);
        n_ww += __shfl_xor_sync(full, n_ww, o);
        n_mig += __shfl_xor_sync(full, n_mig, o);
        mx_it = max(mx_it, __shfl_xor_sync(full, mx_it, o));
        mn_err = min(mn_err, __shfl_xor_sync(full, mn_err, o));
        mx_state = max(mx_state, __shfl_xor_sync(full, mx_state, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (s_steps) atomicAdd(&p.rep->particle_steps, s_steps);
        if (s_ref) atomicAdd(&p.rep->cache_refills, s_ref);
        if (n_err) atomicAdd(&p.rep->n_error, (unsigned long long)n_err);
        if (n_del) atomicAdd(&p.rep->n_deleted, (unsigned long long)n_del);
        if (n_oot) atomicAdd(&p.rep->n_out_of_time, (unsigned long long)n_oot);
        if (n_ww) atomicAdd(&p.rep->n_wait_window, (unsigned long long)n_ww);
        if (n_mig) atomicAdd(&p.rep->n_migrate, (unsigned long long)n_mig);
        if (mx_it) atomicMax(&p.rep->max_iters_done, mx_it);
        if (mn_err != LLONG_MAX) atomicMin(&p.rep->first_error_iter, mn_err);
        if (mx_state) atomicMax(&p.rep->max_state, mx_state);
    }
}

template <class A, class D, class DK, bool HT, bool KHT, bool CG>
static cudaError_t launch1(const AdvDiffParams& q, cudaStream_t s) {
    using SU = typename decltype(EvalCtx<A, D, 2>::cor)::S;
    using SK = typename decltype(EvalCtx<A, DK, 1>::cor)::S;
    const size_t smem = ((CG ? (size_t)0 : (size_t)2 * 16 * sizeof(SU)) + (size_t)16 * sizeof(SK)) * PB_BLOCK;
    if (smem > 48 * 1024) {
        cudaError_t ce = cudaFuncSetAttribute(advdiff_kernel<A, D, DK, HT, KHT, CG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (ce != cudaSuccess) return ce;
    }
    advdiff_kernel<A, D, DK, HT, KHT, CG><<<(unsigned)((q.base.P.n + PB_BLOCK - 1) / PB_BLOCK), PB_BLOCK, smem, s>>>(q);
    return cudaGetLastError();
}

template <class A, class D, class DK, bool CG>
static cudaError_t launch_t(const AdvDiffParams& q, bool ht, bool kht, cudaStream_t s) {
    if (CG) {  // (CGridPolicy handles the time axis at run time: the HT instantiation only types the unused A-grid context)
        return kht ? launch1<A, D, DK, true, true, CG>(q, s) : launch1<A, D, DK, true, false, CG>(q, s);
    }
    if (ht) return kht ? launch1<A, D, DK, true, true, CG>(q, s) : launch1<A, D, DK, true, false, CG>(q, s);
    return launch1<A, D, DK, false, false, CG>(q, s);  // no time axis on the grid: no field can have a time dimension
}
template <class A, bool CG>
static cudaError_t launch_a(const AdvDiffParams& q, bool d64, bool k64, bool ht, bool kht, cudaStream_t s) {
    if (d64) return k64 ? launch_t<A, double, double, CG>(q, ht, kht, s) : launch_t<A, double, float, CG>(q, ht, kht, s);
    return k64 ? launch_t<A, float, double, CG>(q, ht, kht, s) : launch_t<A, float, float, CG>(q, ht, kht, s);
}

// scheme 0 = M1, 1 = EM.  uv_/kh_: dtype and time dimension of U,V and of the two Kh fields.
cudaError_t launch_advdiff(const AdvectParams& p, const FieldDev& fkz, const FieldDev& fkm, int em, double dres, double deg2m_sq,
                           bool coord_f64, bool uv_f64, bool kh_f64, bool uv_time, bool kh_time, bool cgrid, int* iters, cudaStream_t s) {
    AdvDiffParams q{};
    q.base = p;
    q.iters = iters;
    q.fkz = fkz; q.fkm = fkm;
    q.em = em;
    q.spherical = p.g.spherical;
    q.dres_f32 = (float)dres;
    q.two_dres = 2 * dres;
    q.deg2m = p.g.deg2m;
    q.deg2m_sq = deg2m_sq;
    if (cgrid) return coord_f64 ? launch_a<double, true>(q, uv_f64, kh_f64, uv_time, kh_time, s) : launch_a<float, true>(q, uv_f64, kh_f64, uv_time, kh_time, s);
    return coord_f64 ? launch_a<double, false>(q, uv_f64, kh_f64, uv_time, kh_time, s) : launch_a<float, false>(q, uv_f64, kh_f64, uv_time, kh_time, s);
}
