// rk45.cuh -- the AdvectionRK45 kernel template (see rk45.cu for the restated algorithm), shared by the A-grid launcher
// (rk45.cu) and the C-grid / curvilinear launcher (cgrid.cu).
#pragma once
#include "common.cuh"

struct Rk45Params {
    AdvectParams base;   // grid, field, particles, dt (sign), endtime, max_iters, report
    double* dt;          // per-particle dt (particles.dt, float64)
    double* next_dt;     // per-particle next_dt, widened to float64
    int* iters;          // loop iterations each particle took part in (for the batch-level clamp, below); a launch that
                         // continues the previous one after a time-window wait (resume without kernels_only) starts from it
    int next_dt_f32;     // the Particle's next_dt Variable is float32 (the default dtype): round on assignment
    double tol, min_dt, max_dt;
};

// value * python-float constant: float32 arithmetic when the value is a float32 array element (weak scalar)
__device__ __forceinline__ double mulc(const Val& a, double c) { return a.f32 ? (double)((float)a.v * (float)c) : a.v * c; }

template <class Policy>
__global__ void __launch_bounds__(PB_BLOCK_THREADS, PB_MINBLOCKS) rk45_kernel(const Rk45Params q) {
    const AdvectParams& p = q.base;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    LaneTally tally;  // refills: the number of field evaluations (6 per attempt)
    if (i < p.P.n) {
        // Butcher tableau of _advection.py:96-106, the same Python float expressions
        const double c[5] = {1.0 / 4.0, 3.0 / 8.0, 12.0 / 13.0, 1.0, 1.0 / 2.0};
        const double A[5][5] = {{1.0 / 4.0, 0.0, 0.0, 0.0, 0.0},
                                {3.0 / 32.0, 9.0 / 32.0, 0.0, 0.0, 0.0},
                                {1932.0 / 2197.0, -7200.0 / 2197.0, 7296.0 / 2197.0, 0.0, 0.0},
                                {439.0 / 216.0, -8.0, 3680.0 / 513.0, -845.0 / 4104.0, 0.0},
                                {-8.0 / 27.0, 2.0, -3544.0 / 2565.0, 1859.0 / 4104.0, -11.0 / 40.0}};
        const double b4[5] = {25.0 / 216.0, 0.0, 1408.0 / 2565.0, 2197.0 / 4104.0, -1.0 / 5.0};
        const double b5[6] = {16.0 / 135.0, 0.0, 6656.0 / 12825.0, 28561.0 / 56430.0, -9.0 / 50.0, 2.0 / 55.0};

        Lane L = load_lane(p, i);
        float &x = L.x, &y = L.y, &z = L.z, &dx = L.dx, &dy = L.dy, &dz = L.dz;
        double& t = L.t;
        double dt = q.dt[i], ndt = q.next_dt[i];
        typename Policy::Ctx e;
        Policy::init(e, p, p.P.ei[i]);
        e.state = initial_state(p, i);
        e.refills = 0;
        e.out_of_time = false;
        if constexpr (Policy::BATCH_LEN_Z) {
            if (p.batch_levels & PB_BATCH_TWO_Z) e.len_z = 1;
        }
        const int sign = p.dt > 0 ? 1 : -1;  // compute_time_direction (kernel.py:186)
        bool first_attempt = true, halo = false;
        // a resumed launch of the same Kernel.execute call (time-slab streaming) continues the lane's iteration count, so the
        // first-iteration batch rules, max_iters and the finalize clamp see the iterations of the whole call
        long long it = (p.resume && !p.kernels_only) ? (long long)q.iters[i] : 0;
        [[maybe_unused]] int mig_col = -1;  // column slabs: the column of the cell a leaving lane's search found
        for (;; ++it) {
            if (p.max_iters >= 0 && it >= p.max_iters) break;
            const double tte = sign * (p.endtime - t);
            if (!((e.state == PB_SUCCESS || e.state == PB_EVALUATE) && tte >= 0)) break;
            // mode D: not ours (any more).  Tested before the window wait: the new owner, whose window slides in lock-step with this
            // one, makes the same wait decision
            if constexpr (columns_v<Policy>) {
                // column slabs: the owner of the cell the first attempt's first search finds (that search, run here and reused)
                const int col = Policy::owner_search(p, e, it == 0 && first_attempt && p.hint_all_zero, x, y);
                if (col >= 0 && !((double)col >= p.g.own_lo && (double)col < p.g.own_hi)) {
                    tally.migrate = true;
                    mig_col = col;
                    break;
                }
            } else if (p.g.decomposed && !((double)x >= p.g.own_lo && (double)x < p.g.own_hi)) {
                tally.migrate = true;
                break;
            }
            dt = clamp_dt(dt, tte, sign);
            if (dt == 0.0 && tte > 0) {  // the reference never terminates here (t cannot advance): report instead of spinning
                tally.stalled = true;
                break;
            }
            // every attempt of this iteration samples inside [t, t + dt] (a rejected attempt halves dt); a wait leaves state, dt and
            // next_dt as they are
            if (window_wait(p, t, t + dt, t)) {
                tally.wait_window = true;
                break;
            }
            tally.steps++;
            do {  // kernel.py:206-216: the kernel, then again for as long as it asks to be repeated
                const double sgn_dt = dt > 0 ? 1.0 : (dt < 0 ? -1.0 : 0.0);  // np.sign(particles.dt)
                Val u[6], v[6], wdummy;
                // curvilinear grids: the reference skips the hint test of a whole batch whose hinted xi are all 0
                // (index_search.py:269) -- the first evaluation of the call (the host passes hint_all_zero)
                const bool first_batch = it == 0 && first_attempt;  // the first attempt of the first iteration: the whole evaluated view
                const bool nohint1 = first_batch && p.hint_all_zero;
                first_attempt = false;
                if constexpr (Policy::RUNTIME_DTYPE) {
                    // ONE eval call site (the policy branches at run time on the position dtype): the six evaluations of the
                    // heavy curvilinear search + C-grid code share their instructions
#pragma unroll 1
                    for (int k = 0; k < 6; ++k) {
                        double xs = (double)x, ys = (double)y, ts = t;
                        if (k > 0) {
                            double sx = mulc(u[0], A[k - 1][0]), sy = mulc(v[0], A[k - 1][0]);
                            for (int j = 1; j < k; ++j) {
                                sx = sx + u[j].v * A[k - 1][j];
                                sy = sy + v[j].v * A[k - 1][j];
                            }
                            xs = (double)x + sx * dt;
                            ys = (double)y + sy * dt;
                            ts = t + c[k - 1] * dt;
                        }
                        if constexpr (Policy::BATCH_LEN_T) e.len_t = (k == 0 && first_batch && (p.batch_levels & 1)) ? 1 : -1;
                        Policy::eval_rt(p, e, k == 0 && nohint1, ts, (double)z, ys, xs, /*xy_f32=*/k == 0, /*z_f32=*/true, u[k], v[k], wdummy);
                    }
                } else {
                if constexpr (Policy::BATCH_LEN_T) e.len_t = (first_batch && (p.batch_levels & 1)) ? 1 : -1;  // see common.cuh, stage 1
                Policy::template eval<float, float, float>(p, e, nohint1, t, z, y, x, u[0], v[0], wdummy);
                if constexpr (Policy::BATCH_LEN_T) e.len_t = -1;
#pragma unroll 1
                for (int k = 0; k < 5; ++k) {
                    double sx = mulc(u[0], A[k][0]), sy = mulc(v[0], A[k][0]);
                    for (int j = 1; j <= k; ++j) {
                        sx = sx + u[j].v * A[k][j];
                        sy = sy + v[j].v * A[k][j];
                    }
                    const double xs = (double)x + sx * dt, ys = (double)y + sy * dt;
                    Policy::template eval<float, double, double>(p, e, false, t + c[k] * dt, z, ys, xs, u[k + 1], v[k + 1], wdummy);
                }
                }
                tally.refills += 6;
                // mode D: a stage position left the owned + halo columns (state 99, which the line `e.state = good ? ...` below
                // would overwrite): the lane stops with it
                if (p.g.decomposed && e.state == 99) {
                    halo = true;
                    break;
                }
                double x4 = mulc(u[0], b4[0]), y4 = mulc(v[0], b4[0]), x5 = mulc(u[0], b5[0]), y5 = mulc(v[0], b5[0]);
                for (int j = 1; j < 5; ++j) {
                    x4 = x4 + u[j].v * b4[j];
                    y4 = y4 + v[j].v * b4[j];
                }
                for (int j = 1; j < 6; ++j) {
                    x5 = x5 + u[j].v * b5[j];
                    y5 = y5 + v[j].v * b5[j];
                }
                x4 = x4 * dt; y4 = y4 * dt; x5 = x5 * dt; y5 = y5 * dt;
                const double ex = x5 - x4, ey = y5 - y4;
                const double kappa = sqrt(ex * ex + ey * ey);  // np.pow(., 2) with a scalar exponent 2 is a square
                const bool good = (kappa <= q.tol) || (fabs(dt) <= fabs(q.min_dt));
                dx = (float)((double)dx + (good ? x5 : 0.0));
                dy = (float)((double)dy + (good ? y5 : 0.0));
                const bool inc = good && (kappa <= q.tol / 10) && (fabs(dt * 2) <= fabs(q.max_dt));
                ndt = inc ? dt * 2 : dt;
                if (q.next_dt_f32) ndt = (double)(float)ndt;  // stored into the float32 Variable
                if (fabs(ndt) > fabs(q.max_dt)) {
                    ndt = q.max_dt * sgn_dt;
                    if (q.next_dt_f32) ndt = (double)(float)ndt;
                }
                e.state = good ? (int)PB_EVALUATE : (int)PB_REPEAT;
                if (!good) dt = dt / 2;
                // applied to every particle of the view, accepted ones included (:148-153): an accepted step whose
                // clamped dt is below min_dt still advances t by min_dt in the position update
                if (fabs(dt) < fabs(q.min_dt)) dt = q.min_dt * sgn_dt;
            } while (e.state == PB_REPEAT);
            if (halo) break;
            if (p.kernels_only) { ++it; break; }  // mixed lists: the host finishes the iteration (stepwise.py)
            if (p.delete_on_error && e.state >= 50) e.state = PB_DELETE;  // never true after RK45 (see the header comment)
            if (e.state == PB_EVALUATE || e.state == PB_SUCCESS) {
                x = x + dx; y = y + dy; z = z + dz;
                t = t + dt;
                dx = 0.f; dy = 0.f; dz = 0.f;
                dt = ndt;  // kernel.py:118-120
            }
            if (e.state == PB_EVALUATE && t == p.endtime) e.state = PB_END_OF_LOOP;
        }
        Policy::finish(e, p);
        tally.iters = it;
        tally.state = tally.stalled ? (int)PB_ERROR : e.state;
        store_lane(p, i, L, tally.state, e.ei);
        q.dt[i] = dt;
        q.next_dt[i] = ndt;
        q.iters[i] = (int)it;
        if (tally.migrate && p.mig.on) {
            const MigResume rs{dt, ndt, (int)it, 0};
            if constexpr (columns_v<Policy>) tally.migrate = mig_deliver_column(p, i, mig_col, L, tally.state, e.ei, &rs);
            else tally.migrate = mig_deliver(p, i, L, tally.state, e.ei, &rs);
        }
    }
    publish(tally, p.rep);
}
