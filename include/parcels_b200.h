/* parcels_b200.h -- C-ABI of libparcels_b200.so: the H100 (sm_90a) replacement for the hot path
 * ParticleSet.execute(AdvectionRK4 | AdvectionRK4_3D | AdvectionEE | AdvectionRK2[_3D] [+ DiffusionUniformKh]
 *                     | AdvectionRK45 | AdvectionDiffusionM1 | AdvectionDiffusionEM   [+ delete-on-error handler])
 * on rectilinear A-grids (XLinear_Velocity, XFreeslip, XPartialslip, nearest node) and rectilinear / curvilinear
 * C-grids (CGrid_Velocity), plus Field.eval / VectorField.eval sampling, the ParticleFile row selection and the
 * multi-GPU particle migration.
 *
 * The reference (Parcels v4-alpha, pure Python/NumPy) has no FFI; this header DEFINES the
 * drop-in boundary (SURVEY.md 8b).  Each entry point cites the reference interface it
 * replaces (paths relative to /root/reference/src/parcels).  All functions return 0 on
 * success and a negative pb_status on failure; pb_last_error_string() describes the failure.
 * One engine per GPU; an engine is driven by one host thread; all device work is ordered on
 * an engine-owned CUDA stream.  Plain pointers and sizes only -- no torch / numpy types.
 */
#ifndef PARCELS_B200_H
#define PARCELS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB_ABI_VERSION 1
#define PB_MAX_FIELDS 16 /* field slots per engine: 0..2 = U, V, W; 3.. = scalar fields */

typedef struct pb_engine pb_engine;

enum pb_status {
    PB_OK = 0,
    PB_ERR_INVALID = -1,     /* bad argument / unsupported configuration                      */
    PB_ERR_CUDA = -2,        /* CUDA runtime error (message in pb_last_error_string)           */
    PB_ERR_STATE = -3,       /* call order violated (e.g. advect before grid/field upload)     */
    PB_ERR_NO_DEVICE = -4    /* no CUDA device: there is NO CPU fallback                       */
};

/* Velocity-field slots (VectorField components, _core/field.py:198-240). */
enum pb_field_slot { PB_FIELD_U = 0, PB_FIELD_V = 1, PB_FIELD_W = 2 };

/* Advection scheme (kernels/_advection.py). */
enum pb_scheme {
    PB_ADVECTION_NONE = 0,    /* no advection kernel in the list (e.g. [DiffusionUniformKh] alone) */
    PB_ADVECTION_EE = 1,      /* :78-82   */
    PB_ADVECTION_RK2 = 2,     /* :20-27   */
    PB_ADVECTION_RK2_3D = 3,  /* :30-39   */
    PB_ADVECTION_RK4 = 4,     /* :42-55   */
    PB_ADVECTION_RK4_3D = 5,  /* :58-75   */
    PB_ADVECTION_RK45 = 6     /* :85-155: adaptive step, own entry point pb_advect_rk45 */
};

/* Particle status codes written by the device: identical to _core/statuscodes.py:19-34. */
enum pb_state {
    PB_SUCCESS = 0, PB_END_OF_LOOP = 1, PB_EVALUATE = 10, PB_REPEAT = 20, PB_DELETE = 30,
    PB_STOP_EXECUTION = 40, PB_STOP_ALL_EXECUTION = 41, PB_ERROR = 50, PB_ERROR_INTERPOLATION = 51,
    PB_ERROR_GRID_SEARCHING = 52, PB_ERROR_OUT_OF_BOUNDS = 60, PB_ERROR_THROUGH_SURFACE = 61,
    PB_ERROR_OUTSIDE_TIME_INTERVAL = 70
};

/* ---- engine life cycle ------------------------------------------------------------------ */
int32_t pb_abi_version(void);
const char* pb_last_error_string(void);
int32_t pb_device_count(void);
/* Creates an engine on CUDA device `device` (fails with PB_ERR_NO_DEVICE when there is none). */
int32_t pb_engine_create(int32_t device, pb_engine** out);
void pb_engine_destroy(pb_engine* e);
/* Blocks until all work queued on the engine's stream has finished. */
int32_t pb_engine_synchronize(pb_engine* e);

/* Device timing on the engine's own stream (torch.cuda.Event only sees torch's streams):
 * begin records a CUDA event, end records a second one, waits for it and returns the elapsed ms. */
int32_t pb_timer_begin(pb_engine* e);
int32_t pb_timer_end_ms(pb_engine* e, float* ms);

/* ---- grid: replaces XGrid.search inputs (_core/xgrid.py:316-356) --------------------------
 * Rectilinear grid: 1-D node coordinates lon[nx], lat[ny], depth[nz] (depth may be NULL/nz=0:
 * the grid has no Z axis) of dtype float32 (coord_is_f64=0) or float64 (=1) -- the dtype is
 * part of the contract because the reference's arithmetic promotes on it
 * (_core/index_search.py:47-51).  time_s[nt]: seconds since the start of the field's time
 * interval (float64), nt<2 or NULL => the field has no time dimension
 * (_core/index_search.py:77-83).  xdim/ydim/zdim_cells: cell counts used by ravel_index
 * (_core/basegrid.py:83-118, _core/xgrid.py:21-24,208-231; depend on SGRID padding).
 * The engine copies everything to HBM; the host keeps ownership of its buffers. */
int32_t pb_grid_upload_rectilinear(pb_engine* e, const void* lon, int64_t nx, const void* lat, int64_t ny,
                                   const void* depth, int64_t nz, int32_t coord_is_f64,
                                   const double* time_s, int64_t nt, int32_t spherical, double deg2m,
                                   int64_t xdim_cells, int64_t ydim_cells, int64_t zdim_cells);

/* Curvilinear grid: 2-D node coordinates lon2d/lat2d of shape (ny, nx), C-contiguous.  Cell search =
 * hint test + spatial-hash fallback (_core/index_search.py:94-295).  The hash table is the CSR table
 * of _core/spatialhash.py:269-387 (unique Morton keys ascending, per-key start/count, flat face ids
 * j*(nx-1)+i ascending within a key), built ONCE on the host (parcels_b200/spatialhash.py) so that the
 * candidate order -- "first containing face wins", :511-535 -- is the reference's; hash_box6 =
 * (xmin, xmax, ymin, ymax, zmin, zmax) of the hash grid, hash_bitwidth the quantisation (:212-228);
 * face_qbox[(ny-1)*(nx-1)] = each face's quantised bounding box packed 6 x 10 bits (xlo | xhi<<10 | ylo<<20 |
 * yhi<<30 | zlo<<40 | zhi<<50), i.e. the set of hash cells the face is listed under (:269-300).
 * The query itself runs on the device.
 * hash_keys = hash_starts = hash_counts = hash_faces = NULL (n_keys, n_entries ignored): the table is BUILT ON THE DEVICE
 * from face_qbox (count -> scan -> expand -> 64-bit radix sort by (key, face) -> CSR, csrc/hashbuild.cu).  The float part of
 * the reference's constructor (:45-228: xyz in the coordinate dtype, per-face min/max, quantisation, bitwidth budget)
 * stays with the caller -- it is what fixes the boxes, and the table is a pure integer function of them, so both routes
 * give the reference's table bit for bit.  pb_hash_table_size / pb_hash_table_download read the resident table back. */
int32_t pb_grid_upload_curvilinear(pb_engine* e, const void* lon2d, const void* lat2d, int64_t ny, int64_t nx,
                                   const void* depth, int64_t nz, int32_t coord_is_f64, const double* time_s,
                                   int64_t nt, int32_t spherical, double deg2m, int64_t xdim_cells,
                                   int64_t ydim_cells, int64_t zdim_cells, const uint32_t* hash_keys,
                                   const int64_t* hash_starts, const int64_t* hash_counts, int64_t n_keys,
                                   const uint32_t* hash_faces, int64_t n_entries, const double* hash_box6,
                                   int32_t hash_bitwidth, const uint64_t* face_qbox);

int32_t pb_hash_table_size(pb_engine* e, int64_t* n_keys, int64_t* n_entries);
int32_t pb_hash_table_download(pb_engine* e, uint32_t* keys, int64_t* starts, int64_t* counts, uint32_t* faces);

/* Vector interpolator of fieldset.UV / UVW (VectorField.interp_method, _core/field.py:236-246):
 * XLinear_Velocity (A-grid, interpolators/_xinterpolators.py:169-190) or CGrid_Velocity (:193-332)
 * with the SGRID staggering offsets of _get_offsets_dictionary (:99-109: 1 for LOW padding).
 * Rectilinear A-grids also take XFreeslip / XPartialslip (_Spatialslip, :385-495) and the per-component
 * nearest-node interpolator (XNearest, :515-560, wrapped as XNearest_Velocity by the reference's
 * tests/test_interpolation.py:279-294). */
enum pb_interp {
    PB_INTERP_XLINEAR_VELOCITY = 0,
    PB_INTERP_CGRID_VELOCITY = 1,
    PB_INTERP_XFREESLIP = 2,
    PB_INTERP_XPARTIALSLIP = 3,
    PB_INTERP_XNEAREST_VELOCITY = 4
};
int32_t pb_set_interpolation(pb_engine* e, int32_t method, int32_t off_x, int32_t off_y, int32_t off_z);

/* ---- field data: replaces ModelData.field_data -> xarray .isel gathers -------------------
 * (_core/model.py:67-77, interpolators/_xinterpolators.py:25-96).  C-contiguous (T,Z,Y,X),
 * float32 or float64, NaNs already filled (model.py:135-143).  Size-1 dims are never indexed
 * (mock dims, _core/xgrid.py:71-105).  Staged through pinned memory, async H2D. */
int32_t pb_field_upload(pb_engine* e, int32_t slot, const void* data, int32_t data_is_f64, int64_t T,
                        int64_t Z, int64_t Y, int64_t X);
/* Same, but `data` is already a DEVICE pointer owned by the caller (e.g. a torch tensor) that
 * must outlive the engine's use of it; nothing is copied. */
int32_t pb_field_attach_device(pb_engine* e, int32_t slot, const void* dev_data, int32_t data_is_f64,
                               int64_t T, int64_t Z, int64_t Y, int64_t X);
int32_t pb_field_clear(pb_engine* e, int32_t slot);

/* Time-slab streaming -- GPU analogue of the reference's WindowedArray (_core/_windowed_array.py:25-97,
 * _core/model.py:79-113): keep only `window_levels` consecutive time levels of U, V, W in HBM.
 * pb_field_window_create allocates window_levels + 1 ring slots per component (level L lives in slot
 * L % (window_levels + 1)); pb_field_window_load copies ONE level (Z*Y*X values, host memory, ideally pinned)
 * into its slot asynchronously on a copy stream -- also while pb_advect_async is running, as long as that
 * level is outside the window in use; pb_field_window_set(first, n) declares levels [first, first+n) resident
 * for the next advect calls (stream-ordered after the pending loads).  pb_advect stops a particle whose next
 * step would sample outside the resident levels (pb_report.n_wait_window): slide the window and call
 * pb_advect again with resume = 1.  A step that straddles a time level samples 3 levels, so window_levels = 3 is
 * the general minimum (2 suffices only when no step straddles a level).  pb_advect_rk45 and pb_advect_diffusion
 * wait the same way (RK45: the span [t, t + dt] of the particle's clamped dt; M1 / EM: its time t) and are resumed the
 * same way; a resumed launch (resume = 1 without kernels_only) continues every particle's loop-iteration count, so the
 * result -- the Wiener increments of M1 / EM included -- is the resident one bit for bit.  pb_sample_velocity returns
 * PB_ERR_INVALID when a finite sample time inside the time axis lies outside the resident levels.
 * Scalar fields (slots 3..) stream the same way.  All windowed slots of one engine share one window_levels and the one
 * window that pb_field_window_set declares; an engine may window scalar slots only.  pb_sample_scalar on a windowed slot
 * returns PB_ERR_INVALID for a non-resident sample time as pb_sample_velocity does, and pb_advect_diffusion reads windowed
 * Kh slots through the window of U, V (which must then be windowed too). */
/* pb_field_window_create: slot 0 .. PB_MAX_FIELDS - 1; allocates and zeroes window_levels + 1 levels of the slot. */
int32_t pb_field_window_create(pb_engine* e, int32_t slot, int32_t data_is_f64, int64_t T_total, int64_t Z, int64_t Y,
                               int64_t X, int32_t window_levels);
/* pb_field_window_load: a slot made by pb_field_window_create (0 .. PB_MAX_FIELDS - 1); level < T_total. */
int32_t pb_field_window_load(pb_engine* e, int32_t slot, int64_t level, const void* host_level_data);
/* pb_field_window_set: the window of every windowed slot; first_level + n_levels <= the grid's time levels (nt). */
int32_t pb_field_window_set(pb_engine* e, int64_t first_level, int64_t n_levels);

/* ---- particles: replaces the SoA dict of create_particle_data (_core/particle.py:182-222)
 * Host arrays are the pset._data ndarrays themselves (x,y,z,dx,dy,dz float32; t float64;
 * state int32; ei = LAST column of the (N, ngrids) int32 `ei` array, _core/field.py:279;
 * particle_id int64).  upload copies host -> HBM; download copies back in the ORIGINAL order
 * (the device may keep particles permuted). */
int32_t pb_particles_upload(pb_engine* e, int64_t n, const float* x, const float* y, const float* z,
                            const float* dx, const float* dy, const float* dz, const double* t,
                            const int32_t* state, const int32_t* ei, const int64_t* particle_id);
int32_t pb_particles_download(pb_engine* e, int64_t n, float* x, float* y, float* z, float* dx, float* dy,
                              float* dz, double* t, int32_t* state, int32_t* ei);
/* Device-resident bench support: snapshot / restore the particle SoA inside HBM. */
int32_t pb_particles_snapshot(pb_engine* e);
int32_t pb_particles_restore(pb_engine* e);
int64_t pb_particles_count(pb_engine* e);

/* ---- output path: replaces ParticleFile.write's row selection + column copies (_core/particlefile.py:142-221)
 * and Kernel.remove_deleted (_core/kernel.py:98-106) for a particle set that stays resident in HBM ----------
 * pb_output_select evaluates `_to_write_particles` (:198-221) on the device for the resident particles:
 *   finite t  and  t_out - |dt/2| <= t <= t_out + |dt/2|          (dt: the nominal step Kernel.execute leaves
 * in particles.dt, kernel.py:225-226), in storage order, and returns the number of rows.  pb_output_gather
 * copies ONLY those rows of the written columns (Variable.to_write, _core/particle.py:123-175: x, y, z, t,
 * particle_id; NULL = skip the column) and, optionally, their storage indices (np.where(...)[0]) to the host.
 * pb_particles_remove_deleted drops particles in state Delete keeping the storage order, as
 * ParticleSet.remove_indices -> np.delete does (_core/particleset.py:247-250). */
int32_t pb_output_select(pb_engine* e, double t_out, double dt, int64_t* n_selected);
int32_t pb_output_gather(pb_engine* e, int64_t n_selected, int64_t* index, float* x, float* y, float* z, double* t,
                         int64_t* particle_id);
int32_t pb_particles_remove_deleted(pb_engine* e, int64_t* n_left);

/* ---- the hot path: replaces Kernel.execute(pset, endtime, dt) (_core/kernel.py:174-247) -- */
#define PB_BATCH_FIRST_EVAL_TWO_T 1
#define PB_BATCH_TWO_Z 2
typedef struct pb_advect_args {
    int32_t scheme;            /* enum pb_scheme                                                */
    int32_t diffusion;         /* 1: DiffusionUniformKh fused after the advection kernel
                                  (kernels/_advectiondiffusion.py:120-153)                      */
    int32_t delete_on_error;   /* 1: a trailing error handler turns every state >= 50 into
                                  Delete (reference idiom tests/common_kernels.py:12-13)        */
    int32_t kh_spherical;      /* mesh of the constant Kh fields                                */
    double dt;                 /* signed time step, seconds                                     */
    double endtime;            /* seconds since the start of the time interval                  */
    double kh_zonal;           /* constant-field values (m^2/s)                                 */
    double kh_meridional;
    double kh_deg2m;
    uint64_t seed;             /* Philox4x32-10 key for the Wiener increments                   */
    uint64_t rng_call;         /* counter word: index of this Kernel.execute call               */
    int64_t max_iters;         /* <0: run to endtime; >=0: at most this many loop iterations
                                  (used to replay up to the first error, see INTEGRATION.md)    */
    int32_t hint_all_zero;     /* curvilinear grids: 1 when the hinted xi (unravel of ei) of every
                                  evaluated particle is 0 -- the reference then skips the hint test for
                                  the whole batch at the first eval (_core/index_search.py:269-282)   */
    int32_t resume;            /* 1: continue the same Kernel.execute call after a migration round
                                  (mode D): particle states are NOT reset to Evaluate            */
    int32_t kernels_only;      /* 1: run the kernel functions of ONE loop iteration on the evaluated particles
                                  and return (dx/dy/dz accumulated, state/ei updated) WITHOUT the position
                                  update, EndofLoop and delete bookkeeping -- the host finishes the iteration
                                  (used when the kernel list also holds user Python kernels)              */
    int32_t batch_levels;      /* what the reference decides per BATCH of an evaluation and a lane cannot know by itself
                                  (`lenT = 2 if any(tau > 0)`, `lenZ = 2 if any(zeta > 0)`, _xinterpolators.py:130-131,400-401):
                                  PB_BATCH_FIRST_EVAL_TWO_T (1): some evaluated particle of the call's FIRST loop iteration is not
                                    exactly on the first time level -- two time levels for the whole batch of that evaluation,
                                    which promotes the value of a particle AT the first level to float64 (matters on float32
                                    grids; tau == 0 exists only at the first level, so later evaluations cannot mix);
                                  PB_BATCH_TWO_Z (2): some evaluated particle lies below the first depth level -- XFreeslip /
                                    XPartialslip then test the second depth level for land for EVERY particle, also one that
                                    sits exactly on the first level (taken as constant over the call) */
} pb_advect_args;

typedef struct pb_report {
    int64_t particle_steps;    /* particle-steps evaluated (one step = all RK stages)           */
    int64_t n_error;           /* particles that ended in a state >= 50                          */
    int64_t n_deleted;         /* particles that ended in state Delete (30)                     */
    int64_t first_error_iter;  /* smallest loop iteration at which an error state arose (with delete_on_error: at which a
                                * particle sampled outside the time interval), or -1 */
    int64_t n_out_of_time;     /* particles that sampled outside the time interval (state 70)    */
    int64_t max_iters_done;    /* largest per-particle iteration count                          */
    int64_t cache_refills;     /* corner-cache refills (diagnostic: HBM gathers actually made)   */
    int64_t n_migrate;         /* mode D: particles that left the owned slab and wait for migration */
    int64_t n_wait_window;     /* time-slab streaming: particles whose next step needs a non-resident level */
    double wait_t_min;         /* smallest / largest time of those particles (valid when n_wait_window > 0) */
    double wait_t_max;
    int32_t max_state;
    int32_t kernel_variant;    /* 0: generic kernel family; 1: specialised RK4 kernel (float64 grid, float32 interleaved data) */
    float kernel_ms;           /* CUDA-event time of the advection kernel on the engine stream   */
    float reserved2;
} pb_report;

/* Runs the inner loop of Kernel.execute for every particle until `endtime` (or an error /
 * deletion / max_iters).  Synchronous: returns after the kernel has finished and `rep` is
 * filled.  Particle arrays stay in HBM; call pb_particles_download to read them back. */
int32_t pb_advect(pb_engine* e, const pb_advect_args* args, pb_report* rep);
/* Asynchronous variant: enqueues on the engine stream and returns; the report is available
 * after pb_engine_synchronize() through pb_last_report(). */
int32_t pb_advect_async(pb_engine* e, const pb_advect_args* args);
int32_t pb_last_report(pb_engine* e, pb_report* rep);

/* Kernel.execute on HOST particle arrays in one call (the shape of the reference's own call: pset._data in, pset._data out,
 * _core/kernel.py:174-247), software-pipelined: the set is cut into `n_chunks` chunks (whole thread blocks; at most one per
 * 37888 particles), each chunk is copied in, snapshotted (pb_particles_snapshot's layout, so pb_particles_restore rewinds the
 * whole set), advected and -- when `download` != 0 -- copied back in one in-order stream, with up to four chunk streams in flight:
 * the copies of one chunk run under the kernels of the others.  Equivalent to pb_particles_upload + pb_particles_snapshot +
 * pb_advect (+ pb_particles_download): identical particle results and report; pb_report.kernel_ms is the device time of the whole
 * pipelined pass, copies included.  The arrays play both roles (input, and output when `download`); dx / dy / dz may be NULL
 * (zeros, not copied back); particle_id may be NULL without diffusion.  Page-locked host arrays make the copies fully
 * asynchronous; pageable arrays work, with less overlap.  Not for time-windowed fieldsets. */
typedef struct pb_particle_arrays {
    float *x, *y, *z, *dx, *dy, *dz;
    double* t;
    int32_t* state;
    int32_t* ei;
    const int64_t* particle_id;
} pb_particle_arrays;
int32_t pb_advect_host(pb_engine* e, const pb_advect_args* args, int64_t n, const pb_particle_arrays* arrays, int32_t download,
                       int32_t n_chunks, pb_report* rep);

/* ---- AdvectionRK45 (kernels/_advection.py:85-155) under Kernel.execute's Repeat / next_dt state machine
 * (_core/kernel.py:108-120,199-216,224-226): every particle carries its own dt and next_dt; a rejected step
 * (error estimate kappa > tol) sets state Repeat and is retried with dt / 2 inside the same loop iteration; an
 * accepted one may double next_dt; after the position update dt <- next_dt; dt is never reset to the nominal step.
 * tol is in the units of the mesh (the reference divides fieldset.RK45_tol by deg2m on spherical meshes when the
 * Kernel is built, kernel.py:144-145 -- the caller does the same).  dt_inout / next_dt_inout: host arrays of
 * pb_particles_count() float64 (next_dt widened; next_dt_is_f32 = the Particle's next_dt Variable is float32, the
 * default dtype, so assignments to it round to float32).  On return dt_inout holds particles.dt exactly as the
 * reference leaves it, including its batch-level clamp of the particles that left the loop early (kernel.py:199-203).
 * pb_report: particle_steps = accepted steps, cache_refills = field evaluations (6 per attempt), n_error = particles
 * whose dt is 0 before endtime (state 50; the reference's loop never terminates on those).
 * XLinear_Velocity / XFreeslip / XPartialslip on rectilinear A-grids, CGrid_Velocity on rectilinear and curvilinear C-grids,
 * resident or time-windowed (pb_field_window_create): a particle whose next iteration's span [t, t + dt] is not resident stops
 * with its state, dt and next_dt unchanged (pb_report.n_wait_window); after pb_field_window_set, call again with resume = 1:
 * the engine keeps every particle's iteration count between the launches, and clamps the dt of the particles that left the
 * loop early (above) only after the launch that leaves nobody waiting. */
typedef struct pb_rk45_args {
    double dt;      /* nominal dt of ParticleSet.execute: only its sign is used (compute_time_direction) */
    double endtime;
    double tol, min_dt, max_dt; /* fieldset.RK45_tol (mesh units), RK45_min_dt, RK45_max_dt */
    int64_t max_iters;          /* < 0: run to endtime */
    int32_t next_dt_is_f32;
    int32_t delete_on_error;
    int32_t kernels_only;       /* 1: ONE loop iteration's kernel work only -- the RK45 attempts of every evaluated particle until
                                   its step is accepted (kernel.py:206-216), dx / dy, dt, next_dt, state, ei written back, no position
                                   update, no batch-level dt clamp of finished particles (mixed lists: the host finishes the iteration) */
    int32_t resume;             /* 1: particle states are NOT reset to Evaluate */
    int32_t hint_all_zero;      /* curvilinear grids, like the pb_advect_args field: the first evaluation of the call skips the hint test */
    int32_t batch_levels;       /* like the pb_advect_args field; the time bit applies to the first attempt of the first iteration */
} pb_rk45_args;
int32_t pb_advect_rk45(pb_engine* e, const pb_rk45_args* args, double* dt_inout, double* next_dt_inout, pb_report* rep);
/* The same loop on the RESIDENT dt / next_dt / iteration columns of pb_particles_upload_resume (read them back with
 * pb_particles_download_resume): the route of a domain-decomposed engine (mode D, below), where these travel with the particles,
 * and the one RK45 entry point that runs there (rectilinear grids: XLinear_Velocity, XFreeslip, XPartialslip, CGrid_Velocity).
 * kernels_only must be 0.  A particle that
 * leaves the owned slab stops mid-call with its dt, next_dt and iteration count, and the launch with resume = 1 on its new owner
 * continues it.  Without waiting (pb_last_report collects the report); no batch-level clamp of the particles that left the loop
 * early: pb_rk45_finalize_resident does it once the whole call is done, with the call's iteration count over all launches and
 * ranks (the maximum of every pb_report.max_iters_done). */
int32_t pb_advect_rk45_resident_async(pb_engine* e, const pb_rk45_args* args);
int32_t pb_rk45_finalize_resident(pb_engine* e, double dt, double endtime, int64_t total_iters);

/* ---- AdvectionDiffusionM1 / AdvectionDiffusionEM (kernels/_advectiondiffusion.py:21-117) under Kernel.execute's loop:
 * 2-D advection with fieldset.UV plus diffusion with the spatially varying diffusivity fields Kh_zonal / Kh_meridional
 * -- scalar fields on the same rectilinear grid (XLinear), uploaded into slots >= 3 with pb_field_upload -- and their
 * central-difference gradients over fieldset.dres.  Seven field evaluations per particle and step, each raising the
 * particle's state and `ei` like Field.eval (_core/field.py:144-191); unit conversion of the diffusivities on spherical
 * meshes as meters_to_degrees_zonal / _meridional (:11-18: float32 cos of the float32 latitude).  dres is the Python float
 * the reference adds to the float32 positions (weak scalar: positions stay float32); deg2m_sq = pow(grid.deg2m, 2).
 * The Wiener increments come from the engine's Philox4x32-10 stream keyed like pb_advect's DiffusionUniformKh (the
 * reference draws from NumPy's global MT19937: statistical parity, bit parity of the deterministic part).
 * Same loop semantics, max_iters replay contract and pb_report as pb_advect.  Rectilinear grids, resident or time-windowed
 * U, V: a particle whose time t is not inside the resident levels stops (pb_report.n_wait_window); after
 * pb_field_window_set, call again with resume = 1 -- the engine keeps every particle's iteration count between the
 * launches, so the Wiener increments, first_error_iter and max_iters are those of one resident launch.
 * pb_advect_diffusion_async: the same launch without waiting (pb_last_report collects the report, like pb_advect_async). */
enum pb_advdiff_scheme { PB_ADVDIFF_M1 = 0, PB_ADVDIFF_EM = 1 };
typedef struct pb_advdiff_args {
    int32_t scheme;             /* enum pb_advdiff_scheme */
    int32_t delete_on_error;
    int32_t kh_zonal_slot;      /* field slots (>= 3) of Kh_zonal / Kh_meridional: same dtype, both with or both without time */
    int32_t kh_meridional_slot;
    double dt;
    double endtime;
    double dres;                /* fieldset.dres */
    double deg2m_sq;            /* pow(Kh_meridional.grid.deg2m, 2); unused on flat meshes */
    uint64_t seed;
    uint64_t rng_call;
    int64_t max_iters;          /* < 0: run to endtime */
    int32_t kernels_only;       /* 1: the kernel function of ONE loop iteration only (mixed lists, as in pb_advect_args) */
    int32_t resume;             /* 1: particle states are NOT reset to Evaluate (the host drives the loop) */
    int32_t batch_levels;       /* like the pb_advect_args field; the time bit applies to every sample of the first iteration */
    int32_t reserved;
} pb_advdiff_args;
int32_t pb_advect_diffusion(pb_engine* e, const pb_advdiff_args* args, pb_report* rep);
int32_t pb_advect_diffusion_async(pb_engine* e, const pb_advdiff_args* args);

/* VectorField.eval at n arbitrary sample points (fieldset.UV[t, z, y, x] / fieldset.UVW[...],
 * _core/field.py:250-304): time + grid search, interpolation, unit conversion, error states
 * (state_out starts at Evaluate and is raised like particles.state), ei_out = ravel_index of the cell.
 * positions_are_f32 = 1 evaluates with float32 positions (a particle's own arrays), 0 with float64
 * (an RK stage position) -- the reference's arithmetic promotes on that dtype.  ei_hint (may be NULL)
 * seeds the curvilinear search like particles.ei does; no_hint = 1 skips the hint test.  Time-windowed U, V, W: every
 * finite sample time inside the time axis must lie within the resident levels, else PB_ERR_INVALID. */
int32_t pb_sample_velocity(pb_engine* e, int64_t n, const double* t, const double* z, const double* y, const double* x,
                           int32_t positions_are_f32, int32_t three_d, const int32_t* ei_hint, int32_t no_hint,
                           double* u, double* v, double* w, int32_t* ei_out, int32_t* state_out);

/* ---- scalar sampling: replaces Field.eval / fieldset.P[particles] (_core/field.py:144-202) for fields on the
 * rectilinear grid.  Scalar fields live in slots 3 .. PB_MAX_FIELDS-1 of pb_field_upload (0..2 are U, V, W);
 * a field with one time level has no time dimension (no time search, field.py:112-117).  method: the field's
 * ScalarInterpolator -- XLinear (_xinterpolators.py:112-153), XNearest (:515-560) or CGrid_Tracer (:335-383, uses
 * the staggering offsets of pb_set_interpolation).  Index search, `ei` write-back and state codes are those of
 * pb_sample_velocity; out-of-bounds samples are 0.  On curvilinear grids: CGrid_Tracer and XNearest (the cell comes from the
 * curvilinear search, ei_hint = NULL sends the whole batch through the spatial hash like the reference's `if np.any(xi)`).  value_is_f32 (optional): 1 where NumPy's promotion makes the
 * reference's value float32 (the value returned is that float32 number, widened). */
enum pb_scalar_interp {
    PB_SCALAR_XLINEAR = 0, PB_SCALAR_XNEAREST = 1, PB_SCALAR_CGRID_TRACER = 2,
    PB_SCALAR_XLINEAR_INVDIST_LAND = 3 /* XLinearInvdistLandTracer (:556-613): land corners (~0) left out */
};
int32_t pb_sample_scalar(pb_engine* e, int32_t slot, int32_t method, int64_t n, const double* t, const double* z,
                         const double* y, const double* x, int32_t positions_are_f32, const int32_t* ei_hint,
                         double* value, int32_t* value_is_f32, int32_t* ei_out, int32_t* state_out);

/* ---- multi-GPU mode D: X-slab domain decomposition with particle migration (SURVEY.md 8e) ------------
 * The reference has no distributed layer; this is new.  Each rank's engine holds the columns
 * lon[xi_offset : xi_offset + nx_local] of the global rectilinear grid (its owned columns + a halo) and the
 * matching field slab; pass the GLOBAL xdim_cells to pb_grid_upload_rectilinear so that `ei` stays global.
 * bounds[nranks+1]: rank r advances particles with bounds[r] <= x < bounds[r+1] (rank 0 also everything left
 * of bounds[1], the last rank everything right of bounds[nranks-1]); pb_advect stops a particle as soon as
 * it leaves the owned interval (pb_report.n_migrate).  A stage position outside owned+halo columns is a
 * halo violation: state 99, counted in n_error (the DeleteParticle handler leaves it alone, so pb_report.max_state shows it).
 * Migration round: pb_migrate_count -> (exchange counts) -> pb_migrate_pack -> all-to-all-v of the 48-byte
 * records over NCCL -> pb_migrate_unpack (compacts the stayers, appends the arrivals) -> pb_advect(resume=1). */
int32_t pb_decomp_set(pb_engine* e, int32_t nranks, int32_t rank, const double* bounds, int64_t xi_offset,
                      int32_t left_is_global, int32_t right_is_global);
int32_t pb_migrate_count(pb_engine* e, int64_t* counts /* [nranks] records to send to each rank */);
int32_t pb_migrate_pack(pb_engine* e, void* sendbuf_dev, int64_t capacity_records);
int32_t pb_migrate_unpack(pb_engine* e, const void* recvbuf_dev, int64_t n_in);
/* Mode D on a CURVILINEAR grid: column slabs.  The engine keeps the whole horizontal grid uploaded with
 * pb_grid_upload_curvilinear (lon / lat, the spherical cell projections, the spatial hash -- built exactly as on one GPU) and the
 * node columns [xi_offset, xi_offset + X) of U, V, W (pb_field_upload with X < nx: owned cells + halo).  Every search therefore
 * finds the single-GPU cell (yi, i) with a GLOBAL column i; rank r owns the cells with col_edges[r] <= i < col_edges[r+1]
 * (col_edges[0] = 0, col_edges[nranks] = nx - 1).  At the top of every iteration a lane runs the search of its first evaluation
 * (same hint, same rule) and that evaluation reuses it; a lane whose cell is another rank's stops with its ei untouched
 * (pb_report.n_migrate), one whose search finds no cell stays and raises the single-GPU error.  A stage position whose cell
 * needs a node column outside the slab is a halo violation (state 99).  The in-kernel delivery routes by the found column;
 * the collective transport classifies with pb_migrate_classify_columns instead of pb_migrate_count: the same search, no_hint =
 * the hint rule of the next launch's first iteration (with resumable state resident: of the lanes whose iteration count is 0).
 * pb_advect (fixed-step schemes, CGrid_Velocity or XLinear_Velocity) and pb_advect_rk45_resident_async (CGrid_Velocity) run on
 * such an engine; pb_sample_velocity and pb_sample_scalar refuse it (PB_ERR_STATE: the sampling kernels index the fields by
 * global column).  Grids whose faces overlap (duplicated wrap columns, a north fold) are not supported. */
int32_t pb_decomp_set_columns(pb_engine* e, int32_t nranks, int32_t rank, const int64_t* col_edges, int64_t xi_offset,
                              int32_t left_is_global, int32_t right_is_global);
int32_t pb_migrate_classify_columns(pb_engine* e, int32_t no_hint, int64_t* counts /* [nranks] */);
/* Device bytes the engine holds for its grid (coordinates, time axis, cell tables, cell projections, spatial hash) and for its
 * fields (every field slot, the node-interleaved copy). */
int32_t pb_memory_bytes(pb_engine* e, int64_t* grid_bytes, int64_t* field_bytes);
/* AdvectionRK45 (pb_advect_rk45_resident_async) and AdvectionDiffusionM1 / EM (pb_advect_diffusion) under mode D: a lane stopped
 * mid-call continues on its new owner with its dt, next_dt and iteration count (M1 / EM: the count keys the Wiener increments,
 * so the decomposed run draws the single-GPU run's increments).  pb_particles_upload_resume makes them resident columns (after
 * pb_particles_upload, which drops them; NULL arrays upload zeros), and from then on every move of the set carries them:
 * compaction, snapshot / restore, the in-kernel delivery (a 24-byte record per particle at the index of its 48-byte record, in
 * the inbox after the record slots) and the collective exchange -- pb_migrate_pack_resume / pb_migrate_unpack_resume fill and
 * read a second buffer of PB_MIGRATION_RESUME_BYTES per record, exchanged with the same counts as the records (the plain
 * pack / unpack refuse an engine with resident resumable state). */
#define PB_MIGRATION_RESUME_BYTES 24
int32_t pb_particles_upload_resume(pb_engine* e, int64_t n, const double* dt, const double* next_dt, const int32_t* iters);
int32_t pb_particles_download_resume(pb_engine* e, int64_t n, double* dt, double* next_dt, int32_t* iters);
int32_t pb_migrate_pack_resume(pb_engine* e, void* sendbuf_dev, void* resume_sendbuf_dev, int64_t capacity_records);
int32_t pb_migrate_unpack_resume(pb_engine* e, const void* recvbuf_dev, const void* resume_recvbuf_dev, int64_t n_in);

/* In-kernel migration over peer memory (one box: NVLink / NVSwitch).  No reference counterpart.  Every rank owns an INBOX
 * (two slots of `capacity_records` 48-byte records + an arrival counter each) in its own HBM; its peers map it through CUDA IPC.
 * Once connected, pb_advect itself delivers a particle that left the owned slab: the lane claims a slot in the new owner's inbox
 * with one system-scope atomic and stores the record there (pb_report.n_migrate = records delivered + records that found the
 * inbox full and wait on this rank for the next round).  There is no pack pass and no all-to-all.
 * Set-up:  pb_migrate_p2p_init (allocates the inbox; returns its 64-byte IPC handle and, for peers living in the SAME process,
 *          its address) -> the caller exchanges handles / addresses (e.g. torch.distributed.all_gather_object) ->
 *          pb_migrate_p2p_connect(handles[nranks * 64] or NULL, local_bases[nranks] or NULL; a non-zero local base wins).
 * Round:   pb_advect(resume = round > 0) on every rank -> a BARRIER that orders every rank's kernel before the next call
 *          (e.g. the all-reduce of n_migrate that also decides termination) -> pb_migrate_p2p_finish: drops the delivered
 *          records from the resident set (order-preserving), appends the arrivals, flips to the other inbox slot.  Every rank
 *          calls it in every round.  Repeat until the all-reduced n_migrate is 0. */
#define PB_IPC_HANDLE_BYTES 64
int32_t pb_migrate_p2p_init(pb_engine* e, int64_t capacity_records, uint8_t* ipc_handle /* [64] or NULL */, uint64_t* local_base /* or NULL */);
int32_t pb_migrate_p2p_connect(pb_engine* e, const uint8_t* ipc_handles, const uint64_t* local_bases);
int32_t pb_migrate_p2p_finish(pb_engine* e, int64_t* n_arrived, int64_t* n_resident);
/* back to the collective transport (a peer could not be mapped): pb_advect stops delivering by itself; the inbox stays allocated */
int32_t pb_migrate_p2p_disable(pb_engine* e);
#define PB_MIGRATION_RECORD_BYTES 48
/* particle ids in device order (after migrations the order on a rank is arbitrary) */
int32_t pb_particles_download_ids(pb_engine* e, int64_t n, int64_t* particle_id);

/* Marks every particle currently in state Evaluate/Success whose time-to-endtime >= 0 with
 * ErrorOutsideTimeInterval (70): the reference flags the WHOLE evaluated view when any particle
 * samples outside the time interval (_core/index_search.py:85-86, _core/field.py:31-44). */
int32_t pb_flag_view_outside_time(pb_engine* e, double dt, double endtime);
/* The same view under the DeleteParticle handler (state >= 50 -> Delete, reference tests' DeleteParticle kernel): every
 * particle of the view ends in state Delete (30).  pb_report.first_error_iter of a delete_on_error launch that saw
 * n_out_of_time > 0 is the iteration to replay to. */
int32_t pb_delete_view_outside_time(pb_engine* e, double dt, double endtime);

/* Pure helper used by tests: the engine's Philox4x32-10 + Box-Muller normals for
 * (seed, rng_call, iteration, particle_id), computed ON THE DEVICE. out = 2 doubles per id. */
int32_t pb_debug_normals(pb_engine* e, uint64_t seed, uint64_t rng_call, int64_t iter, int64_t n,
                         const int64_t* particle_id, double* out);

/* Pure helper used by tests: the hand-written math primitives of the kernels (the same inline functions, not copies),
 * evaluated ON THE DEVICE element by element.  out = 2 doubles per element:
 *   PB_MATH_COS_NP                cos_np(a[i]), 0                  (common.cuh: cos of a latitude in radians)
 *   PB_MATH_SIN_LAT               sin_lat(a[i]), 0                 (cgrid.cuh: sin of a latitude in radians)
 *   PB_MATH_SINCOS_LON            sin, cos of sincos_lon(a[i])     (cgrid.cuh: of a longitude in radians)
 *   PB_MATH_DIV_BY_CACHED         div_by_cached(a[i], b[i], r), r  (common.cuh; r = 1.0 / b[i] computed on the device)
 *   PB_MATH_DIV_BY_CACHED_GUARDED div_by_cached_guarded(a[i], b[i], r), r
 *   PB_MATH_BOX_MULLER_F32        zx, zy of box_muller_f32((uint32_t)a[i], (uint32_t)b[i])  (the two Philox words)
 *   PB_MATH_COSF                  cosf_ool((float)a[i]), 0         (cgrid.cuh: CUDA's float32 cosf; the float32 result widened)
 *   PB_MATH_SINF                  sinf_ool((float)a[i]), 0         (cgrid.cuh: CUDA's float32 sinf)
 *   PB_MATH_COS                   cos_ool(a[i]), 0                 (cgrid.cuh: CUDA's float64 cos -- the per-cell table, sinx)
 *   PB_MATH_SIN                   sin_ool(a[i]), 0                 (cgrid.cuh: CUDA's float64 sin)
 * b may be NULL for every op but the three binary ones (DIV_BY_CACHED, DIV_BY_CACHED_GUARDED, BOX_MULLER_F32). */
enum pb_math_op {
    PB_MATH_COS_NP = 0, PB_MATH_SIN_LAT = 1, PB_MATH_SINCOS_LON = 2, PB_MATH_DIV_BY_CACHED = 3, PB_MATH_DIV_BY_CACHED_GUARDED = 4,
    PB_MATH_BOX_MULLER_F32 = 5, PB_MATH_COSF = 6, PB_MATH_SINF = 7, PB_MATH_COS = 8, PB_MATH_SIN = 9
};
int32_t pb_debug_math(pb_engine* e, int32_t op, int64_t n, const double* a, const double* b, double* out);
/* The device cell table of axis `axis` (0 lon, 1 lat, 2 depth, 3 time) of a float64 rectilinear grid: `cells` records of 4 doubles
 * {lo, hi, 1 / (hi - lo), 0} into `out`; `cells` must be the axis' node count - 1.  PB_ERR_INVALID when there is no such table. */
int32_t pb_debug_axis_cells(pb_engine* e, int32_t axis, int64_t cells, double* out);
/* Threads per block the particle kernels of a family are launched with (as the library was built): the lane / warp / block a
 * particle runs in is its storage position's, i.e. position % block and position / block.  PB_ERR_INVALID for an unknown family. */
enum pb_launch_family {
    PB_BLOCK_AGRID_FAST = 0, /* the specialised RK4 kernel (afast.cu) */
    PB_BLOCK_AGRID = 1,      /* the generic A-grid kernels (agrid.cu) */
    PB_BLOCK_CGRID = 2,      /* rectilinear and curvilinear C-grids (cgrid.cu) */
    PB_BLOCK_CURV_AGRID = 3, /* XLinear_Velocity on curvilinear grids (curva.cu) */
    PB_BLOCK_SAMPLE_FLAGS = 4 /* the batch-level lenT / lenZ pre-pass of pb_sample_velocity / pb_sample_scalar */
};
int32_t pb_debug_launch_block(int32_t family);

/* ---- host-side passes of Kernel.execute / ParticleSet.execute over the particle columns, multi-threaded ----------------
 * The reference makes a few whole-column passes per call on the host: `pset._data["dt"][:] = dt` (_core/particleset.py:405,
 * _core/kernel.py:225-226), `particle_release_times.min() / .max()` (_core/particleset.py:541-544), `state[:] = Evaluate`
 * (_core/kernel.py:188).  At 1e7 particles a single NumPy thread spends longer on them than the device on the copies; these
 * helpers split the column over a few host threads (memory-bandwidth bound).  No engine, no device. */
int32_t pb_host_fill_f64(double* p, int64_t n, double value);
int32_t pb_host_fill_i32(int32_t* p, int64_t n, int32_t value);
int32_t pb_host_copy_strided_i32(int32_t* dst, int64_t dst_stride, const int32_t* src, int64_t src_stride, int64_t n); /* strides in elements */
/* min and max of p[0..n) ignoring NaNs; *has_nan = 1 when any element is NaN (NumPy's min / max then return NaN);
 * n == 0: *mn = +inf, *mx = -inf */
int32_t pb_host_min_max_f64(const double* p, int64_t n, double* mn, double* mx, int32_t* has_nan);
/* Kernel.remove_deleted -> ParticleSet.remove_indices (_core/kernel.py:98-106, _core/particleset.py:247-250: np.delete on every
 * column) for host arrays: rows with state == delete_state are dropped from `ncols` columns, order preserved, out of place
 * (src[c] -> dst[c], row_bytes[c] bytes per row, dst sized for pb_host_count_keep rows); the rows are split over host threads. */
int64_t pb_host_count_keep(const int32_t* state, int64_t n, int32_t delete_state);
int32_t pb_host_compact(const int32_t* state, int64_t n, int32_t delete_state, int32_t ncols, const void* const* src,
                        void* const* dst, const int64_t* row_bytes);

#ifdef __cplusplus
}
#endif
#endif /* PARCELS_B200_H */
