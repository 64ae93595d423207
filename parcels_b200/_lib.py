"""ctypes binding of ``libparcels_b200.so`` (C-ABI: ``include/parcels_b200.h``).

The shared library is built in-tree by ``parcels_b200.build`` (nvcc, sm_90a only).  If it is
missing or a symbol is absent, importing the engine fails loudly -- there is no fallback.
"""

from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PB_LIB", os.path.join(HERE, "lib", "libparcels_b200.so"))  # PB_LIB: tuning variants

c_f32p = C.POINTER(C.c_float)
c_f64p = C.POINTER(C.c_double)
c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)


class ParticleArrays(C.Structure):
    """pb_particle_arrays: the host columns of the particle SoA (pb_advect_host)."""

    _fields_ = [(k, C.c_void_p) for k in ("x", "y", "z", "dx", "dy", "dz", "t", "state", "ei", "particle_id")]


class AdvectArgs(C.Structure):
    _fields_ = [
        ("scheme", C.c_int32),
        ("diffusion", C.c_int32),
        ("delete_on_error", C.c_int32),
        ("kh_spherical", C.c_int32),
        ("dt", C.c_double),
        ("endtime", C.c_double),
        ("kh_zonal", C.c_double),
        ("kh_meridional", C.c_double),
        ("kh_deg2m", C.c_double),
        ("seed", C.c_uint64),
        ("rng_call", C.c_uint64),
        ("max_iters", C.c_int64),
        ("hint_all_zero", C.c_int32),
        ("resume", C.c_int32),
        ("kernels_only", C.c_int32),
        ("batch_levels", C.c_int32),
    ]


class Rk45Args(C.Structure):
    _fields_ = [
        ("dt", C.c_double),
        ("endtime", C.c_double),
        ("tol", C.c_double),
        ("min_dt", C.c_double),
        ("max_dt", C.c_double),
        ("max_iters", C.c_int64),
        ("next_dt_is_f32", C.c_int32),
        ("delete_on_error", C.c_int32),
        ("kernels_only", C.c_int32),
        ("resume", C.c_int32),
        ("hint_all_zero", C.c_int32),
        ("batch_levels", C.c_int32),
    ]


class AdvDiffArgs(C.Structure):
    _fields_ = [
        ("scheme", C.c_int32),
        ("delete_on_error", C.c_int32),
        ("kh_zonal_slot", C.c_int32),
        ("kh_meridional_slot", C.c_int32),
        ("dt", C.c_double),
        ("endtime", C.c_double),
        ("dres", C.c_double),
        ("deg2m_sq", C.c_double),
        ("seed", C.c_uint64),
        ("rng_call", C.c_uint64),
        ("max_iters", C.c_int64),
        ("kernels_only", C.c_int32),
        ("resume", C.c_int32),
        ("batch_levels", C.c_int32),
        ("kernel_variant", C.c_int32),
    ]


class Report(C.Structure):
    _fields_ = [
        ("particle_steps", C.c_int64),
        ("n_error", C.c_int64),
        ("n_deleted", C.c_int64),
        ("first_error_iter", C.c_int64),
        ("n_out_of_time", C.c_int64),
        ("max_iters_done", C.c_int64),
        ("cache_refills", C.c_int64),
        ("n_migrate", C.c_int64),
        ("n_wait_window", C.c_int64),
        ("wait_t_min", C.c_double),
        ("wait_t_max", C.c_double),
        ("max_state", C.c_int32),
        ("kernel_variant", C.c_int32),
        ("kernel_ms", C.c_float),
        ("reserved2", C.c_float),
    ]


# every symbol include/parcels_b200.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "pb_abi_version": (C.c_int32, []),
    "pb_last_error_string": (C.c_char_p, []),
    "pb_device_count": (C.c_int32, []),
    "pb_engine_create": (C.c_int32, [C.c_int32, C.POINTER(_P)]),
    "pb_engine_destroy": (None, [_P]),
    "pb_engine_synchronize": (C.c_int32, [_P]),
    "pb_timer_begin": (C.c_int32, [_P]),
    "pb_timer_end_ms": (C.c_int32, [_P, C.POINTER(C.c_float)]),
    "pb_grid_upload_rectilinear": (
        C.c_int32,
        [_P, _P, C.c_int64, _P, C.c_int64, _P, C.c_int64, C.c_int32, _P, C.c_int64, C.c_int32, C.c_double,
         C.c_int64, C.c_int64, C.c_int64],
    ),  # fmt: skip
    "pb_grid_upload_curvilinear": (
        C.c_int32,
        [_P, _P, _P, C.c_int64, C.c_int64, _P, C.c_int64, C.c_int32, _P, C.c_int64, C.c_int32, C.c_double, C.c_int64,
         C.c_int64, C.c_int64, _P, _P, _P, C.c_int64, _P, C.c_int64, _P, C.c_int32, _P],
    ),  # fmt: skip
    "pb_hash_table_size": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pb_hash_table_download": (C.c_int32, [_P, _P, _P, _P, _P]),
    "pb_set_interpolation": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "pb_field_upload": (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64]),
    "pb_field_attach_device": (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64]),
    "pb_field_clear": (C.c_int32, [_P, C.c_int32]),
    "pb_field_window_create": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int32]),
    "pb_field_window_load": (C.c_int32, [_P, C.c_int32, C.c_int64, _P]),
    "pb_field_window_set": (C.c_int32, [_P, C.c_int64, C.c_int64]),
    "pb_particles_upload": (C.c_int32, [_P, C.c_int64] + [_P] * 10),
    "pb_particles_download": (C.c_int32, [_P, C.c_int64] + [_P] * 9),
    "pb_particles_snapshot": (C.c_int32, [_P]),
    "pb_particles_restore": (C.c_int32, [_P]),
    "pb_particles_count": (C.c_int64, [_P]),
    "pb_output_select": (C.c_int32, [_P, C.c_double, C.c_double, C.POINTER(C.c_int64)]),
    "pb_output_gather": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, _P]),
    "pb_particles_remove_deleted": (C.c_int32, [_P, C.POINTER(C.c_int64)]),
    "pb_advect": (C.c_int32, [_P, C.POINTER(AdvectArgs), C.POINTER(Report)]),
    "pb_advect_async": (C.c_int32, [_P, C.POINTER(AdvectArgs)]),
    "pb_advect_host": (C.c_int32, [_P, C.POINTER(AdvectArgs), C.c_int64, C.POINTER(ParticleArrays), C.c_int32, C.c_int32, C.POINTER(Report)]),
    "pb_advect_rk45": (C.c_int32, [_P, _P, _P, _P, _P]),
    "pb_advect_diffusion": (C.c_int32, [_P, C.POINTER(AdvDiffArgs), C.POINTER(Report)]),
    "pb_last_report": (C.c_int32, [_P, C.POINTER(Report)]),
    "pb_sample_velocity": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P, _P]),
    "pb_sample_scalar": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P, _P, C.c_int32, _P, _P, _P, _P, _P]),
    "pb_decomp_set": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int32, C.c_int32]),
    "pb_migrate_count": (C.c_int32, [_P, _P]),
    "pb_migrate_pack": (C.c_int32, [_P, _P, C.c_int64]),
    "pb_migrate_unpack": (C.c_int32, [_P, _P, C.c_int64]),
    "pb_migrate_p2p_init": (C.c_int32, [_P, C.c_int64, _P, _P]),
    "pb_migrate_p2p_connect": (C.c_int32, [_P, _P, _P]),
    "pb_migrate_p2p_finish": (C.c_int32, [_P, _P, _P]),
    "pb_migrate_p2p_disable": (C.c_int32, [_P]),
    "pb_particles_download_ids": (C.c_int32, [_P, C.c_int64, _P]),
    "pb_flag_view_outside_time": (C.c_int32, [_P, C.c_double, C.c_double]),
    "pb_delete_view_outside_time": (C.c_int32, [_P, C.c_double, C.c_double]),
    "pb_debug_normals": (C.c_int32, [_P, C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, _P, _P]),
    "pb_debug_math": (C.c_int32, [_P, C.c_int32, C.c_int64, _P, _P, _P]),
    "pb_host_fill_f64": (C.c_int32, [_P, C.c_int64, C.c_double]),
    "pb_host_fill_i32": (C.c_int32, [_P, C.c_int64, C.c_int32]),
    "pb_host_min_max_f64": (C.c_int32, [_P, C.c_int64, _P, _P, _P]),
    "pb_host_copy_strided_i32": (C.c_int32, [_P, C.c_int64, _P, C.c_int64, C.c_int64]),
    "pb_host_count_keep": (C.c_int64, [_P, C.c_int64, C.c_int32]),
    "pb_host_compact": (C.c_int32, [_P, C.c_int64, C.c_int32, C.c_int32, _P, _P, _P]),
}

_lib = None


class EngineError(RuntimeError):
    pass


def load():
    """Load the shared library and bind every declared symbol (raises if anything is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). parcels_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    if lib.pb_abi_version() != 1:
        raise EngineError(f"ABI version mismatch: library {lib.pb_abi_version()} != binding 1")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().pb_last_error_string()
        raise EngineError(f"libparcels_b200 error {rc}: {msg.decode() if msg else ''}")


def ptr(a):
    """Raw data pointer of a C-contiguous ndarray (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return a.ctypes.data_as(C.c_void_p)
