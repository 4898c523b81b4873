"""ctypes binding of libdmv_b200.so (include/dmv_b200.h).  There is no CPU fallback: if the library
is missing it is built with nvcc, and any call that needs a device fails loudly without one."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

_lib = None


class DmvError(RuntimeError):
    pass


class BasisDesc(C.Structure):
    _fields_ = [
        ("number_sites", C.c_int32), ("hamming_weight", C.c_int32), ("spin_inversion", C.c_int32),
        ("has_permutations", C.c_int32), ("group_order", C.c_int64),
        ("perms", C.c_void_p), ("flips", C.c_void_p), ("characters", C.c_void_p),
    ]


class ExternalArray(C.Structure):   # chpl_external_array
    _fields_ = [("elts", C.c_void_p), ("num_elts", C.c_uint64), ("freer", C.CFUNCTYPE(None, C.c_void_p))]


class OperatorDesc(C.Structure):
    _fields_ = [
        ("n_off", C.c_int64), ("off_v", C.c_void_p), ("off_m", C.c_void_p), ("off_r", C.c_void_p),
        ("off_x", C.c_void_p), ("off_s", C.c_void_p),
        ("n_diag", C.c_int64), ("diag_v", C.c_void_p), ("diag_m", C.c_void_p), ("diag_r", C.c_void_p),
        ("diag_s", C.c_void_p),
    ]


DMV_F64, DMV_C128 = 1, 2

# every symbol include/dmv_b200.h declares: (name, restype, argtypes)
_SIGNATURES = [
    ("ls_chpl_init", None, []),
    ("ls_chpl_finalize", None, []),
    ("dmv_last_error", C.c_char_p, []),
    ("dmv_version", C.c_int, []),
    ("dmv_launch_count", C.c_int64, []),
    ("dmv_context_create", C.c_int, [C.POINTER(BasisDesc), C.POINTER(OperatorDesc), C.c_int, C.c_int, C.c_int,
                                     C.POINTER(C.c_void_p)]),
    ("dmv_context_destroy", C.c_int, [C.c_void_p]),
    ("dmv_set_stream", C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    ("dmv_synchronize", C.c_int, [C.c_void_p]),
    ("dmv_set_option", C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    ("dmv_get_info", C.c_int64, [C.c_void_p, C.c_char_p]),
    ("dmv_basis_build", C.c_int, [C.c_void_p]),
    ("dmv_set_representatives", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    ("dmv_number_states", C.c_int64, [C.c_void_p]),
    ("dmv_get_representatives", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_state_index", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    ("dmv_state_info", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_locale_idx_of", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]),
    ("dmv_max_number_off_diag", C.c_int64, [C.c_void_p]),
    ("dmv_compute_off_diag", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int,
                                       C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_local_matvec", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_matvec", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_plan", C.c_int, [C.c_void_p, C.c_void_p]),
    ("dmv_generate", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_outgoing", C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                               C.POINTER(C.c_int64)]),
    ("dmv_accumulate", C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_hashed_positions", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_permute", C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    ("dmv_block_to_hashed", C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    ("dmv_hashed_to_block", C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    ("dmv_replicated_setup", C.c_int, [C.c_void_p]),
    ("dmv_replicated_product", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_comm_unique_id", C.c_int, [C.c_void_p]),
    ("dmv_comm_init", C.c_int, [C.c_void_p, C.c_void_p]),
    ("dmv_matvec_batch", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_lanczos", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_uint64, C.POINTER(C.c_double), C.c_void_p,
                              C.POINTER(C.c_int), C.POINTER(C.c_double)]),
    ("dmv_expm_multiply", C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_double, C.POINTER(C.c_int), C.POINTER(C.c_double)]),
    ("dmv_eigsh", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_uint64,
                            C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                            C.POINTER(C.c_int)]),
    ("dmv_zz_correlations", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_pm_correlations", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_apply_spin", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                 C.c_void_p]),
    ("dmv_reduced_density_matrix", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                             C.c_void_p]),
    ("dmv_rdm_layout", C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                 C.c_void_p]),
    ("dmv_lanczos_quadrature", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    ("dmv_last_timings", C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_int]),
    ("dmv_timing_name", C.c_char_p, [C.c_int]),
    ("dmv_number_terms", C.c_int64, [C.c_void_p]),
    ("dmv_bind_operator", C.c_int, [C.c_void_p, C.c_void_p]),
    ("ls_chpl_matrix_vector_product", None, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("ls_chpl_primme_matvec", None, [C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int64),
                                     C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]),
    ("dmv_apply_diag", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    ("dmv_apply_off_diag", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("ls_chpl_operator_apply_diag", None, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(ExternalArray), C.c_int64]),
    ("ls_chpl_operator_apply_off_diag", None, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(ExternalArray),
                                               C.POINTER(ExternalArray), C.POINTER(ExternalArray), C.c_int64]),
    ("ls_chpl_enumerate_representatives", None, [C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(ExternalArray)]),
    ("dmv_debug_tridiagonal_lowest", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_void_p]),
    ("dmv_debug_tridiagonal_expm", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p]),
    ("dmv_debug_hermitian_eigen", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_debug_tridiagonal_quadrature", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_debug_zz_symmetrize", C.c_int, [C.POINTER(BasisDesc), C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dmv_debug_pm_classes", C.c_int, [C.POINTER(BasisDesc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_double, C.c_void_p, C.c_void_p]),
    ("dmv_debug_spin_weights", C.c_int, [C.POINTER(BasisDesc), C.POINTER(BasisDesc), C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    ("dmv_debug_compile_group", C.c_int, [C.POINTER(BasisDesc), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    ("dmv_debug_ordered_table", C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    ("dmv_debug_dense_order", C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    ("dmv_debug_torus_sq_rows", C.c_int, [C.POINTER(BasisDesc), C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    ("dmv_debug_rows_store", C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    ("dmv_debug_rows_store_plan", C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                            C.c_int, C.c_void_p, C.c_void_p]),
    ("dmv_debug_rows_store_coefficients", C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                                    C.POINTER(C.c_int)]),
    ("dmv_debug_solver_kernel", C.c_int, [C.c_char_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_double, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                          C.POINTER(C.c_int)]),
]

EXPORTED_SYMBOLS = [s[0] for s in _SIGNATURES]


def library_path() -> str:
    return _build.LIB


def lib():
    global _lib
    if _lib is None:
        path = _build.LIB
        if not os.path.exists(path):
            path = _build.build()   # raises if nvcc is missing: no fallback
        L = C.CDLL(path)
        for name, restype, argtypes in _SIGNATURES:
            fn = getattr(L, name)   # AttributeError if the library does not export the symbol
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise DmvError(lib().dmv_last_error().decode("utf-8", "replace"))
