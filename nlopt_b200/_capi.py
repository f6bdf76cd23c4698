"""ctypes binding of the NLopt C ABI (reference: src/api/nlopt.h:203-301).

The same binder works for any shared library that exports that ABI: the product
library ``libnlopt_b200.so`` (default) or -- in tests only -- the unmodified
reference compiled into ``oracle/_ref/libnlopt_ref.so``.  Nothing here computes
anything; it declares argument types and loads the library.
"""
from __future__ import annotations

import ctypes as C
import os

c_double_p = C.POINTER(C.c_double)

# callback shapes, reference nlopt.h:60-66
NLOPT_FUNC = C.CFUNCTYPE(C.c_double, C.c_uint, c_double_p, c_double_p, C.c_void_p)
NLOPT_MFUNC = C.CFUNCTYPE(None, C.c_uint, c_double_p, C.c_uint, c_double_p, c_double_p, C.c_void_p)
NLOPT_PRECOND = C.CFUNCTYPE(None, C.c_uint, c_double_p, c_double_p, c_double_p, C.c_void_p)
# extension: device callback (include/nlopt_b200.h)
NLOPT_B200_DFUNC = C.CFUNCTYPE(C.c_double, C.c_uint, C.c_ulonglong, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p)
# terms callbacks (nlopt_b200_dtfunc) and the host finishes of the asynchronous forms
NLOPT_B200_DTFUNC = C.CFUNCTYPE(None, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p,
                                C.c_void_p, C.c_void_p)
NLOPT_B200_DFINISH = C.CFUNCTYPE(C.c_double, C.c_double, C.c_void_p)
NLOPT_B200_DMFINISH = C.CFUNCTYPE(None, C.c_uint, c_double_p, c_double_p, C.c_void_p)


class Shard(C.Structure):
    """nlopt_b200_shard: this rank's part of the library's variable / group / virtual-shard geometry"""
    _fields_ = [("n", C.c_ulonglong), ("n_local", C.c_ulonglong), ("j0", C.c_ulonglong), ("nchunks", C.c_ulonglong),
                ("chunk0", C.c_ulonglong), ("groups_total", C.c_uint), ("group0", C.c_uint), ("groups_local", C.c_uint),
                ("groups_per_vshard", C.c_uint), ("vshard0", C.c_uint), ("local_vshards", C.c_uint), ("rank", C.c_int),
                ("world", C.c_int)]

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_DIR = os.path.dirname(PKG_DIR)
# NLOPT_B200_LIBDIR: load an alternative build of the same library (tools/trace_solve.py: instrumented build)
LIB_DIR = os.environ.get("NLOPT_B200_LIBDIR", PKG_DIR)
DEFAULT_LIB = os.path.join(LIB_DIR, "libnlopt_b200.so")


class Stats(C.Structure):
    _fields_ = [
        ("dual_evals", C.c_longlong), ("dual_solves", C.c_longlong), ("outer_iters", C.c_longlong),
        ("seconds_total", C.c_double), ("seconds_callbacks", C.c_double),
        ("seconds_dual_kernel", C.c_double),
        ("h2d_bytes", C.c_longlong), ("d2h_bytes", C.c_longlong), ("kernel_launches", C.c_longlong),
        ("seconds_setup", C.c_double), ("seconds_dual_wall", C.c_double), ("seconds_eval_wall", C.c_double),
        ("seconds_glue_wall", C.c_double), ("dual_operand_bytes", C.c_longlong),
        ("sigma_palette", C.c_longlong), ("sigma_index_mismatches", C.c_longlong),
    ]


# name -> (restype, argtypes); the standard object API
_STD = {
    "nlopt_algorithm_name": (C.c_char_p, [C.c_int]),
    "nlopt_algorithm_to_string": (C.c_char_p, [C.c_int]),
    "nlopt_algorithm_from_string": (C.c_int, [C.c_char_p]),
    "nlopt_result_to_string": (C.c_char_p, [C.c_int]),
    "nlopt_result_from_string": (C.c_int, [C.c_char_p]),
    "nlopt_version": (None, [C.POINTER(C.c_int)] * 3),
    "nlopt_srand": (None, [C.c_ulong]),
    "nlopt_srand_time": (None, []),
    "nlopt_create": (C.c_void_p, [C.c_int, C.c_uint]),
    "nlopt_destroy": (None, [C.c_void_p]),
    "nlopt_copy": (C.c_void_p, [C.c_void_p]),
    "nlopt_optimize": (C.c_int, [C.c_void_p, c_double_p, c_double_p]),
    "nlopt_set_min_objective": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p]),
    "nlopt_set_max_objective": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p]),
    "nlopt_set_precond_min_objective": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_void_p]),
    "nlopt_set_precond_max_objective": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_void_p]),
    "nlopt_get_algorithm": (C.c_int, [C.c_void_p]),
    "nlopt_get_dimension": (C.c_uint, [C.c_void_p]),
    "nlopt_get_errmsg": (C.c_char_p, [C.c_void_p]),
    "nlopt_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_double]),
    "nlopt_get_param": (C.c_double, [C.c_void_p, C.c_char_p, C.c_double]),
    "nlopt_has_param": (C.c_int, [C.c_void_p, C.c_char_p]),
    "nlopt_num_params": (C.c_uint, [C.c_void_p]),
    "nlopt_nth_param": (C.c_char_p, [C.c_void_p, C.c_uint]),
    "nlopt_set_lower_bounds": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_lower_bounds1": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_set_lower_bound": (C.c_int, [C.c_void_p, C.c_int, C.c_double]),
    "nlopt_get_lower_bounds": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_upper_bounds": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_upper_bounds1": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_set_upper_bound": (C.c_int, [C.c_void_p, C.c_int, C.c_double]),
    "nlopt_get_upper_bounds": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_remove_inequality_constraints": (C.c_int, [C.c_void_p]),
    "nlopt_add_inequality_constraint": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_double]),
    "nlopt_add_precond_inequality_constraint":
        (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_add_inequality_mconstraint":
        (C.c_int, [C.c_void_p, C.c_uint, NLOPT_MFUNC, C.c_void_p, c_double_p]),
    "nlopt_remove_equality_constraints": (C.c_int, [C.c_void_p]),
    "nlopt_add_equality_constraint": (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_double]),
    "nlopt_add_precond_equality_constraint":
        (C.c_int, [C.c_void_p, NLOPT_FUNC, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_add_equality_mconstraint":
        (C.c_int, [C.c_void_p, C.c_uint, NLOPT_MFUNC, C.c_void_p, c_double_p]),
    "nlopt_set_stopval": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_stopval": (C.c_double, [C.c_void_p]),
    "nlopt_set_ftol_rel": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_ftol_rel": (C.c_double, [C.c_void_p]),
    "nlopt_set_ftol_abs": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_ftol_abs": (C.c_double, [C.c_void_p]),
    "nlopt_set_xtol_rel": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_xtol_rel": (C.c_double, [C.c_void_p]),
    "nlopt_set_xtol_abs1": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_set_xtol_abs": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_get_xtol_abs": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_x_weights1": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_set_x_weights": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_get_x_weights": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_maxeval": (C.c_int, [C.c_void_p, C.c_int]),
    "nlopt_get_maxeval": (C.c_int, [C.c_void_p]),
    "nlopt_get_numevals": (C.c_int, [C.c_void_p]),
    "nlopt_set_maxtime": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_maxtime": (C.c_double, [C.c_void_p]),
    "nlopt_force_stop": (C.c_int, [C.c_void_p]),
    "nlopt_set_force_stop": (C.c_int, [C.c_void_p, C.c_int]),
    "nlopt_get_force_stop": (C.c_int, [C.c_void_p]),
    "nlopt_set_local_optimizer": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_set_population": (C.c_int, [C.c_void_p, C.c_uint]),
    "nlopt_get_population": (C.c_uint, [C.c_void_p]),
    "nlopt_set_vector_storage": (C.c_int, [C.c_void_p, C.c_uint]),
    "nlopt_get_vector_storage": (C.c_uint, [C.c_void_p]),
    "nlopt_set_default_initial_step": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_initial_step": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_set_initial_step1": (C.c_int, [C.c_void_p, C.c_double]),
    "nlopt_get_initial_step": (C.c_int, [C.c_void_p, c_double_p, c_double_p]),
    "nlopt_set_munge": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "nlopt_munge_data": (None, [C.c_void_p, C.c_void_p, C.c_void_p]),
    # deprecated one-call API (reference nlopt.h:305-343)
    "nlopt_minimize": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, c_double_p, c_double_p, c_double_p, c_double_p,
                                 C.c_double, C.c_double, C.c_double, C.c_double, c_double_p, C.c_int, C.c_double]),
    "nlopt_minimize_constrained": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t,
                                             c_double_p, c_double_p, c_double_p, c_double_p, C.c_double, C.c_double, C.c_double,
                                             C.c_double, c_double_p, C.c_int, C.c_double]),
    "nlopt_minimize_econstrained": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t,
                                              C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, c_double_p, c_double_p, c_double_p,
                                              c_double_p, C.c_double, C.c_double, C.c_double, C.c_double, c_double_p, C.c_double,
                                              C.c_double, C.c_int, C.c_double]),
    "nlopt_get_local_search_algorithm": (None, [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "nlopt_set_local_search_algorithm": (None, [C.c_int, C.c_int, C.c_int]),
    "nlopt_get_stochastic_population": (C.c_int, []),
    "nlopt_set_stochastic_population": (None, [C.c_int]),
}

# additive extensions, include/nlopt_b200.h
_EXT = {
    "nlopt_b200_set_min_objective_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "nlopt_b200_add_inequality_constraint_device":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_b200_set_min_objective_device2": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "nlopt_b200_set_max_objective_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "nlopt_b200_set_max_objective_device2": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "nlopt_b200_set_max_objective_sharded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "nlopt_b200_add_inequality_constraint_device2":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int]),
    "nlopt_b200_add_equality_constraint_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_b200_add_equality_constraint_device2":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int]),
    "nlopt_b200_add_inequality_mconstraint_device2":
        (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, c_double_p, C.c_int]),
    "nlopt_b200_add_equality_mconstraint_device2":
        (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, c_double_p, C.c_int]),
    "nlopt_b200_set_min_objective_terms": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "nlopt_b200_set_max_objective_terms": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "nlopt_b200_add_inequality_constraint_terms":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int]),
    "nlopt_b200_add_equality_constraint_terms":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int]),
    "nlopt_b200_add_inequality_mconstraint_terms":
        (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, c_double_p, C.c_int]),
    "nlopt_b200_add_equality_mconstraint_terms":
        (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, c_double_p, C.c_int]),
    # __device__ functors given as source, compiled at run time (nlopt_b200_jit)
    "nlopt_b200_jit_create": (C.c_void_p, [C.c_char_p, C.c_char_p, C.POINTER(C.c_char_p), C.c_int]),
    "nlopt_b200_jit_destroy": (None, [C.c_void_p]),
    "nlopt_b200_jit_errmsg": (C.c_char_p, [C.c_void_p]),
    "nlopt_b200_jit_log": (C.c_char_p, [C.c_void_p]),
    "nlopt_b200_jit_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "nlopt_b200_jit_image": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "nlopt_b200_jit_set_min_objective": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "nlopt_b200_jit_set_max_objective": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "nlopt_b200_jit_add_inequality_constraint":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_b200_jit_add_equality_constraint":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_b200_jit_add_inequality_mconstraint":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, c_double_p]),
    "nlopt_b200_jit_add_equality_mconstraint":
        (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, c_double_p]),
    "nlopt_b200_shard_geometry": (None, [C.c_ulonglong, C.c_int, C.c_int, C.c_void_p]),
    "nlopt_b200_set_min_objective_sharded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "nlopt_b200_add_inequality_constraint_sharded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double]),
    "nlopt_b200_optimize_device": (C.c_int, [C.c_void_p, C.c_void_p, c_double_p]),
    "nlopt_b200_set_lower_bounds_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_b200_set_upper_bounds_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_b200_set_xtol_abs_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_b200_set_x_weights_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_b200_set_initial_step_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "nlopt_b200_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "nlopt_b200_dual_create": (C.c_void_p, [C.c_int, C.c_uint, C.c_uint]),
    "nlopt_b200_dual_destroy": (None, [C.c_void_p]),
    "nlopt_b200_dual_errmsg": (C.c_char_p, [C.c_void_p]),
    "nlopt_b200_dual_upload": (C.c_int, [C.c_void_p] + [c_double_p] * 6),
    "nlopt_b200_dual_fill_synthetic": (C.c_int, [C.c_void_p, C.c_ulonglong]),
    "nlopt_b200_dual_set_scalars": (C.c_int, [C.c_void_p, C.c_double, C.c_double, c_double_p, c_double_p]),
    "nlopt_b200_dual_eval": (C.c_int, [C.c_void_p, c_double_p, C.c_int, c_double_p, c_double_p]),
    "nlopt_b200_dual_solve": (C.c_int, [C.c_void_p, c_double_p, c_double_p, c_double_p, C.c_double, C.c_int, c_double_p,
                                        C.POINTER(C.c_int), C.POINTER(C.c_long), c_double_p]),
    "nlopt_b200_dual_download_xcur": (C.c_int, [C.c_void_p, c_double_p]),
    "nlopt_b200_dual_download": (C.c_int, [C.c_void_p, C.c_char_p, c_double_p]),
    "nlopt_b200_dual_sigma_init": (C.c_int, [C.c_void_p, c_double_p, C.c_double]),
    "nlopt_b200_dual_end_outer": (C.c_int, [C.c_void_p, C.c_int, C.c_double, c_double_p, c_double_p,
                                            c_double_p, C.POINTER(C.c_int)]),
    "nlopt_b200_dual_set_prev": (C.c_int, [C.c_void_p, c_double_p, c_double_p, c_double_p]),
    "nlopt_b200_dual_time": (C.c_int, [C.c_void_p, c_double_p, C.c_int, C.c_int, c_double_p]),
    "nlopt_b200_dual_configure": (C.c_int, [C.c_void_p, C.c_char_p, C.c_longlong]),
    "nlopt_b200_dual_query": (C.c_longlong, [C.c_void_p, C.c_char_p]),
    "nlopt_b200_comm_unique_id": (C.c_int, [C.c_char_p]),
    "nlopt_b200_comm_init": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.c_int]),
    "nlopt_b200_comm_finalize": (C.c_int, []),
    "nlopt_b200_comm_rank": (C.c_int, []),
    "nlopt_b200_comm_world": (C.c_int, []),
    "nlopt_b200_shard_range": (None, [C.c_ulonglong, C.c_int, C.c_int,
                                      C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]),
    "nlopt_b200_release_cached_memory": (None, []),
    "nlopt_b200_device_count": (C.c_int, []),
    "nlopt_b200_build_info": (C.c_char_p, []),
}

STD_SYMBOLS = tuple(_STD)
EXT_SYMBOLS = tuple(_EXT)


class Library:
    """A loaded shared library exporting the NLopt C ABI (and, for the product, the extensions)."""

    def __init__(self, path: str | None = None, extensions: bool | None = None):
        self.path = path or DEFAULT_LIB
        if not os.path.exists(self.path):
            raise OSError(
                f"{self.path} not found -- build it first: python -c 'import __graft_entry__ as g; g.build()'")
        # RTLD_LOCAL: the reference library (tests) exports the same nlopt_* names; neither may
        # interpose on the other
        self.dll = C.CDLL(self.path, mode=C.RTLD_LOCAL)
        self.has_extensions = (path is None) if extensions is None else extensions
        for name, (res, args) in _STD.items():
            fn = getattr(self.dll, name)
            fn.restype, fn.argtypes = res, args
            setattr(self, name, fn)
        if self.has_extensions:
            for name, (res, args) in _EXT.items():
                fn = getattr(self.dll, name)
                fn.restype, fn.argtypes = res, args
                setattr(self, name, fn)


_default = None


def default_library() -> Library:
    """The product library; NLOPT_B200_LIBRARY_PATH points the module at another library exporting the NLopt C ABI
    (tests: the CPU-backed build of the host logic, or the reference itself)."""
    global _default
    if _default is None:
        alt = os.environ.get("NLOPT_B200_LIBRARY_PATH")
        _default = Library(alt, extensions=False) if alt else Library()
    return _default
