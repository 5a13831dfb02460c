"""ctypes loader for libjolt_b200.so (the C ABI declared in include/jolt_b200.h).

There is no fallback of any kind: if the shared library is missing the import fails, and if no
CUDA device is present every compute entry point returns JB_ERR_NO_DEVICE, surfaced here as
`JoltB200Error`."""
from __future__ import annotations

import ctypes
import pathlib

_HERE = pathlib.Path(__file__).resolve().parent
LIB_PATH = _HERE / "libjolt_b200.so"

c_u64p = ctypes.POINTER(ctypes.c_uint64)
c_size_t = ctypes.c_size_t
c_void_p = ctypes.c_void_p

# name -> (restype, argtypes); must list every symbol of include/jolt_b200.h (tests check this)
SIGNATURES = {
    "jb_version": (ctypes.c_char_p, []),
    "jb_status_str": (ctypes.c_char_p, [ctypes.c_int]),
    "jb_device_count": (ctypes.c_int, []),
    "jb_ctx_create": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(c_void_p)]),
    "jb_ctx_create_on_stream": (ctypes.c_int, [ctypes.c_int, c_void_p, ctypes.POINTER(c_void_p)]),
    "jb_ctx_destroy": (None, [c_void_p]),
    "jb_last_error": (ctypes.c_char_p, [c_void_p]),
    "jb_ctx_synchronize": (ctypes.c_int, [c_void_p]),
    "jb_ctx_launch_count": (ctypes.c_uint64, [c_void_p]),
    "jb_table_upload": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p]),
    "jb_table_alloc": (ctypes.c_int, [c_void_p, c_size_t, c_u64p]),
    "jb_table_wrap_device": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, c_u64p]),
    "jb_table_len": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.POINTER(c_size_t)]),
    "jb_table_device_ptr": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.POINTER(c_void_p)]),
    "jb_table_download": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_u64p, c_size_t]),
    "jb_table_clone": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_u64p]),
    "jb_table_free": (ctypes.c_int, [c_void_p, ctypes.c_uint64]),
    "jb_table_bind": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_u64p, ctypes.c_int]),
    "jb_table_upload_small": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]),
    "jb_table_bind_small": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, ctypes.c_int, c_u64p, ctypes.c_int,
                                           ctypes.POINTER(ctypes.c_uint64)]),
    "jb_eq_evals": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p, c_u64p]),
    "jb_eq_evals_aligned_block": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_size_t, c_size_t, c_u64p]),
    "jb_member_create": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, ctypes.c_int, ctypes.POINTER(c_void_p)]),
    "jb_member_create_sop": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_size_t, ctypes.c_int, ctypes.POINTER(c_void_p)]),
    "jb_member_num_tables": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_size_t)]),
    "jb_member_context": (c_void_p, [c_void_p]),
    "jb_scheduler_create": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), c_size_t, ctypes.POINTER(c_void_p)]),
    "jb_scheduler_prove_round": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, c_u64p]),
    "jb_scheduler_finish_rounds": (ctypes.c_int, [c_void_p, c_void_p, c_size_t]),
    "jb_scheduler_destroy": (None, [c_void_p]),
    "jb_member_num_rounds": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_size_t)]),
    "jb_member_degree": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_size_t)]),
    "jb_member_prove_round": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p, c_u64p]),
    "jb_member_finish_rounds": (ctypes.c_int, [c_void_p, c_u64p]),
    "jb_member_final_evals": (ctypes.c_int, [c_void_p, c_u64p]),
    "jb_eq_member_create": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p, c_size_t, c_u64p, ctypes.c_int,
                                           ctypes.POINTER(c_void_p)]),
    "jb_eq_member_scalar": (ctypes.c_int, [c_void_p, c_u64p]),
    "jb_member_create_expr": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_void_p, c_size_t, c_u64p, c_size_t, c_u64p,
                                             ctypes.c_int, ctypes.POINTER(c_void_p)]),
    "jb_member_create_expr_sources": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, c_size_t, c_void_p, c_size_t, c_u64p,
                                                     c_size_t, c_u64p, ctypes.c_int, ctypes.POINTER(c_void_p)]),
    "jb_member_prove_round_partials": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, ctypes.c_int, c_void_p]),
    "jb_ctx_set_verify_rounds": (ctypes.c_int, [c_void_p, ctypes.c_int]),
    "jb_partials_finalize": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, c_u64p]),
    "jb_lanes_reduce_host": (ctypes.c_int, [c_u64p, c_size_t, c_u64p]),
    "jb_wide_lanes_reduce_host": (ctypes.c_int, [c_u64p, c_size_t, c_u64p]),
    "jb_round_evals_from_kernel_values": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, c_u64p, c_u64p, c_u64p]),
    "jb_member_export_table": (ctypes.c_int, [c_void_p, c_size_t, c_void_p, c_size_t, ctypes.POINTER(c_size_t)]),
    "jb_comm_unique_id": (ctypes.c_int, [ctypes.POINTER(ctypes.c_uint8), ctypes.c_char_p]),
    "jb_comm_init": (ctypes.c_int, [c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint8), ctypes.c_char_p]),
    "jb_comm_destroy": (ctypes.c_int, [c_void_p]),
    "jb_comm_p2p_handle": (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint8)]),
    "jb_comm_p2p_open": (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint8)]),
    "jb_sharded_member_create": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, ctypes.c_int, c_size_t, ctypes.POINTER(c_void_p)]),
    "jb_member_destroy": (None, [c_void_p]),
    "jb_prove_batch": (ctypes.c_int, [ctypes.POINTER(c_void_p), c_void_p, c_size_t, c_size_t, c_size_t, c_u64p,
                                      ctypes.c_int, c_void_p, c_void_p, c_u64p, c_u64p, c_u64p, c_u64p,
                                      ctypes.POINTER(c_size_t)]),
    "jb_absorb_round_splitmix125": (ctypes.c_int, [c_void_p, c_size_t, c_u64p, c_size_t, c_u64p]),
    "jb_srs_upload_affine": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p]),
    "jb_srs_upload_jacobian": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p]),
    "jb_srs_generate_multiples": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p]),
    "jb_srs_precompute": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.c_int]),
    "jb_srs_len": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.POINTER(c_size_t)]),
    "jb_srs_download_affine": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_u64p, c_size_t]),
    "jb_srs_free": (ctypes.c_int, [c_void_p, ctypes.c_uint64]),
    "jb_msm_g1": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, c_u64p, c_size_t, c_u64p]),
    "jb_msm_g1_small": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, c_void_p, c_size_t, ctypes.c_int, c_u64p]),
    "jb_msm_g1_batch": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, ctypes.POINTER(c_void_p), ctypes.POINTER(c_size_t),
                                        ctypes.POINTER(ctypes.c_int), c_u64p]),
    "jb_msm_g1_rows": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_void_p, c_size_t, c_size_t, ctypes.c_int, c_u64p]),
    "jb_msm_g1_one_hot_rows": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.POINTER(c_void_p), c_size_t, ctypes.c_int,
                                              c_size_t, c_size_t, c_size_t, ctypes.c_int, c_u64p]),
    "jb_msm_g1_table": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, ctypes.c_uint64, c_size_t, c_u64p]),
    "jb_table_evaluate_batch": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, c_u64p, c_size_t, c_u64p]),
    "jb_small_evaluate_batch": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), c_size_t, ctypes.POINTER(ctypes.c_int),
                                               c_size_t, ctypes.c_int, c_u64p, c_size_t, c_u64p]),
    "jb_one_hot_evaluate": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), c_size_t, ctypes.c_int, c_size_t, c_size_t,
                                           ctypes.c_int, ctypes.c_int, c_u64p, c_u64p]),
    "jb_one_hot_pushforward": (ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), c_size_t, ctypes.c_int, c_size_t,
                                              c_size_t, ctypes.c_int, c_u64p, c_u64p]),
    "jb_table_linear_combination": (ctypes.c_int, [c_void_p, c_void_p, c_size_t, c_size_t, c_u64p]),
    "jb_ctx_diag": (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_double)]),
    "jb_ctx_run_log": (ctypes.c_int, [c_void_p, c_u64p, c_size_t, ctypes.POINTER(c_size_t)]),
    "jb_ctx_timing_enable": (ctypes.c_int, [c_void_p, ctypes.c_int, ctypes.c_uint64]),
    "jb_ctx_timing_collect": (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_int), c_u64p, ctypes.POINTER(ctypes.c_int),
                                             ctypes.POINTER(ctypes.c_double), c_size_t, ctypes.POINTER(c_size_t)]),
    "jb_diag_mul_throughput": (ctypes.c_int, [c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.POINTER(ctypes.c_double)]),
    "jb_g1_batch_add": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_u64p, ctypes.POINTER(ctypes.c_uint32), c_size_t, c_u64p]),
    "jb_msm_g1_sharded": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, c_u64p, c_size_t, c_u64p]),
    "jb_msm_g1_device": (ctypes.c_int, [c_void_p, ctypes.c_uint64, c_size_t, c_void_p, c_size_t, c_u64p]),
    "jb_hyperkzg_open": (ctypes.c_int, [c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_u64p, c_size_t, c_void_p, c_void_p,
                                        c_void_p, c_u64p, c_u64p, c_u64p]),
    "jb_vec_op": (ctypes.c_int, [c_void_p, ctypes.c_int, ctypes.c_int, c_u64p, c_u64p, c_u64p, c_size_t]),
}

JB_OK, JB_ERR_NO_DEVICE, JB_ERR_CUDA, JB_ERR_INVALID, JB_ERR_OOM, JB_ERR_ROUND_CHECK, JB_ERR_UNSUPPORTED, \
    JB_ERR_LENGTH = range(8)


class JoltB200Error(RuntimeError):
    def __init__(self, status: int, detail: str):
        self.status = status
        super().__init__(f"jolt_b200 status {status}: {detail}")


class BatchMemberC(ctypes.Structure):
    _fields_ = [("input_claim", ctypes.c_uint64 * 4), ("coefficient", ctypes.c_uint64 * 4),
                ("rounds", c_size_t), ("offset", c_size_t)]


class RoundWorkC(ctypes.Structure):
    _fields_ = [("member", c_size_t), ("round", c_size_t), ("has_bind", ctypes.c_int), ("has_claim", ctypes.c_int),
                ("bind", ctypes.c_uint64 * 4), ("claim", ctypes.c_uint64 * 4)]


JB_EXPR_MAX_TABLES, JB_EXPR_MAX_MONOMIALS, JB_EXPR_MAX_DEGREE = 8, 16, 6


class MonomialC(ctypes.Structure):
    _fields_ = [("coeff", ctypes.c_uint64 * 4), ("degree", ctypes.c_uint32),
                ("table", ctypes.c_uint32 * JB_EXPR_MAX_DEGREE)]


JB_SOURCE_TABLE, JB_SOURCE_COMPACT, JB_SOURCE_ONE_HOT = 0, 1, 2


class SourceC(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("kind", ctypes.c_int), ("on_device", ctypes.c_int), ("table", ctypes.c_uint64),
                ("values", c_void_p), ("K", c_size_t), ("r_addr", c_u64p)]


JB_LC_TABLE, JB_LC_COMPACT, JB_LC_ONE_HOT = 0, 1, 2


class LcTermC(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("kind", ctypes.c_int), ("on_device", ctypes.c_int), ("layout", ctypes.c_int),
                ("table", ctypes.c_uint64), ("values", c_void_p), ("len", c_size_t), ("K", c_size_t),
                ("coeff", ctypes.c_uint64 * 4)]


class FinishWorkC(ctypes.Structure):
    _fields_ = [("member", c_size_t), ("bind", ctypes.c_uint64 * 4)]


HKZG_R_FN = ctypes.CFUNCTYPE(ctypes.c_int, c_void_p, c_u64p, c_size_t, c_u64p)
HKZG_Q_FN = ctypes.CFUNCTYPE(ctypes.c_int, c_void_p, c_u64p, c_size_t, c_u64p)
ABSORB_FN = ctypes.CFUNCTYPE(ctypes.c_int, c_void_p, c_size_t, c_u64p, c_size_t, c_u64p)

_lib = None


def load():
    """Loads the CUDA extension; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError(
                f"{LIB_PATH} is missing - build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(jolt_b200 has no CPU fallback)")
        lib = ctypes.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
