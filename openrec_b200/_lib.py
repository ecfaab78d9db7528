"""ctypes binding of liborx.so (declared in include/orx.h).

There is NO CPU fallback: if the shared library is missing this module raises at import of
the first symbol; if no CUDA device is present every compute entry point returns ORX_ERR_CUDA,
which `check` turns into a RuntimeError.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "liborx.so")

ORX_PAIR_BPR, ORX_PAIR_UCML = 0, 1
ORX_POINT_GMF, ORX_POINT_WRMF = 0, 1
ORX_SCORE_DOT, ORX_SCORE_NEG_SQDIST = 0, 1
ORX_OPT_SGD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_LAZY, ORX_OPT_ADAM_DENSE, ORX_OPT_ROWWISE_ADAGRAD = 0, 1, 2, 3, 5   # 4: unassigned
ORX_OPT_MOMENTUM, ORX_OPT_NESTEROV = 6, 8   # 7: unassigned
ORX_OP_GEMM, ORX_OP_INTERACT_FWD, ORX_OP_INTERACT_BWD, ORX_OP_PAIRWISE_STEP, ORX_OP_POINTWISE_STEP = 0, 1, 2, 3, 4
ORX_OP_SCORE_RANK, ORX_OP_SCORE_TOPK, ORX_OP_SCORE_RANK_SHARD, ORX_OP_SCORE_TOPK_SHARD = 5, 6, 7, 8
ORX_OP_POINTWISE_GRAD_ROWS, ORX_OP_CENSOR_SHARD, ORX_OP_CROSS, ORX_OP_PAIRWISE_STEP_BF16 = 9, 10, 11, 12
ORX_OP_POINTWISE_STEP_BF16, ORX_OP_SCORE_RANK_BF16, ORX_OP_SCORE_TOPK_BF16 = 13, 14, 15
ORX_VARIANT_GEMM_TMA, ORX_VARIANT_GEMM_SIMT, ORX_VARIANT_INTERACT_WARP, ORX_VARIANT_INTERACT = 0, 1, 2, 3
ORX_VARIANT_STEP, ORX_VARIANT_STEP_PIPE, ORX_VARIANT_STEP_GENERIC = 4, 5, 6
ORX_VARIANT_RANK_SMEM, ORX_VARIANT_RANK_GLOBAL, ORX_VARIANT_TOPK = 7, 8, 9
ORX_VARIANT_CENSOR_VEC, ORX_VARIANT_CENSOR_SCALAR = 10, 11
ORX_VARIANT_CROSS_VEC, ORX_VARIANT_CROSS_SCALAR = 12, 13
ORX_CROSS_TOP, ORX_CROSS_MID, ORX_CROSS_FINAL = 0, 1, 2
ORX_CENSOR_SHARD_MAX_IDS = 1 << 28
ORX_MAX_AT = 8
ORX_BAG_MAX_TABLES = 63
ORX_MAX_TOPK = 1024
ORX_DISPATCH_LOG_CAP = 64


class OrxOpt(C.Structure):
    _fields_ = [("kind", C.c_int32), ("lr", C.c_float), ("eps", C.c_float), ("beta1", C.c_float),
                ("beta2", C.c_float), ("step", C.c_int64)]


class OrxTable(C.Structure):
    _fields_ = [("var", C.c_void_p), ("s0", C.c_void_p), ("s1", C.c_void_p), ("rows", C.c_int64),
                ("dim", C.c_int32)]


class OrxTableBf16(C.Structure):
    _fields_ = [("var", C.c_void_p), ("s0", C.c_void_p), ("s1", C.c_void_p), ("rows", C.c_int64),
                ("dim", C.c_int32)]


class OrxShard(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("dim", C.c_int32), ("batch_cap", C.c_int32),
                ("home_cap", C.c_int32), ("req_cap", C.c_int32), ("gin_cap", C.c_int32), ("timeout_ms", C.c_int32),
                ("tripbox", C.c_void_p), ("idbox", C.c_void_p), ("got", C.c_void_p), ("gotb", C.c_void_p),
                ("gin", C.c_void_p), ("ginb", C.c_void_p), ("meta", C.c_void_p), ("flags", C.c_void_p)]


class OrxRowShard(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("total_users", C.c_int64), ("total_items", C.c_int64),
                ("local_users", C.c_int64), ("local_items", C.c_int64)]


class OrxSampler(C.Structure):
    _fields_ = [("rec_user", C.c_void_p), ("rec_item", C.c_void_p), ("perm_cur", C.c_void_p), ("perm_next", C.c_void_p),
                ("cursor", C.c_int64), ("n_records", C.c_int64), ("csr_off", C.c_void_p), ("csr_items", C.c_void_p),
                ("total_users", C.c_int32), ("total_items", C.c_int32)]


_vp, _i32, _i64, _f, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_uint64
_T = C.POINTER(OrxTable)
_TB = C.POINTER(OrxTableBf16)
_O = C.POINTER(OrxOpt)
_S = C.POINTER(OrxShard)

# name -> argtypes (restype is int unless noted); mirrors include/orx.h one to one
SIGNATURES = {
    "orx_abi_version": [],
    "orx_last_error_string": [],
    "orx_create": [C.c_int, C.POINTER(_vp)],
    "orx_destroy": [_vp],
    "orx_device_count": [C.POINTER(C.c_int)],
    "orx_stream_synchronize": [_vp, _vp],
    "orx_debug_set_epoch": [_vp, C.c_uint32],
    "orx_debug_dispatch_log": [_vp, C.POINTER(_i32), _i32, C.POINTER(_i32)],
    "orx_debug_pair_records": [_vp, _i32, _vp, _i32, _vp],
    "orx_debug_round_bf16": [_vp, _vp, _vp, _i64, _i64, _i32, _i32, _u64, _i64, _vp],
    "orx_profile_enable": [_vp, _i32],
    "orx_profile_read": [_vp, C.POINTER(C.c_float), _i32, C.POINTER(_i32)],
    "orx_fill_uniform": [_vp, _vp, _i64, _f, _f, _u64, _vp],
    "orx_gather": [_vp, _vp, _i64, _i32, _vp, _i32, _i64, _vp, _vp, _vp],
    "orx_censor": [_vp, _vp, _i64, _i32, _vp, _i32, _f, _vp],
    "orx_censor_shard": [_vp, _vp, _i64, _i32, _i64, _i32, _i32, _vp, _i32, _i64, _i32, _f, _vp],
    "orx_pairwise_step": [_vp, _i32, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _O, _vp, _vp],
    "orx_pairwise_step_host": [_vp, _i32, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _O, _vp, _vp],
    "orx_pairwise_prefetch": [_vp, _T, _T, _vp, _vp, _vp, _i32, _i32, _i32, _vp],
    "orx_pairwise_fwd": [_vp, _i32, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _vp, _vp],
    "orx_pairwise_grad": [_vp, _i32, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_pairwise_step_bf16": [_vp, _i32, _TB, _TB, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _O, _u64, _vp, _vp],
    "orx_pairwise_step_host_bf16": [_vp, _i32, _TB, _TB, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _O, _u64, _vp, _vp],
    "orx_pairwise_fwd_bf16": [_vp, _i32, _TB, _TB, _T, _vp, _vp, _vp, _i32, _f, _vp, _vp],
    "orx_pairwise_grad_bf16": [_vp, _i32, _TB, _TB, _T, _vp, _vp, _vp, _i32, _f, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp,
                               _vp],
    "orx_censor_bf16": [_vp, _vp, _i64, _i32, _vp, _i32, _f, _vp],
    "orx_sparse_apply": [_vp, _T, _vp, _vp, _i32, _O, _vp],
    "orx_sparse_apply_strided": [_vp, _T, _vp, _i64, _vp, _i64, _i32, _O, _vp],
    "orx_gather_strided": [_vp, _vp, _i64, _i32, _vp, _i64, _i64, _vp, _i64, _vp, _vp],
    "orx_bag_gather": [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _i64, C.POINTER(_i32), _i32, _i32, _vp,
                       _i64, _vp, _vp],
    "orx_gather_strided_bf16": [_vp, _vp, _i64, _i32, _vp, _i64, _i64, _vp, _i64, _vp, _vp],
    "orx_bag_gather_bf16": [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _i64, C.POINTER(_i32), _i32, _i32,
                            _vp, _i64, _vp, _vp],
    "orx_bag_sparse_apply": [_vp, _T, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _O, _vp],
    "orx_sparse_apply_strided_bf16": [_vp, _TB, _vp, _i64, _vp, _i64, _i32, _O, _u64, _vp],
    "orx_bag_sparse_apply_bf16": [_vp, _TB, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _O, _u64, _vp],
    "orx_mlp_layer_fwd": [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _i64, _vp],
    "orx_mlp_layer_bwd": [_vp, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _vp, _vp],
    "orx_interact_fwd": [_vp, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp],
    "orx_interact_bwd": [_vp, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64,
                         _vp],
    "orx_pred_loss": [_vp, _vp, _vp, _i32, _i32, _f, _vp, _vp, _vp, _vp],
    "orx_cross_fwd": [_vp, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _vp],
    "orx_cross_bwd": [_vp, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _vp,
                      _i64, _vp, _i64, _vp],
    "orx_peer_alloc": [_vp, _i64, C.POINTER(_vp), C.c_char_p],
    "orx_peer_open": [_vp, C.c_char_p, C.POINTER(_vp)],
    "orx_peer_close": [_vp, _vp],
    "orx_peer_free": [_vp, _vp],
    "orx_shard_sizes": [_S, C.POINTER(_i64)],
    "orx_shard_step": [_vp, _i32, _S, _T, _T, _T, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _i64, _i64, _f, _f, _f, _f, _O,
                       _i32, _i32, _i32, _vp, _vp],
    "orx_owner_bucket_combined": [_vp, _vp, _i32, _i32, _i64, _i32, _vp, _vp, _vp, _vp],
    "orx_pairwise_grad_rows": [_vp, _i32, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _f, _f, _f, _f, _vp, _vp, _vp],
    "orx_lookup_bucket": [_vp, _vp, _i32, _i32, C.POINTER(_i64), _i32, _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_rows_segment_sum": [_vp, _vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp],
    "orx_bag_shard_lookups": [_vp, _vp, _i32, _i32, C.POINTER(_i32), C.POINTER(_i64), _vp, _vp],
    "orx_bag_segment_sum": [_vp, _vp, _i64, _i32, _i32, C.POINTER(_i32), _i32, _vp, _i32, _vp, _vp, _i32, _vp, _vp],
    "orx_pointwise_shard_lookups": [_vp, _vp, _vp, _i32, _i64, _i64, _vp, _vp],
    "orx_pointwise_serve": [_vp, _vp, _vp, _vp, _i32, _i64, _i64, _i64, _vp, _i32, _i64, _vp, _vp, _vp, _vp],
    "orx_pointwise_grad_rows": [_vp, _i32, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _f, _f, _i32, _f, _f, _f, _i32, _vp,
                                _vp, _vp, _vp],
    "orx_rows_scale": [_vp, _vp, _i64, _i32, _vp, _vp],
    "orx_pointwise_step": [_vp, _i32, _T, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _f, _f, _O, _vp, _vp],
    "orx_pointwise_fwd": [_vp, _i32, _T, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _vp, _vp],
    "orx_pointwise_grad": [_vp, _i32, _T, _T, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _f, _f,
                           _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_pointwise_step_bf16": [_vp, _i32, _TB, _TB, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _f, _f, _O, _u64, _vp,
                                _vp],
    "orx_pointwise_fwd_bf16": [_vp, _i32, _TB, _TB, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _vp, _vp],
    "orx_pointwise_grad_bf16": [_vp, _i32, _TB, _TB, _T, _T, _vp, _vp, _vp, _i32, _f, _f, _i32, _f, _f,
                                _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_dense_apply": [_vp, _vp, _vp, _vp, _vp, _i64, _O, _vp],
    "orx_score_all": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp],
    "orx_score_all_bf16": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp],
    "orx_sample_pairwise": [_vp, C.POINTER(OrxSampler), _u64, _i64, _i32, _vp, _vp, _vp, _vp],
    "orx_sample_stratified": [_vp, C.POINTER(OrxSampler), _u64, _i64, _i32, _f, _vp, _vp, _vp, _vp, _vp],
    "orx_sample_per_positive": [_vp, C.POINTER(OrxSampler), _u64, _i64, _i32, _i32, _vp, _vp, _vp, _vp],
    "orx_rank_metrics": [_vp, _vp, _vp, _vp, _i32, _i64, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp],
    "orx_score_rank": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _i32,
                       C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp],
    "orx_score_rank_bf16": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _i32,
                            C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp],
    "orx_score_topk": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp],
    "orx_score_topk_bf16": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp],
    "orx_score_rank_shard_sizes": [_i32, _i32, _i32, C.POINTER(_i64)],
    "orx_score_rank_shard": [_vp, _i32, _i32, C.POINTER(OrxRowShard), _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp,
                             _i32, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_score_rank_listed": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                              _i32, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp],
    "orx_score_rank_listed_bf16": [_vp, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _i32, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp],
    "orx_score_rank_listed_shard": [_vp, _i32, _i32, C.POINTER(OrxRowShard), _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp,
                                    _vp, _vp, _vp, _vp, _i32, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "orx_score_topk_shard": [_vp, _i32, _i32, C.POINTER(OrxRowShard), _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _i32,
                             _vp, _vp, _vp, _vp, _vp],
}

_lib = None


def lib():
    """Load liborx.so once.  Fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"liborx.so not found at {LIB_PATH}: build it with `python -m openrec_b200.build` "
                "(there is no CPU fallback)")
        l = C.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(l, name)
            fn.argtypes = argtypes
            fn.restype = C.c_char_p if name == "orx_last_error_string" else C.c_int
        _lib = l
    return _lib


def last_error() -> str:
    s = lib().orx_last_error_string()
    return s.decode() if s else ""


def check(rc: int, what: str = "liborx"):
    if rc != 0:
        raise RuntimeError(f"{what} failed (status {rc}): {last_error()}")
