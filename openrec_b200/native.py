"""Thin torch-tensor front of the C-ABI: torch owns device memory and streams (plumbing),
liborx does all the arithmetic.  Every function enqueues on torch's current CUDA stream."""
from __future__ import annotations

import ctypes as C
from collections import namedtuple

import torch

from . import _lib
from ._lib import (ORX_OP_GEMM, ORX_OP_INTERACT_BWD, ORX_OP_INTERACT_FWD, ORX_OP_PAIRWISE_STEP, ORX_OP_POINTWISE_STEP,
                   ORX_OP_POINTWISE_GRAD_ROWS, ORX_OP_CENSOR_SHARD, ORX_VARIANT_CENSOR_SCALAR, ORX_VARIANT_CENSOR_VEC,
                   ORX_OP_SCORE_RANK, ORX_OP_SCORE_RANK_SHARD, ORX_OP_SCORE_TOPK, ORX_OP_SCORE_TOPK_SHARD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_DENSE, ORX_OPT_ADAM_LAZY, ORX_OPT_SGD,
                   ORX_OPT_ROWWISE_ADAGRAD, ORX_OPT_MOMENTUM, ORX_OPT_NESTEROV, ORX_PAIR_BPR,
                   ORX_PAIR_UCML, ORX_POINT_GMF, ORX_POINT_WRMF, ORX_SCORE_DOT, ORX_SCORE_NEG_SQDIST, ORX_VARIANT_GEMM_SIMT,
                   ORX_VARIANT_GEMM_TMA, ORX_VARIANT_INTERACT, ORX_VARIANT_INTERACT_WARP, ORX_VARIANT_RANK_GLOBAL,
                   ORX_VARIANT_RANK_SMEM, ORX_VARIANT_STEP, ORX_VARIANT_STEP_GENERIC, ORX_VARIANT_STEP_PIPE,
                   ORX_VARIANT_TOPK, ORX_OP_CROSS, ORX_VARIANT_CROSS_VEC, ORX_VARIANT_CROSS_SCALAR, ORX_CROSS_TOP,
                   ORX_CROSS_MID, ORX_CROSS_FINAL, ORX_OP_PAIRWISE_STEP_BF16, ORX_OP_POINTWISE_STEP_BF16, OrxOpt,
                   ORX_OP_SCORE_RANK_BF16, ORX_OP_SCORE_TOPK_BF16, OrxTable, OrxTableBf16)

__all__ = ["Engine", "engine", "table", "opt", "ORX_PAIR_BPR", "ORX_PAIR_UCML", "ORX_POINT_GMF", "ORX_POINT_WRMF",
           "ORX_OPT_SGD", "ORX_OPT_ADAGRAD", "ORX_OPT_ADAM_LAZY", "ORX_OPT_ADAM_DENSE", "ORX_OPT_ROWWISE_ADAGRAD",
           "ORX_OPT_MOMENTUM", "ORX_OPT_NESTEROV", "ORX_SCORE_DOT",
           "ORX_SCORE_NEG_SQDIST", "ORX_OP_GEMM", "ORX_OP_INTERACT_FWD", "ORX_OP_INTERACT_BWD", "ORX_OP_PAIRWISE_STEP",
           "ORX_OP_POINTWISE_STEP", "ORX_VARIANT_GEMM_TMA", "ORX_VARIANT_GEMM_SIMT", "ORX_VARIANT_INTERACT_WARP",
           "ORX_VARIANT_INTERACT", "ORX_VARIANT_STEP", "ORX_VARIANT_STEP_PIPE", "ORX_VARIANT_STEP_GENERIC",
           "ORX_OP_SCORE_RANK", "ORX_VARIANT_RANK_SMEM", "ORX_VARIANT_RANK_GLOBAL", "ORX_OP_SCORE_TOPK",
           "ORX_VARIANT_TOPK", "ORX_OP_SCORE_RANK_SHARD", "ORX_OP_SCORE_TOPK_SHARD", "ORX_OP_POINTWISE_GRAD_ROWS",
           "ORX_OP_CENSOR_SHARD", "ORX_VARIANT_CENSOR_VEC", "ORX_VARIANT_CENSOR_SCALAR", "ORX_OP_CROSS",
           "ORX_VARIANT_CROSS_VEC", "ORX_VARIANT_CROSS_SCALAR", "ORX_CROSS_TOP", "ORX_CROSS_MID", "ORX_CROSS_FINAL",
           "ORX_OP_PAIRWISE_STEP_BF16", "ORX_OP_POINTWISE_STEP_BF16", "ORX_OP_SCORE_RANK_BF16",
           "ORX_OP_SCORE_TOPK_BF16", "table_bf16", "as_table",
           "Dispatch", "RowShard", "rowshard", "shard_rows"]

_engines = {}

# one record of orx_debug_dispatch_log: which kernel an orx_mlp_layer_* / orx_interact_* call or a sparse step launched
# (the field meanings per op are in include/orx.h)
Dispatch = namedtuple("Dispatch", "op variant ta tb m n k s")

# geometry of a row-sharded table pair: row r of every table lives on rank r % world at local row r // world
RowShard = namedtuple("RowShard", "world rank total_users total_items local_users local_items")


def shard_rows(total, rank, world):
    """The local row count of `rank` in the row-sharded layout of a `total`-row table: ceil((total - rank) / world),
    0 for a rank past the table's end.  A rank without rows stores a 1-row dummy: its shard has max(rows, 1) rows."""
    return max((int(total) - rank + world - 1) // world, 0)


def rowshard(world, rank, total_users, total_items):
    """RowShard of `rank` (local_* from shard_rows)."""
    return RowShard(world, rank, total_users, total_items, shard_rows(total_users, rank, world),
                    shard_rows(total_items, rank, world))


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _f32(t, name):
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise ValueError(f"{name}: expected a contiguous float32 CUDA tensor")
    return t


def ids32(t):
    """int32 contiguous CUDA ids (Keras Embedding casts other integer dtypes to int32)."""
    if not t.is_cuda:
        raise ValueError("ids must live on the CUDA device")
    if t.dtype != torch.int32:
        t = t.to(torch.int32)
    return t.contiguous().reshape(-1)


def table(var, s0=None, s1=None, kind=None):
    """orx_table_t for a [rows, dim] variable and its optimizer slots.  With kind=ORX_OPT_ROWWISE_ADAGRAD, s0 is the
    table's one accumulator per row: ``[rows]`` or ``[rows, 1]``, anything else is refused."""
    _f32(var, "var"), _f32(s0, "s0"), _f32(s1, "s1")
    rows, dim = (var.shape[0], var.shape[1]) if var.dim() == 2 else (1, var.numel())
    if kind == ORX_OPT_ROWWISE_ADAGRAD and s0 is not None and tuple(s0.shape) not in ((rows,), (rows, 1)):
        raise ValueError(f"s0: a row-wise Adagrad accumulator has one element per row, shape ({rows},) or ({rows}, 1), "
                         f"got {tuple(s0.shape)}")
    return OrxTable(var.data_ptr(), s0.data_ptr() if s0 is not None else None,
                    s1.data_ptr() if s1 is not None else None, rows, dim)


def _bf16(t, name):
    if not (t.is_cuda and t.dtype == torch.bfloat16 and t.is_contiguous()):
        raise ValueError(f"{name}: expected a contiguous bfloat16 CUDA tensor")
    return t


def _score_tables(op, user_tab, item_tab):
    """-> (entry point, user_tab, item_tab) of scoring call `op` for the tables' dtype: op itself on float32 tables, its
    _bf16 form on bfloat16 ones (bit-equal to op on their float32 upcast).  Mixed dtypes are refused."""
    if user_tab.dtype == torch.float32 and item_tab.dtype == torch.float32:
        return op, _f32(user_tab, "user_tab"), _f32(item_tab, "item_tab")
    if user_tab.dtype == torch.bfloat16 and item_tab.dtype == torch.bfloat16:
        return op + "_bf16", _bf16(user_tab, "user_tab"), _bf16(item_tab, "item_tab")
    raise ValueError(f"{op}: user_tab and item_tab must both be float32 or both bfloat16, got {user_tab.dtype} and "
                     f"{item_tab.dtype}")


def _sr_seed(sr_seed, op):
    """The uint64 rounding seed of a bf16 table's apply; a bf16 table has no default seed."""
    if sr_seed is None:
        raise ValueError(f"{op}: a bfloat16 table's updates need sr_seed")
    return int(sr_seed) & 0xFFFFFFFFFFFFFFFF


def table_bf16(var, s0=None, s1=None, kind=None):
    """orx_table_bf16_t for a bfloat16 [rows, dim] variable and its float32 optimizer slots (checked as in table)."""
    _bf16(var, "var"), _f32(s0, "s0"), _f32(s1, "s1")
    rows, dim = var.shape[0], var.shape[1]
    if kind == ORX_OPT_ROWWISE_ADAGRAD and s0 is not None and tuple(s0.shape) not in ((rows,), (rows, 1)):
        raise ValueError(f"s0: a row-wise Adagrad accumulator has one element per row, shape ({rows},) or ({rows}, 1), "
                         f"got {tuple(s0.shape)}")
    return OrxTableBf16(var.data_ptr(), s0.data_ptr() if s0 is not None else None,
                        s1.data_ptr() if s1 is not None else None, rows, dim)


def as_table(t):
    """The orx_table_t with the fields of an orx_table_bf16_t t (orx_pairwise_prefetch reads its rows and dim)."""
    return t if isinstance(t, OrxTable) else OrxTable(t.var, t.s0, t.s1, t.rows, t.dim)


def opt(kind, lr, eps=1e-7, beta1=0.9, beta2=0.999, step=1):
    """orx_opt_t.  Under ORX_OPT_MOMENTUM / ORX_OPT_NESTEROV, beta1 is the momentum coefficient."""
    return OrxOpt(kind, lr, eps, beta1, beta2, step)


def _csr(off, items, n_rows):
    """Check a per-user CSR list (int64 offsets [n_rows + 1], int32 items, on the device) -> (off, items or None when
    empty); (None, None) when off is None."""
    if off is None:
        return None, None
    if not (off.is_cuda and off.dtype == torch.int64 and off.is_contiguous()):
        raise ValueError("CSR offsets: expected a contiguous int64 CUDA tensor")
    if not (items.is_cuda and items.dtype == torch.int32 and items.is_contiguous()):
        raise ValueError("CSR items: expected a contiguous int32 CUDA tensor")
    if off.numel() != n_rows + 1:
        raise ValueError("CSR offsets must have one entry per user row plus one")
    return off, items if items.numel() else None


class Engine:
    """One liborx context (workspace) per CUDA device."""

    def __init__(self, index: int):
        self.index = index
        self.lib = _lib.lib()
        h = C.c_void_p()
        _lib.check(self.lib.orx_create(index, C.byref(h)), "orx_create")
        self.h = h
        self.device = torch.device("cuda", index)

    def close(self):
        if self.h:
            self.lib.orx_destroy(self.h)
            self.h = None

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    make_table = staticmethod(table)
    make_opt = staticmethod(opt)

    # ---- measurement hook ----
    def profile_enable(self, on=True):
        _lib.check(self.lib.orx_profile_enable(self.h, 1 if on else 0))

    def profile_read(self, n_phases=3):
        """-> ([ms per phase] summed over the recorded steps, n_steps); phases: see orx_profile_enable in orx.h."""
        ms = (C.c_float * n_phases)()
        n = C.c_int32()
        _lib.check(self.lib.orx_profile_read(self.h, ms, n_phases, C.byref(n)))
        return list(ms), n.value

    # ---- LatentFactor ------------------------------------------------------------------
    def fill_uniform(self, dst, lo, hi, seed):
        _lib.check(self.lib.orx_fill_uniform(self.h, _ptr(_f32(dst, "dst")), dst.numel(), lo, hi, seed, self.stream()))

    def gather(self, tab, ids, n_bad=None):
        is64 = ids.dtype == torch.int64
        if not is64:
            ids = ids32(ids)
        ids = ids.contiguous().reshape(-1)
        out = torch.empty((ids.numel(), tab.shape[1]), dtype=torch.float32, device=tab.device)
        _lib.check(self.lib.orx_gather(self.h, _ptr(_f32(tab, "tab")), tab.shape[0], tab.shape[1], _ptr(ids),
                                       1 if is64 else 0, ids.numel(), _ptr(out), _ptr(n_bad), self.stream()))
        return out

    def censor(self, tab, ids, min_norm=0.1):
        ids = ids32(ids)
        _lib.check(self.lib.orx_censor(self.h, _ptr(_f32(tab, "tab")), tab.shape[0], tab.shape[1], _ptr(ids),
                                       ids.numel(), min_norm, self.stream()))

    def censor_shard(self, tab, total_rows, world, rank, ids, n_per_block, block_stride, n_blocks, first=0,
                     min_norm=0.1):
        """censor of a row-sharded table (orx_censor_shard in include/orx.h): tab is this rank's shard (row r of the
        global table at local row r // world of rank r % world; a rank without rows passes its 1-row dummy), ids a flat
        int32 tensor of GLOBAL ids holding n_blocks blocks of n_per_block, block b from element first + b * block_stride.
        This rank censors each row it owns once."""
        if not (ids.is_cuda and ids.dtype == torch.int32 and ids.is_contiguous()):
            raise ValueError("ids: expected a contiguous int32 CUDA tensor")
        if n_per_block * n_blocks and first + (n_blocks - 1) * block_stride + n_per_block > ids.numel():
            raise ValueError("the id blocks run past the end of ids")
        local = shard_rows(total_rows, rank, world)
        if tab.shape[0] < max(local, 1):
            raise ValueError(f"the shard has {tab.shape[0]} rows; rank {rank} of {world} owns {local}")
        _lib.check(self.lib.orx_censor_shard(self.h, _ptr(_f32(tab, "tab")), tab.shape[0], tab.shape[1],
                                             int(total_rows), int(world), int(rank),
                                             C.c_void_p(ids.data_ptr() + 4 * int(first)), int(n_per_block),
                                             int(block_stride), int(n_blocks), min_norm, self.stream()),
                   "orx_censor_shard")

    # ---- pairwise ----------------------------------------------------------------------
    def pairwise_step(self, kind, user, item, bias, uid, pid, nid, o, out4, margin=0.5, c_loss=1.0, c_l2=1.0):
        _lib.check(self.lib.orx_pairwise_step(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                              _ptr(pid), _ptr(nid), uid.numel(), margin, c_loss, c_l2, C.byref(o),
                                              _ptr(out4), self.stream()), "orx_pairwise_step")

    def pairwise_step_host(self, kind, user, item, bias, uid_h, pid_h, nid_h, o, out4_h, margin=0.5, c_loss=1.0,
                           c_l2=1.0):
        """ids / out4 are (pinned) HOST tensors; copies ride the same stream as the kernels."""
        _lib.check(self.lib.orx_pairwise_step_host(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                                   _ptr(uid_h), _ptr(pid_h), _ptr(nid_h), uid_h.numel(), margin,
                                                   c_loss, c_l2, C.byref(o), _ptr(out4_h), self.stream()),
                   "orx_pairwise_step_host")

    def pairwise_step_bf16(self, kind, user, item, bias, uid, pid, nid, o, sr_seed, out4, margin=0.5, c_loss=1.0,
                           c_l2=1.0):
        """pairwise_step on bf16 user / item tables (table_bf16), rounding seeded with sr_seed."""
        _lib.check(self.lib.orx_pairwise_step_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                                   _ptr(pid), _ptr(nid), uid.numel(), margin, c_loss, c_l2, C.byref(o),
                                                   int(sr_seed), _ptr(out4), self.stream()), "orx_pairwise_step_bf16")

    def pairwise_step_host_bf16(self, kind, user, item, bias, uid_h, pid_h, nid_h, o, sr_seed, out4_h, margin=0.5,
                                c_loss=1.0, c_l2=1.0):
        _lib.check(self.lib.orx_pairwise_step_host_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                                        _ptr(uid_h), _ptr(pid_h), _ptr(nid_h), uid_h.numel(), margin,
                                                        c_loss, c_l2, C.byref(o), int(sr_seed), _ptr(out4_h),
                                                        self.stream()), "orx_pairwise_step_host_bf16")

    def pairwise_fwd_bf16(self, kind, user, item, bias, uid, pid, nid, out4, margin=0.5):
        _lib.check(self.lib.orx_pairwise_fwd_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                                  _ptr(pid), _ptr(nid), uid.numel(), margin, _ptr(out4),
                                                  self.stream()), "orx_pairwise_fwd_bf16")

    def pairwise_grad_bf16(self, kind, user, item, bias, uid, pid, nid, margin=0.5, c_loss=1.0, c_l2=1.0, *,
                           d_user=None, d_pos=None, d_neg=None, d_bp=None, d_bn=None, g_out=None):
        _lib.check(self.lib.orx_pairwise_grad_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                                   _ptr(pid), _ptr(nid), uid.numel(), margin, c_loss, c_l2,
                                                   _ptr(d_user), _ptr(d_pos), _ptr(d_neg), _ptr(d_bp), _ptr(d_bn),
                                                   _ptr(g_out), self.stream()), "orx_pairwise_grad_bf16")

    def censor_bf16(self, tab, ids, min_norm=0.1):
        ids = ids32(ids)
        _lib.check(self.lib.orx_censor_bf16(self.h, _ptr(_bf16(tab, "tab")), tab.shape[0], tab.shape[1], _ptr(ids),
                                            ids.numel(), min_norm, self.stream()), "orx_censor_bf16")

    def debug_round_bf16(self, x, row0, dim, table, sr_seed, step):
        """-> bfloat16 tensor: the stochastic rounding of bf16 tables applied to the float32 CUDA tensor x, element i
        taken as (row0 + i // dim, i % dim) of table `table` (0 user, 1 item) at (sr_seed, step)."""
        x = _f32(x, "x")
        out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        _lib.check(self.lib.orx_debug_round_bf16(self.h, _ptr(x), _ptr(out), x.numel(), int(row0), int(dim),
                                                 int(table), int(sr_seed), int(step), self.stream()),
                   "orx_debug_round_bf16")
        return out

    def pairwise_prefetch(self, user, item, uid, pid, nid, opt_kind, ids_ready=False):
        """Pipelining hint: build the batch index of these id tensors on the side stream now (the next pairwise_step
        with these very tensors consumes it).  ids_ready=True: the tensors are already complete (pre-staged batches),
        so the build does not wait for anything queued on the current stream."""
        user, item = as_table(user), as_table(item)
        _lib.check(self.lib.orx_pairwise_prefetch(self.h, C.byref(user), C.byref(item), _ptr(uid), _ptr(pid), _ptr(nid),
                                                  uid.numel(), opt_kind, 1 if ids_ready else 0, self.stream()),
                   "orx_pairwise_prefetch")

    def debug_set_epoch(self, epoch):
        _lib.check(self.lib.orx_debug_set_epoch(self.h, epoch), "orx_debug_set_epoch")

    def debug_dispatch_log(self):
        """-> [Dispatch] launched by this engine's DLRM calls and sparse steps since the last read (oldest first), and
        clears them."""
        rec = (C.c_int32 * (8 * _lib.ORX_DISPATCH_LOG_CAP))()
        n = C.c_int32()
        _lib.check(self.lib.orx_debug_dispatch_log(self.h, rec, _lib.ORX_DISPATCH_LOG_CAP, C.byref(n)),
                   "orx_debug_dispatch_log")
        return [Dispatch(*rec[8 * i:8 * i + 8]) for i in range(n.value)]

    def debug_pair_records(self, index_set, B):
        """-> int32 [B, 4] CUDA tensor: the records {flags, du, dp, dn} a prefetch resolved for index set 1 or 2."""
        rec = torch.empty((B, 4), dtype=torch.int32, device=self.device)
        _lib.check(self.lib.orx_debug_pair_records(self.h, index_set, _ptr(rec), B, self.stream()),
                   "orx_debug_pair_records")
        return rec

    def pairwise_fwd(self, kind, user, item, bias, uid, pid, nid, out4, margin=0.5):
        _lib.check(self.lib.orx_pairwise_fwd(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                             _ptr(pid), _ptr(nid), uid.numel(), margin, _ptr(out4), self.stream()),
                   "orx_pairwise_fwd")

    def pairwise_grad(self, kind, user, item, bias, uid, pid, nid, margin=0.5, c_loss=1.0, c_l2=1.0, *, d_user=None,
                      d_pos=None, d_neg=None, d_bp=None, d_bn=None, g_out=None):
        _lib.check(self.lib.orx_pairwise_grad(self.h, kind, C.byref(user), C.byref(item), C.byref(bias), _ptr(uid),
                                              _ptr(pid), _ptr(nid), uid.numel(), margin, c_loss, c_l2, _ptr(d_user),
                                              _ptr(d_pos), _ptr(d_neg), _ptr(d_bp), _ptr(d_bn), _ptr(g_out),
                                              self.stream()), "orx_pairwise_grad")

    # ---- un-fused sparse apply / multi-GPU building blocks ------------------------------
    def sparse_apply(self, tab, ids, values, o):
        n = 0 if ids is None else ids.numel()
        _lib.check(self.lib.orx_sparse_apply(self.h, C.byref(tab), _ptr(ids), _ptr(values), n, C.byref(o),
                                             self.stream()), "orx_sparse_apply")

    def sparse_apply_strided(self, tab, ids2d, col, values3d, o, sr_seed=None):
        """ids = ids2d[:, col] (int32 [n, F]); value rows = values3d[:, col, :] ([n, F, D]) -- no copies.  A bf16 table
        (table_bf16) takes orx_sparse_apply_strided_bf16, its updates rounded with sr_seed (required)."""
        n, F = ids2d.shape
        D = values3d.shape[2]
        args = (C.c_void_p(ids2d.data_ptr() + 4 * col), F, C.c_void_p(values3d.data_ptr() + 4 * col * D),
                values3d.shape[1] * D, n, C.byref(o))
        if isinstance(tab, OrxTableBf16):
            op = "orx_sparse_apply_strided_bf16"
            _lib.check(self.lib.orx_sparse_apply_strided_bf16(self.h, C.byref(tab), *args, _sr_seed(sr_seed, op),
                                                              self.stream()), op)
        else:
            _lib.check(self.lib.orx_sparse_apply_strided(self.h, C.byref(tab), *args, self.stream()),
                       "orx_sparse_apply_strided")

    # ---- DLRM pieces (2-D operands may be column-slices: the leading dimension is taken from stride(0)) ----
    @staticmethod
    def _ld(t):
        if t.dim() != 2 or t.stride(1) != 1:
            raise ValueError("expected a 2-D float32 view with unit inner stride")
        return t.stride(0)

    def gather_strided(self, tab, ids2d, col, out2d, n_bad=None):
        """out2d[b] = tab[ids2d[b, col]] (float32 rows; a bfloat16 tab takes orx_gather_strided_bf16, widened exactly)."""
        n, F = ids2d.shape
        op = "orx_gather_strided_bf16" if tab.dtype == torch.bfloat16 else "orx_gather_strided"
        if tab.dtype == torch.bfloat16:
            _bf16(tab, "tab")
        _lib.check(getattr(self.lib, op)(self.h, _ptr(tab), tab.shape[0], tab.shape[1],
                                         C.c_void_p(ids2d.data_ptr() + 4 * col), F, n, _ptr(out2d), self._ld(out2d),
                                         _ptr(n_bad), self.stream()), op)

    def bag_gather(self, tabs, sparse, col_off, mode, out2d, n_bad=None):
        """Multi-hot lookup of every table in one launch (orx_bag_gather in include/orx.h): sparse int32 [B, C] on the
        device, col_off [T + 1] host ints (table k's bag = columns col_off[k] .. col_off[k+1]), mode 0 sum / 1 mean;
        out2d [B, >= T*D] (any row stride) gets Z[b, k, :] at columns k*D .. (k+1)*D.  bfloat16 tables take
        orx_bag_gather_bf16 (every table bfloat16; a mix of float32 and bfloat16 tables is refused)."""
        T = len(tabs)
        dtypes = {t.dtype for t in tabs}
        bf16 = torch.bfloat16 in dtypes
        if bf16 and dtypes != {torch.bfloat16}:
            raise ValueError(f"bag_gather: the tables must all be float32 or all bfloat16, got {sorted(map(str, dtypes))}")
        if bf16:
            for k, t in enumerate(tabs):
                _bf16(t, f"tabs[{k}]")
        op = "orx_bag_gather_bf16" if bf16 else "orx_bag_gather"
        if sparse.dtype != torch.int32 or sparse.dim() != 2 or sparse.stride(1) != 1:
            raise ValueError("sparse: expected an int32 [B, C] tensor with unit inner stride")
        if len(col_off) != T + 1:
            raise ValueError("col_off must have T + 1 entries")
        B = sparse.shape[0]
        ptrs = (C.c_void_p * T)(*[t.data_ptr() for t in tabs])
        rows = (C.c_int64 * T)(*[t.shape[0] for t in tabs])
        off = (C.c_int32 * (T + 1))(*[int(x) for x in col_off])
        _lib.check(getattr(self.lib, op)(self.h, ptrs, rows, T, tabs[0].shape[1] if T else 0,
                                         _ptr(sparse) if B else None, max(sparse.stride(0), 1), off, B, int(mode),
                                         _ptr(out2d) if B else None, self._ld(out2d), _ptr(n_bad), self.stream()), op)

    def bag_sparse_apply(self, tab, sparse, col_lo, L, dz2d, mode, o, sr_seed=None):
        """optimizer.apply_gradients of one table's bag lookups (orx_bag_sparse_apply): bag b = sparse[b, col_lo :
        col_lo + L], its pooled gradient row dz2d[b] ([B, D], any row stride), mode 0 sum / 1 mean.  A bf16 table
        (table_bf16) takes orx_bag_sparse_apply_bf16, its updates rounded with sr_seed (required)."""
        B = sparse.shape[0]
        if sparse.dtype != torch.int32 or sparse.dim() != 2 or sparse.stride(1) != 1:
            raise ValueError("sparse: expected an int32 [B, C] tensor with unit inner stride")
        if dz2d.shape[0] != B:
            raise ValueError("one gradient row per bag")
        args = (_ptr(sparse) if B else None, max(sparse.stride(0), 1), int(col_lo), int(L), B,
                _ptr(dz2d) if B else None, self._ld(dz2d), int(mode), C.byref(o))
        if isinstance(tab, OrxTableBf16):
            op = "orx_bag_sparse_apply_bf16"
            _lib.check(self.lib.orx_bag_sparse_apply_bf16(self.h, C.byref(tab), *args, _sr_seed(sr_seed, op),
                                                          self.stream()), op)
        else:
            _lib.check(self.lib.orx_bag_sparse_apply(self.h, C.byref(tab), *args, self.stream()),
                       "orx_bag_sparse_apply")

    def mlp_fwd(self, x, w, bias, act, y):
        _lib.check(self.lib.orx_mlp_layer_fwd(self.h, _ptr(x), self._ld(x), x.shape[0], w.shape[0], _ptr(w), _ptr(bias),
                                              w.shape[1], act, _ptr(y), self._ld(y), self.stream()),
                   "orx_mlp_layer_fwd")

    def mlp_bwd(self, x, y, w, act, dy, dx, dw, db):
        _lib.check(self.lib.orx_mlp_layer_bwd(self.h, _ptr(x), self._ld(x), _ptr(y), self._ld(y), _ptr(w), x.shape[0],
                                              w.shape[0], w.shape[1], act, _ptr(dy), self._ld(dy), _ptr(dx),
                                              self._ld(dx) if dx is not None else 0, _ptr(dw), _ptr(db),
                                              self.stream()), "orx_mlp_layer_bwd")

    def interact_fwd(self, emb3d, dense2d, self_interaction, mode, out2d):
        B, Fm1, D = emb3d.shape
        _lib.check(self.lib.orx_interact_fwd(self.h, _ptr(emb3d), Fm1 * D, _ptr(dense2d), self._ld(dense2d), B,
                                             Fm1 + 1, D, int(self_interaction), mode, _ptr(out2d), self._ld(out2d),
                                             self.stream()), "orx_interact_fwd")

    def interact_bwd(self, emb3d, dense2d, dout2d, self_interaction, mode, demb3d, ddense2d):
        B, Fm1, D = emb3d.shape
        _lib.check(self.lib.orx_interact_bwd(self.h, _ptr(emb3d), Fm1 * D, _ptr(dense2d), self._ld(dense2d),
                                             _ptr(dout2d), self._ld(dout2d), B, Fm1 + 1, D, int(self_interaction),
                                             mode, _ptr(demb3d), Fm1 * D, _ptr(ddense2d), self._ld(ddense2d),
                                             self.stream()), "orx_interact_bwd")

    def cross_fwd(self, x0, xl, y, out):
        """out = x0 * y + xl (orx_cross_fwd): [B, W] views with unit inner stride, any row stride."""
        B, W = x0.shape
        _lib.check(self.lib.orx_cross_fwd(self.h, _ptr(x0), self._ld(x0), _ptr(xl), self._ld(xl), _ptr(y), self._ld(y),
                                          B, W, _ptr(out), self._ld(out), self.stream()), "orx_cross_fwd")

    def cross_bwd(self, mode, G, A, P=None, x0=None, y=None, dy=None, dx_lo=None, dx_hi=None):
        """One backward pass of a cross layer (orx_cross_bwd; the operands each mode reads and writes are in
        include/orx.h).  [B, W] views with unit inner stride; FINAL splits dL/dx0 at dx_lo's width (dx_lo may be None
        for split 0)."""
        B, W = G.shape
        ld = lambda t: self._ld(t) if t is not None else 0
        split = (dx_lo.shape[1] if dx_lo is not None else 0) if mode == ORX_CROSS_FINAL else 0
        _lib.check(self.lib.orx_cross_bwd(self.h, int(mode), B, W, _ptr(G), ld(G), _ptr(P), ld(P), _ptr(x0), ld(x0),
                                          _ptr(y), ld(y), _ptr(A), ld(A), _ptr(dy), ld(dy), split, _ptr(dx_lo),
                                          ld(dx_lo), _ptr(dx_hi), ld(dx_hi), self.stream()), "orx_cross_bwd")

    def pred_loss(self, pred, label, kind, clip, pred_out, dpred, out4):
        _lib.check(self.lib.orx_pred_loss(self.h, _ptr(pred), _ptr(label), pred.numel(), kind, clip, _ptr(pred_out),
                                          _ptr(dpred), _ptr(out4), self.stream()), "orx_pred_loss")

    def owner_bucket_combined(self, ids, n_user, total_users, world):
        """ids = uid | pid | nid -> (counts[world], send_local[n] combined local rows, slot[n])."""
        n = ids.numel()
        counts = torch.empty(world, dtype=torch.int32, device=ids.device)
        send_local = torch.empty(n, dtype=torch.int32, device=ids.device)
        slot = torch.empty(n, dtype=torch.int32, device=ids.device)
        _lib.check(self.lib.orx_owner_bucket_combined(self.h, _ptr(ids), n, n_user, total_users, world, _ptr(counts),
                                                      _ptr(send_local), _ptr(slot), self.stream()),
                   "orx_owner_bucket_combined")
        return counts, send_local, slot

    def lookup_bucket(self, sparse, row_off, world):
        """sparse int32 [B, T] on the device, row_off [T + 1] host ints (the tables' offsets in the concatenated row
        space) -> (counts [world], send_local, slot [B*T], grp_off [B*T + 1], grp_idx [B*T]): the batch's unique valid
        rows in (owner, local row) order and each one's lookups (orx_lookup_bucket in include/orx.h)."""
        if sparse.dtype != torch.int32 or sparse.dim() != 2 or not sparse.is_contiguous():
            raise ValueError("sparse: expected a contiguous int32 [B, T] tensor")
        B, T = sparse.shape
        if len(row_off) != T + 1:
            raise ValueError("row_off must have T + 1 entries")
        dev, n = sparse.device, B * T
        counts = torch.empty(world, dtype=torch.int32, device=dev)
        send_local, slot, grp_idx = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(3))
        grp_off = torch.empty(n + 1, dtype=torch.int32, device=dev)
        off = (C.c_int64 * (T + 1))(*[int(x) for x in row_off])
        _lib.check(self.lib.orx_lookup_bucket(self.h, _ptr(sparse), B, T, off, world, _ptr(counts), _ptr(send_local),
                                              _ptr(slot), _ptr(grp_off), _ptr(grp_idx), self.stream()),
                   "orx_lookup_bucket")
        return counts, send_local, slot, grp_off, grp_idx

    def rows_segment_sum(self, src, grp_off, grp_idx, n_uniq, out=None):
        """src [n, dim] (any row stride) -> out [n_uniq, dim]: row j = the sum of src rows grp_idx[grp_off[j] ..
        grp_off[j+1]), in that order (orx_rows_segment_sum)."""
        n_uniq = int(n_uniq)
        if n_uniq < 0 or n_uniq + 1 > grp_off.numel():
            raise ValueError("n_uniq must lie in [0, grp_off.numel() - 1]")
        if out is None:
            out = torch.empty((n_uniq, src.shape[1]), dtype=torch.float32, device=src.device)
        _lib.check(self.lib.orx_rows_segment_sum(self.h, _ptr(src), self._ld(src), src.shape[1], _ptr(grp_off),
                                                 _ptr(grp_idx), n_uniq, _ptr(out), self.stream()),
                   "orx_rows_segment_sum")
        return out

    def bag_shard_lookups(self, sparse, col_off, row_off):
        """sparse int32 [B, C] on the device (table k's bag = columns col_off[k] .. col_off[k+1]), row_off [T + 1] host
        ints -> int32 [B, C] global rows, -1 for padding and bad ids (orx_bag_shard_lookups in include/orx.h)."""
        if sparse.dtype != torch.int32 or sparse.dim() != 2 or not sparse.is_contiguous():
            raise ValueError("sparse: expected a contiguous int32 [B, C] tensor")
        T = len(col_off) - 1
        if len(row_off) != T + 1 or sparse.shape[1] != col_off[-1]:
            raise ValueError("col_off and row_off need T + 1 entries, and sparse col_off[-1] columns")
        B = sparse.shape[0]
        out = torch.empty_like(sparse)
        co = (C.c_int32 * (T + 1))(*[int(x) for x in col_off])
        ro = (C.c_int64 * (T + 1))(*[int(x) for x in row_off])
        _lib.check(self.lib.orx_bag_shard_lookups(self.h, _ptr(sparse) if B else None, B, T, co, ro,
                                                  _ptr(out) if B else None, self.stream()), "orx_bag_shard_lookups")
        return out

    def bag_segment_sum(self, dz3d, col_off, mode, slot, grp_off, grp_idx, n_uniq, out=None):
        """dz3d [B, T, D] pooled gradient (any batch stride, rows contiguous), the bag layout col_off [T + 1] and the
        bucket of the [B*C, 1] lookups (slot, grp_off, grp_idx, n_uniq) -> out [n_uniq, D]: row j = the sum of its
        lookups' bag gradient rows, each divided by its bag's valid count for a mean (mode 1), in ascending grp_idx
        position (orx_bag_segment_sum)."""
        B, T, D = dz3d.shape
        n_uniq = int(n_uniq)
        if len(col_off) != T + 1 or dz3d.stride(2) != 1 or dz3d.stride(1) != D:
            raise ValueError("col_off needs T + 1 entries, and dz3d contiguous [T, D] rows per sample")
        if n_uniq < 0 or n_uniq + 1 > grp_off.numel():
            raise ValueError("n_uniq must lie in [0, grp_off.numel() - 1]")
        if slot.numel() != B * int(col_off[-1]):
            raise ValueError("slot needs one entry per lookup")
        if out is None:
            out = torch.empty((n_uniq, D), dtype=torch.float32, device=dz3d.device)
        co = (C.c_int32 * (T + 1))(*[int(x) for x in col_off])
        ld = dz3d.stride(0) if B > 1 else T * D
        _lib.check(self.lib.orx_bag_segment_sum(self.h, _ptr(dz3d), ld, T, D, co, int(mode), _ptr(slot), B,
                                                _ptr(grp_off), _ptr(grp_idx), n_uniq, _ptr(out), self.stream()),
                   "orx_bag_segment_sum")
        return out

    def pairwise_grad_rows(self, kind, rows, dim, uslot, pslot, nslot, inv_B, d_rows, out4, margin=0.5, c_loss=1.0,
                           c_l2=1.0):
        _lib.check(self.lib.orx_pairwise_grad_rows(self.h, kind, _ptr(rows), rows.shape[1], dim, _ptr(uslot),
                                                   _ptr(pslot), _ptr(nslot), uslot.numel(), margin, c_loss, c_l2,
                                                   inv_B, _ptr(d_rows), _ptr(out4), self.stream()),
                   "orx_pairwise_grad_rows")

    def sparse_apply_rows(self, tab, ids, values, o):
        """orx_sparse_apply_strided with id i = ids[i] and value row i = values[i] (a 2-D view of any row stride: the
        row-sharded pointwise step applies the bias column of its exchange rows in place)."""
        n = ids.numel()
        if values.shape[0] != n:
            raise ValueError("one value row per id")
        _lib.check(self.lib.orx_sparse_apply_strided(self.h, C.byref(tab), _ptr(ids) if n else None, 1,
                                                     _ptr(values) if n else None, self._ld(values), n, C.byref(o),
                                                     self.stream()), "orx_sparse_apply_strided")

    # ---- row-sharded pointwise step (orx_pointwise_shard.cu) -------------------------------
    def pointwise_shard_lookups(self, uid, iid, total_users, total_items):
        """-> int32 [B, 2] lookups (uid, iid) for orx_lookup_bucket, (-1, -1) for a sample with an id out of range."""
        B = uid.numel()
        if iid.numel() != B:
            raise ValueError("uid and iid must have the same length")
        out = torch.empty((B, 2), dtype=torch.int32, device=uid.device)
        _lib.check(self.lib.orx_pointwise_shard_lookups(self.h, _ptr(uid), _ptr(iid), B, int(total_users),
                                                        int(total_items), _ptr(out), self.stream()),
                   "orx_pointwise_shard_lookups")
        return out

    def pointwise_serve(self, user, item, bias, local_users, local_items, user_rows_per_rank, req, ld):
        """Owner side: -> (rows [n, ld], user_local [n], item_local [n]) for the requested local rows req
        (orx_pointwise_serve in include/orx.h).  user / item / bias are this rank's shards (bias [rows] or [rows, 1])."""
        n = req.numel()
        dev = req.device
        rows = torch.empty((n, ld), dtype=torch.float32, device=dev)
        ul = torch.empty(n, dtype=torch.int32, device=dev)
        il = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(self.lib.orx_pointwise_serve(self.h, _ptr(_f32(user, "user")), _ptr(_f32(item, "item")),
                                                _ptr(_f32(bias, "bias")), user.shape[1], int(local_users),
                                                int(local_items), int(user_rows_per_rank), _ptr(req), n, int(ld),
                                                _ptr(rows), _ptr(ul), _ptr(il), self.stream()), "orx_pointwise_serve")
        return rows, ul, il

    def pointwise_grad_rows(self, kind, rows, dim, slot, label, w, inv_B, a=1.0, b=1.0, use_sigmoid=False,
                            c_loss=1.0, c_l2=1.0, add_w_terms=False):
        """Score, loss and per-lookup gradient rows over fetched rows (orx_pointwise_grad_rows in include/orx.h): rows
        [*, ld] with the bias in column dim, slot int32 [2B] -> (d_rows [2B, ld], gw [dim] (GMF) or None, out2 [2])."""
        B = label.numel()
        if slot.numel() != 2 * B:
            raise ValueError("slot needs two entries (user, item) per sample")
        dev, ld = label.device, rows.shape[1]
        d_rows = torch.empty((2 * B, ld), dtype=torch.float32, device=dev)
        gw = torch.empty(dim, dtype=torch.float32, device=dev) if kind == ORX_POINT_GMF else None
        out2 = torch.empty(2, dtype=torch.float32, device=dev)
        _lib.check(self.lib.orx_pointwise_grad_rows(self.h, kind, _ptr(_f32(rows, "rows")), ld, dim, _ptr(slot),
                                                    _ptr(_f32(label, "label")), _ptr(w), B, a, b, int(use_sigmoid),
                                                    c_loss, c_l2, inv_B, int(add_w_terms), _ptr(d_rows), _ptr(gw),
                                                    _ptr(out2), self.stream()), "orx_pointwise_grad_rows")
        return d_rows, gw, out2

    def rows_scale(self, x, scale):
        """In place: x[r, k] *= scale[k], one rounding (orx_rows_scale).  x: contiguous [rows, dim] float32, or an int32
        tensor holding float bits (the xrows exchange buffer of the shard phases)."""
        dim = scale.numel()
        if not x.is_contiguous() or x.numel() % dim:
            raise ValueError("x must be contiguous with a multiple of scale.numel() elements")
        _lib.check(self.lib.orx_rows_scale(self.h, _ptr(x), x.numel() // dim, dim, _ptr(_f32(scale, "scale")),
                                           self.stream()), "orx_rows_scale")

    # ---- pointwise ---------------------------------------------------------------------
    def pointwise_step(self, kind, user, item, bias, w, uid, iid, label, o, out4, a=1.0, b=1.0, use_sigmoid=False,
                       c_loss=1.0, c_l2=1.0):
        _lib.check(self.lib.orx_pointwise_step(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                               C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                               _ptr(label), uid.numel(), a, b, int(use_sigmoid), c_loss, c_l2,
                                               C.byref(o), _ptr(out4), self.stream()), "orx_pointwise_step")

    def pointwise_fwd(self, kind, user, item, bias, w, uid, iid, label, out4, a=1.0, b=1.0, use_sigmoid=False):
        _lib.check(self.lib.orx_pointwise_fwd(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                              C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                              _ptr(label), uid.numel(), a, b, int(use_sigmoid), _ptr(out4),
                                              self.stream()), "orx_pointwise_fwd")

    def pointwise_grad(self, kind, user, item, bias, w, uid, iid, label, a=1.0, b=1.0, use_sigmoid=False, c_loss=1.0,
                       c_l2=1.0, *, d_user=None, d_item=None, d_bias=None, d_w=None, g_out=None):
        _lib.check(self.lib.orx_pointwise_grad(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                               C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                               _ptr(label), uid.numel(), a, b, int(use_sigmoid), c_loss, c_l2,
                                               _ptr(d_user), _ptr(d_item), _ptr(d_bias), _ptr(d_w), _ptr(g_out),
                                               self.stream()), "orx_pointwise_grad")

    def pointwise_step_bf16(self, kind, user, item, bias, w, uid, iid, label, o, sr_seed, out4, a=1.0, b=1.0,
                            use_sigmoid=False, c_loss=1.0, c_l2=1.0):
        """pointwise_step on bf16 user / item tables (table_bf16), rounding seeded with sr_seed; bias and w fp32."""
        _lib.check(self.lib.orx_pointwise_step_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                                    C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                                    _ptr(label), uid.numel(), a, b, int(use_sigmoid), c_loss, c_l2,
                                                    C.byref(o), int(sr_seed), _ptr(out4), self.stream()),
                   "orx_pointwise_step_bf16")

    def pointwise_fwd_bf16(self, kind, user, item, bias, w, uid, iid, label, out4, a=1.0, b=1.0, use_sigmoid=False):
        _lib.check(self.lib.orx_pointwise_fwd_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                                   C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                                   _ptr(label), uid.numel(), a, b, int(use_sigmoid), _ptr(out4),
                                                   self.stream()), "orx_pointwise_fwd_bf16")

    def pointwise_grad_bf16(self, kind, user, item, bias, w, uid, iid, label, a=1.0, b=1.0, use_sigmoid=False,
                            c_loss=1.0, c_l2=1.0, *, d_user=None, d_item=None, d_bias=None, d_w=None, g_out=None):
        _lib.check(self.lib.orx_pointwise_grad_bf16(self.h, kind, C.byref(user), C.byref(item), C.byref(bias),
                                                    C.byref(w) if w is not None else None, _ptr(uid), _ptr(iid),
                                                    _ptr(label), uid.numel(), a, b, int(use_sigmoid), c_loss, c_l2,
                                                    _ptr(d_user), _ptr(d_item), _ptr(d_bias), _ptr(d_w), _ptr(g_out),
                                                    self.stream()), "orx_pointwise_grad_bf16")

    # ---- dense / inference / metrics -----------------------------------------------------
    def dense_apply(self, var, s0, s1, grad, o):
        _lib.check(self.lib.orx_dense_apply(self.h, _ptr(_f32(var, "var")), _ptr(s0), _ptr(s1),
                                            _ptr(_f32(grad, "grad")), var.numel(), C.byref(o), self.stream()),
                   "orx_dense_apply")

    def score_all(self, kind, user_tab, uid, item_tab, item_bias, scale=None):
        """-> float32 [Bu, I] scores.  user_tab / item_tab both float32 or both bfloat16 (orx_score_all_bf16)."""
        fn, user_tab, item_tab = _score_tables("orx_score_all", user_tab, item_tab)
        uid = ids32(uid)
        out = torch.empty((uid.numel(), item_tab.shape[0]), dtype=torch.float32, device=item_tab.device)
        _lib.check(getattr(self.lib, fn)(self.h, kind, _ptr(user_tab), user_tab.shape[0], _ptr(uid), uid.numel(),
                                         _ptr(scale), _ptr(item_tab), _ptr(item_bias), item_tab.shape[0],
                                         item_tab.shape[1], _ptr(out), self.stream()), fn)
        return out

    def rank_metrics(self, pred, pos, excl, at=(), want=("auc", "ndcg", "recall")):
        pred = _f32(pred.contiguous(), "pred")
        pos = pos.to(torch.uint8).contiguous()
        excl = excl.to(torch.uint8).contiguous()
        R, I = pred.shape
        at_arr = (C.c_int32 * max(len(at), 1))(*[int(k) for k in at])
        auc = torch.empty(R, dtype=torch.float32, device=pred.device) if "auc" in want else None
        ndcg = torch.empty((R, len(at)), dtype=torch.float32, device=pred.device) if "ndcg" in want else None
        rec = torch.empty((R, len(at)), dtype=torch.float32, device=pred.device) if "recall" in want else None
        _lib.check(self.lib.orx_rank_metrics(self.h, _ptr(pred), _ptr(pos), _ptr(excl), R, I, at_arr, len(at),
                                             _ptr(auc), _ptr(ndcg), _ptr(rec), self.stream()), "orx_rank_metrics")
        return auc, ndcg, rec

    def score_rank(self, kind, user_tab, uid, item_tab, item_bias, pos_off, pos_items, excl_off, excl_items, max_pos,
                   at=(), scale=None):
        """score_all + rank_metrics in one pass for the users uid, from CSR lists indexed by user id: positives
        pos_items[pos_off[u]:pos_off[u + 1]] and exclusions likewise (excl_off / excl_items may be None); int64 offsets,
        int32 items, rows sorted and unique.  max_pos bounds every positive row length (a longer row gets NaN outputs).
        user_tab / item_tab both float32 or both bfloat16 (orx_score_rank_bf16).
        -> (auc [Bu], ndcg [Bu, len(at)], recall [Bu, len(at)])."""
        fn, user_tab, item_tab = _score_tables("orx_score_rank", user_tab, item_tab)
        uid = ids32(uid)
        Bu, dev = uid.numel(), item_tab.device
        pos_off, pos_items = _csr(pos_off, pos_items, user_tab.shape[0])
        excl_off, excl_items = _csr(excl_off, excl_items, user_tab.shape[0])
        if pos_off is None:
            raise ValueError("score_rank needs the positives' CSR")
        at_arr = (C.c_int32 * max(len(at), 1))(*[int(k) for k in at])
        auc = torch.empty(Bu, dtype=torch.float32, device=dev)
        ndcg = torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)
        rec = torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)
        _lib.check(getattr(self.lib, fn)(
            self.h, kind, _ptr(user_tab), user_tab.shape[0], _ptr(uid), Bu, _ptr(scale), _ptr(item_tab),
            _ptr(item_bias), item_tab.shape[0], item_tab.shape[1], _ptr(pos_off), _ptr(pos_items), _ptr(excl_off),
            _ptr(excl_items), int(max_pos), at_arr, len(at), _ptr(auc), _ptr(ndcg), _ptr(rec), self.stream()), fn)
        return auc, ndcg, rec

    @staticmethod
    def score_rank_shard_sizes(Bu, dim, max_pos):
        """-> element counts of the exchange buffers (xrows int32, xpred int32, xcnt int64) of score_rank_shard."""
        n3 = (C.c_int64 * 3)()
        _lib.check(_lib.lib().orx_score_rank_shard_sizes(int(Bu), int(dim), int(max_pos), n3),
                   "orx_score_rank_shard_sizes")
        return tuple(n3)

    def score_rank_shard(self, kind, phase, g, user_shard, item_shard, bias_shard, uid, pos_off, pos_items, excl_off,
                         excl_items, max_pos, xrows, xpred, xcnt, at=()):
        """One phase of score_rank over row-sharded tables (orx_score_rank_shard in include/orx.h).  g: RowShard;
        the shards are this rank's rows (bias_shard flat [local_items] or None); uid and the CSR lists are global.  The
        caller sums each exchange buffer over the ranks between phases (openrec_b200.sharded.score_rank_sharded).
        Phase 3 -> (auc [Bu], ndcg [Bu, len(at)], recall [Bu, len(at)]); other phases -> None."""
        uid = ids32(uid)
        Bu, dev = uid.numel(), xrows.device
        pos_off, pos_items = _csr(pos_off, pos_items, g.total_users)
        excl_off, excl_items = _csr(excl_off, excl_items, g.total_users)
        if pos_off is None:
            raise ValueError("score_rank_shard needs the positives' CSR")
        if xrows.dtype != torch.int32 or xpred.dtype != torch.int32 or xcnt.dtype != torch.int64:
            raise ValueError("exchange buffers: xrows / xpred int32, xcnt int64")
        at_arr = (C.c_int32 * max(len(at), 1))(*[int(k) for k in at])
        out = [None] * 3
        if phase == 3:
            out = [torch.empty(Bu, dtype=torch.float32, device=dev),
                   torch.empty((Bu, len(at)), dtype=torch.float32, device=dev),
                   torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)]
        geo = _lib.OrxRowShard(*[int(x) for x in g])
        _lib.check(self.lib.orx_score_rank_shard(
            self.h, kind, int(phase), C.byref(geo), _ptr(_f32(user_shard, "user_shard")),
            _ptr(_f32(item_shard, "item_shard")), _ptr(_f32(bias_shard, "bias_shard")), user_shard.shape[1],
            _ptr(uid), Bu, _ptr(pos_off), _ptr(pos_items), _ptr(excl_off), _ptr(excl_items), int(max_pos), at_arr,
            len(at), _ptr(xrows), _ptr(xpred), _ptr(xcnt), *[_ptr(t) for t in out], self.stream()),
            "orx_score_rank_shard")
        return tuple(out) if phase == 3 else None

    def score_rank_listed(self, kind, user_tab, uid, item_tab, item_bias, pos_off, pos_items, neg_off, neg_items,
                          excl_off, excl_items, max_pos, at=(), scale=None):
        """score_rank with each user ranked against its listed items only (orx_score_rank_listed in include/orx.h):
        positives, listed items (neg_off / neg_items) and exclusions as CSR lists indexed by user id, as in score_rank
        (excl_off / excl_items may be None).  Equals score_all + rank_metrics on the masks pos = P,
        excl = ~(P | L) | E.  user_tab / item_tab both float32 or both bfloat16 (orx_score_rank_listed_bf16).
        -> (auc [Bu], ndcg [Bu, len(at)], recall [Bu, len(at)])."""
        fn, user_tab, item_tab = _score_tables("orx_score_rank_listed", user_tab, item_tab)
        uid = ids32(uid)
        Bu, dev = uid.numel(), item_tab.device
        pos_off, pos_items = _csr(pos_off, pos_items, user_tab.shape[0])
        neg_off, neg_items = _csr(neg_off, neg_items, user_tab.shape[0])
        excl_off, excl_items = _csr(excl_off, excl_items, user_tab.shape[0])
        if pos_off is None or neg_off is None:
            raise ValueError("score_rank_listed needs the positives' and the listed items' CSR")
        at_arr = (C.c_int32 * max(len(at), 1))(*[int(k) for k in at])
        auc = torch.empty(Bu, dtype=torch.float32, device=dev)
        ndcg = torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)
        rec = torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)
        _lib.check(getattr(self.lib, fn)(
            self.h, kind, _ptr(user_tab), user_tab.shape[0], _ptr(uid), Bu, _ptr(scale), _ptr(item_tab),
            _ptr(item_bias), item_tab.shape[0], item_tab.shape[1], _ptr(pos_off), _ptr(pos_items), _ptr(neg_off),
            _ptr(neg_items), _ptr(excl_off), _ptr(excl_items), int(max_pos), at_arr, len(at), _ptr(auc), _ptr(ndcg),
            _ptr(rec), self.stream()), fn)
        return auc, ndcg, rec

    def score_rank_listed_shard(self, kind, phase, g, user_shard, item_shard, bias_shard, uid, pos_off, pos_items,
                                neg_off, neg_items, excl_off, excl_items, max_pos, xrows, xpred, xcnt, at=()):
        """One phase of score_rank_listed over row-sharded tables (orx_score_rank_listed_shard in include/orx.h); the
        shards, exchange buffers and phases are those of score_rank_shard, the listed items' CSR is global.
        Phase 3 -> (auc [Bu], ndcg [Bu, len(at)], recall [Bu, len(at)]); other phases -> None."""
        uid = ids32(uid)
        Bu, dev = uid.numel(), xrows.device
        pos_off, pos_items = _csr(pos_off, pos_items, g.total_users)
        neg_off, neg_items = _csr(neg_off, neg_items, g.total_users)
        excl_off, excl_items = _csr(excl_off, excl_items, g.total_users)
        if pos_off is None or neg_off is None:
            raise ValueError("score_rank_listed_shard needs the positives' and the listed items' CSR")
        if xrows.dtype != torch.int32 or xpred.dtype != torch.int32 or xcnt.dtype != torch.int64:
            raise ValueError("exchange buffers: xrows / xpred int32, xcnt int64")
        at_arr = (C.c_int32 * max(len(at), 1))(*[int(k) for k in at])
        out = [None] * 3
        if phase == 3:
            out = [torch.empty(Bu, dtype=torch.float32, device=dev),
                   torch.empty((Bu, len(at)), dtype=torch.float32, device=dev),
                   torch.empty((Bu, len(at)), dtype=torch.float32, device=dev)]
        geo = _lib.OrxRowShard(*[int(x) for x in g])
        _lib.check(self.lib.orx_score_rank_listed_shard(
            self.h, kind, int(phase), C.byref(geo), _ptr(_f32(user_shard, "user_shard")),
            _ptr(_f32(item_shard, "item_shard")), _ptr(_f32(bias_shard, "bias_shard")), user_shard.shape[1],
            _ptr(uid), Bu, _ptr(pos_off), _ptr(pos_items), _ptr(neg_off), _ptr(neg_items), _ptr(excl_off),
            _ptr(excl_items), int(max_pos), at_arr, len(at), _ptr(xrows), _ptr(xpred), _ptr(xcnt),
            *[_ptr(t) for t in out], self.stream()), "orx_score_rank_listed_shard")
        return tuple(out) if phase == 3 else None

    def score_topk(self, kind, user_tab, uid, item_tab, item_bias, excl_off, excl_items, k, scale=None):
        """The k best eligible items of each user uid in one pass over the item table, without the [Bu, I] score
        matrix: order score descending then item ascending, the user's CSR exclusion row (excl_off / excl_items as in
        score_rank, may be None) and NaN scores left out, slots past the eligible items padded with item -1 and score
        -inf.  -> (items int32 [Bu, k], scores float32 [Bu, k]), scores bit-equal to score_all's (-0.0 may read +0.0).
        user_tab / item_tab both float32 or both bfloat16 (orx_score_topk_bf16)."""
        fn, user_tab, item_tab = _score_tables("orx_score_topk", user_tab, item_tab)
        uid = ids32(uid)
        Bu, dev = uid.numel(), item_tab.device
        excl_off, excl_items = _csr(excl_off, excl_items, user_tab.shape[0])
        k = int(k)
        if not 1 <= k <= _lib.ORX_MAX_TOPK:
            raise ValueError(f"k must lie in [1, {_lib.ORX_MAX_TOPK}]")
        items = torch.empty((Bu, k), dtype=torch.int32, device=dev)
        scores = torch.empty((Bu, k), dtype=torch.float32, device=dev)
        _lib.check(getattr(self.lib, fn)(
            self.h, kind, _ptr(user_tab), user_tab.shape[0], _ptr(uid), Bu, _ptr(scale), _ptr(item_tab),
            _ptr(item_bias), item_tab.shape[0], item_tab.shape[1], _ptr(excl_off), _ptr(excl_items), k, _ptr(items),
            _ptr(scores), self.stream()), fn)
        return items, scores

    def score_topk_shard(self, kind, phase, g, user_shard, item_shard, bias_shard, uid, excl_off, excl_items, k, xrows,
                         xkeys):
        """One phase of score_topk over row-sharded tables (orx_score_topk_shard in include/orx.h).  g: RowShard; the
        shards are this rank's rows (bias_shard flat [local_items] or None); uid and the exclusion CSR are global.
        Exchange buffers: xrows int32 [Bu * dim], xkeys int64 [Bu * world * k], summed over the ranks by the caller
        between phases (openrec_b200.sharded.score_topk_sharded).  Phase 2 -> (items int32 [Bu, k], scores float32
        [Bu, k]); other phases -> None."""
        uid = ids32(uid)
        Bu, dev = uid.numel(), xrows.device
        excl_off, excl_items = _csr(excl_off, excl_items, g.total_users)
        k = int(k)
        if not 1 <= k <= _lib.ORX_MAX_TOPK:
            raise ValueError(f"k must lie in [1, {_lib.ORX_MAX_TOPK}]")
        if xrows.dtype != torch.int32 or xkeys.dtype != torch.int64:
            raise ValueError("exchange buffers: xrows int32, xkeys int64")
        out = [None, None]
        if phase == 2:
            out = [torch.empty((Bu, k), dtype=torch.int32, device=dev),
                   torch.empty((Bu, k), dtype=torch.float32, device=dev)]
        geo = _lib.OrxRowShard(*[int(x) for x in g])
        _lib.check(self.lib.orx_score_topk_shard(
            self.h, kind, int(phase), C.byref(geo), _ptr(_f32(user_shard, "user_shard")),
            _ptr(_f32(item_shard, "item_shard")), _ptr(_f32(bias_shard, "bias_shard")), user_shard.shape[1],
            _ptr(uid), Bu, _ptr(excl_off), _ptr(excl_items), k, _ptr(xrows), _ptr(xkeys), *[_ptr(t) for t in out],
            self.stream()), "orx_score_topk_shard")
        return tuple(out) if phase == 2 else None


def engine(device=None) -> Engine:
    """The per-device engine; raises (no CPU fallback) when CUDA is unavailable."""
    if not torch.cuda.is_available():
        raise RuntimeError("openrec_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    idx = torch.cuda.current_device() if device is None else torch.device(device).index or 0
    e = _engines.get(idx)
    if e is None:
        e = _engines[idx] = Engine(idx)
    return e
