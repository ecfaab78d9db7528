"""Row-sharded BPR / UCML step across the GPUs of one NVSwitch box (SURVEY 8e, BASELINE configs[4]).

The reference is single-device; this is the scale-out of the same synchronous step:
row r of every table lives on rank ``r % R`` at local row ``r // R`` (optimizer slots alongside);
each rank owns B triplets of the global batch.  One step =

  1. orx_owner_bucket_combined: sort this rank's 3B lookups by owner                   (liborx)
  2. all-to-all            : lookup counts, then combined local-row ids, to the owners (NCCL over NVLink)
  3. orx_gather            : owners read the requested rows from their shard          (liborx)
  4. all-to-all            : rows back to the requesters
  5. orx_pairwise_grad_rows: score, loss and per-lookup gradient rows
                             (pre-step values everywhere: nothing has been written yet)
  6. all-to-all            : gradient rows to the owners
  7. orx_sparse_apply      : owners sum duplicates (across ALL ranks' lookups) and apply the
                             optimizer once per unique row                             (liborx)
  8. all-reduce            : (loss, l2_loss), only when the caller asks for the global value

``torch.distributed`` is plumbing (one process per GPU, NCCL; gloo in the CPU logic tests); every
arithmetic op is a liborx kernel reached through ``eng``.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import time
from collections import namedtuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .native import shard_rows


def _a2a(out, inp, out_splits, in_splits):
    dist.all_to_all_single(out, inp, output_split_sizes=out_splits, input_split_sizes=in_splits)


def take_shard(global_rows, rank, world):
    """Rows rank, rank + world, ... of a global table (numpy or torch, host or device): the shard_rows(total, rank,
    world) rows `rank` owns in the row-sharded layout, as a float32 tensor where the input lives."""
    if isinstance(global_rows, torch.Tensor):
        return global_rows[rank::world].to(torch.float32)
    return torch.as_tensor(np.ascontiguousarray(np.asarray(global_rows)[rank::world]), dtype=torch.float32)


def gather_shards(t, total, world, group=None):
    """The global [total, cols] table on every rank from each rank's local rows t ([shard_rows(total, rank, world),
    cols]), a collective call over ``group`` (test and checkpoint helper; sizes must be small)."""
    per = (total + world - 1) // world
    pad = torch.zeros(per, t.shape[1], dtype=t.dtype, device=t.device)
    pad[:t.shape[0]] = t
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.stack(parts, 1).reshape(per * world, t.shape[1])[:total]     # row = local * world + rank


class ShardedPairwise:
    """BPR (kind 0) / UCML (kind 1) with row-sharded tables.  ``eng`` is a native.Engine (or the
    oracle-backed stand-in of tests/fake_engine.py on CPU).

    Local storage is ONE combined table ``[user rows | item rows, D+4]`` per rank (item bias in column D, three
    padding columns keep rows 16-byte aligned), with optimizer slots of the same shape: a lookup is then just
    (owner, combined local row), and a step needs four collectives -- counts, ids, rows, gradient rows."""

    PAD = 4

    def __init__(self, eng, rank, world, total_users, total_items, dim, *, kind=0, opt_kind=1, lr=0.05, eps=1e-7,
                 beta1=0.9, beta2=0.999, margin=0.5, seed=0, init=True):
        self.eng, self.rank, self.world = eng, rank, world
        self.U, self.I, self.D = total_users, total_items, dim
        self.W = dim + self.PAD
        self.kind, self.opt_kind, self.lr, self.eps, self.b1, self.b2, self.margin = kind, opt_kind, lr, eps, beta1, beta2, margin
        self.iterations = 0
        dev = eng.device
        self.ru, self.ri = shard_rows(total_users, rank, world), shard_rows(total_items, rank, world)
        self.table = torch.zeros(self.ru + self.ri, self.W, dtype=torch.float32, device=dev)
        if init:
            tmp = torch.empty(self.ru + self.ri, dim + 1, dtype=torch.float32, device=dev)
            eng.fill_uniform(tmp, -0.05, 0.05, seed * 1000003 + rank * 17)
            self.table[:, :dim + 1] = tmp
            self.table[:self.ru, dim] = 0.0                      # users have no bias column
            del tmp
        n_slots = {0: 0, 1: 1, 2: 2, 3: 2, 6: 1, 8: 1}[opt_kind]     # 6 / 8: momentum, beta1 = its coefficient
        fill = 0.1 if opt_kind == 1 else 0.0
        self.slots = [torch.full_like(self.table, fill) for _ in range(n_slots)] + [None] * (2 - n_slots)
        self.launches_per_step = 3 + 1 + 2 + 3   # bucket(3) gather(1) grad+reduce(2) sparse_apply(3)
        self._loss_local = None

    def step(self, uid, pid, nid, c_loss=1.0, c_l2=1.0, reduce_loss=True):
        """uid/pid/nid: this rank's int32 GLOBAL ids on the device.  Returns a [2] device tensor: the global
        (loss, l2_loss) when ``reduce_loss`` (one extra all-reduce), else this rank's partial sums."""
        eng, R, D, W = self.eng, self.world, self.D, self.W
        B = uid.numel()
        dev = uid.device
        self.iterations += 1
        ids = torch.cat([uid, pid, nid])
        counts, send_local, slot = eng.owner_bucket_combined(ids, B, self.U, R)
        rcounts = torch.empty_like(counts)
        dist.all_to_all_single(rcounts, counts)
        host = torch.stack([counts, rcounts]).cpu()                    # the step's one host sync
        sc, rc = host[0].tolist(), host[1].tolist()
        req = torch.empty(sum(rc), dtype=torch.int32, device=dev)
        _a2a(req, send_local, rc, sc)
        rows = eng.gather(self.table, req)                             # owners read their shard
        got = torch.empty(3 * B, W, dtype=torch.float32, device=dev)
        _a2a(got, rows, sc, rc)
        out4 = torch.zeros(4, dtype=torch.float32, device=dev)
        d_got = torch.empty_like(got)
        eng.pairwise_grad_rows(self.kind, got, D, slot[:B], slot[B:2 * B], slot[2 * B:], 1.0 / (B * R), d_got, out4,
                               self.margin, c_loss, c_l2)
        g_rows = torch.empty_like(rows)
        _a2a(g_rows, d_got, rc, sc)
        o = eng.make_opt(self.opt_kind, self.lr, self.eps, self.b1, self.b2, self.iterations)
        eng.sparse_apply(eng.make_table(self.table, *self.slots), req, g_rows, o)   # dedup across ALL ranks' lookups
        out = out4[:2].clone()
        if reduce_loss:
            dist.all_reduce(out)
        return out

    # ---- helpers for tests: assemble / scatter the global tables
    def load_global(self, user, item, bias):
        r, R, D = self.rank, self.world, self.D
        self.table[:self.ru, :D] = take_shard(user, r, R)
        self.table[self.ru:, :D] = take_shard(item, r, R)
        self.table[self.ru:, D] = take_shard(bias, r, R).reshape(-1)

    def gather_global(self):
        """-> (user, item, bias) full tables on every rank (test helper; sizes must be small)."""
        D = self.D
        return [gather_shards(t, total, self.world) for t, total in
                ((self.table[:self.ru, :D], self.U), (self.table[self.ru:, :D], self.I),
                 (self.table[self.ru:, D:D + 1], self.I))]


def _scale_rows(parts, scale, bufs):
    """GMF: each part's summed xrows (bufs[k][0], float bits) times its w replica scale[k], in place (orx_rows_scale:
    the rounding of u * w in orx_score_rank / orx_score_topk)."""
    if scale is None:
        return
    for (eng, *_), sc, b in zip(parts, scale, bufs):
        if sc is not None:
            eng.rows_scale(b[0], sc.reshape(-1))


def _rank_phases(parts, reduce, Bu, max_pos, scale, phase_call):
    """The four phases of a sharded evaluation (orx_score_rank_shard / orx_score_rank_listed_shard) with ``reduce``
    between them; phase_call(part, phase, bufs) runs one phase on one part.  -> the phase-3 outputs per part."""
    bufs = []
    for eng, kind, user, item, bias, g in parts:
        n3 = eng.score_rank_shard_sizes(Bu, user.shape[1], max_pos)
        dev = item.device
        bufs.append((torch.empty(n3[0], dtype=torch.int32, device=dev), torch.empty(n3[1], dtype=torch.int32, device=dev),
                     torch.empty(n3[2], dtype=torch.int64, device=dev)))
    outs = [None] * len(parts)
    for phase in range(4):   # every part's phase k is issued before any part's phase k + 1
        for k, (part, b) in enumerate(zip(parts, bufs)):
            outs[k] = phase_call(part, phase, b)
        if phase < 3:
            reduce([b[phase] for b in bufs])
        if phase == 0:
            _scale_rows(parts, scale, bufs)
    return outs


def score_rank_sharded(parts, reduce, uid, pos_off, pos_items, excl_off, excl_items, max_pos, at=(), scale=None):
    """Catalogue evaluation (AUC / NDCG / Recall, as native.Engine.score_rank on the global tables) of row-sharded
    tables, each rank counting over its own item rows: the four phases of orx_score_rank_shard, with ``reduce`` between
    them.  parts[k] = (eng, kind, user_shard, item_shard, bias_shard or None, g) for each rank this process drives
    (g: native.RowShard); uid (global user ids) and the global CSR lists live on every part's device.
    ``reduce(tensors)`` replaces each tensor (one per part) in place by its element-wise integer sum over ALL ranks:
    all_reduce_sum(group) when each process is one rank, loopback_sum for virtual ranks on one device.
    ``scale`` (GMF): one [dim] tensor (or None) per part, the score_rank ``scale`` of the global call; the summed user
    rows are scaled after phase 0's reduce.
    -> [(auc, ndcg, recall)] per part, identical on every rank."""
    def phase_call(part, phase, b):
        eng, kind, user, item, bias, g = part
        return eng.score_rank_shard(kind, phase, g, user, item, bias, uid, pos_off, pos_items, excl_off, excl_items,
                                    max_pos, *b, at=at)
    return _rank_phases(parts, reduce, uid.numel(), max_pos, scale, phase_call)


def score_rank_listed_sharded(parts, reduce, uid, pos_off, pos_items, neg_off, neg_items, excl_off, excl_items,
                              max_pos, at=(), scale=None):
    """Listed-candidate evaluation (as native.Engine.score_rank_listed on the global tables: each user ranked against
    its listed items neg_off / neg_items only) of row-sharded tables: the four phases of orx_score_rank_listed_shard.
    ``parts``, ``reduce``, uid, the global CSR lists and ``scale`` are as in score_rank_sharded.
    -> [(auc, ndcg, recall)] per part, identical on every rank."""
    def phase_call(part, phase, b):
        eng, kind, user, item, bias, g = part
        return eng.score_rank_listed_shard(kind, phase, g, user, item, bias, uid, pos_off, pos_items, neg_off,
                                           neg_items, excl_off, excl_items, max_pos, *b, at=at)
    return _rank_phases(parts, reduce, uid.numel(), max_pos, scale, phase_call)


def score_topk_sharded(parts, reduce, uid, excl_off, excl_items, k, scale=None):
    """Top-K retrieval (the k best unseen items of each user uid, as native.Engine.score_topk on the global tables) of
    row-sharded tables, each rank keeping the k best of its own item rows: the three phases of orx_score_topk_shard,
    with ``reduce`` between them.  ``parts``, ``reduce``, uid, the global exclusion CSR and ``scale`` are as in
    score_rank_sharded.  -> [(items int32 [Bu, k], scores float32 [Bu, k])] per part, identical on every rank."""
    Bu, k = uid.numel(), int(k)
    bufs = [(torch.empty(Bu * user.shape[1], dtype=torch.int32, device=item.device),
             torch.empty(Bu * g.world * k, dtype=torch.int64, device=item.device))
            for _, _, user, item, _, g in parts]
    outs = [None] * len(parts)
    for phase in range(3):   # every part's phase p is issued before any part's phase p + 1
        for j, ((eng, kind, user, item, bias, g), b) in enumerate(zip(parts, bufs)):
            outs[j] = eng.score_topk_shard(kind, phase, g, user, item, bias, uid, excl_off, excl_items, k, *b)
        if phase < 2:
            reduce([b[phase] for b in bufs])
        if phase == 0:
            _scale_rows(parts, scale, bufs)
    return outs


def all_reduce_sum(group=None):
    """reduce for score_rank_sharded / score_topk_sharded with one rank per process: an all-reduce (SUM) on torch's
    current stream."""
    def reduce(tensors):
        for t in tensors:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return reduce


def loopback_sum(tensors):
    """reduce for score_rank_sharded / score_topk_sharded with every rank in this process (virtual ranks on one
    device)."""
    total = tensors[0].clone()
    for t in tensors[1:]:
        total += t
    for t in tensors:
        t.copy_(total)


# ---------------------------------------------------------------------------------------
# UCML.censor_vec on row-sharded tables
# ---------------------------------------------------------------------------------------
def censor_gathered(eng, user, item, total_users, total_items, world, rank, ids, B, min_norm=0.1):
    """The three censors of UCML.censor_vec (ucml.py:44-48) on one rank's shards, from the all-gathered ids: ids is the
    flat [world][3][B] int32 block of every rank's (u, p, n).  The user table is censored over every rank's u, then the
    item table over every p, then over every n (orx_censor_shard, on eng's stream).  user / item: this rank's shards."""
    for c, (tab, total) in enumerate(((user, total_users), (item, total_items), (item, total_items))):
        eng.censor_shard(tab, total, world, rank, ids, B, 3 * B, world, first=c * B, min_norm=min_norm)


def censor_vec_sharded(eng, user, item, total_users, total_items, world, rank, uid, pid, nid, group=None,
                       min_norm=0.1):
    """UCML.censor_vec of row-sharded tables (row r on rank r % world at local row r // world), a COLLECTIVE call: every
    rank passes its part (uid, pid, nid) of the global batch, int32 GLOBAL ids on the device, and afterwards the shards
    of all ranks together equal the single-device censor_vec on the concatenation of every rank's ids, bit for bit.
    Each of the three censors deduplicates over the global ids of that call; an item row in both p and n is censored
    twice, p first; ids out of range are skipped.

    This rank packs its ids as [3][B], one all-gather (group, torch's current stream) gives every rank the [world][3][B]
    block, and each rank censors the rows it owns (censor_gathered): 12 B bytes in, 12 world B bytes out, no host sync.
    Every rank must pass the same B, as in the step; this is not checked (a mismatch leaves the collective hanging)."""
    B = uid.numel()
    if pid.numel() != B or nid.numel() != B:
        raise ValueError("uid, pid and nid must have the same length")
    if B == 0:
        return
    packed = torch.stack([uid.reshape(-1), pid.reshape(-1), nid.reshape(-1)]).to(torch.int32).reshape(-1)
    if world == 1:
        ids = packed
    else:
        ids = torch.empty(world * 3 * B, dtype=torch.int32, device=packed.device)
        dist.all_gather_into_tensor(ids, packed, group=group)    # flat [world * 3B]: gloo takes no [world, 3, B] output
    censor_gathered(eng, user, item, total_users, total_items, world, rank, ids, B, min_norm)


# ---------------------------------------------------------------------------------------
# row-sharded DLRM: embedding rows on their owners, Dense layers replicated
# ---------------------------------------------------------------------------------------
def row_offsets(vocab):
    """[T + 1] offsets of T tables of the given vocabularies in one concatenated row space; ValueError when the space
    exceeds 2^31 - 1 rows (global rows are int32)."""
    off = [0]
    for v in vocab:
        if int(v) < 0:
            raise ValueError("a vocabulary size is negative")
        off.append(off[-1] + int(v))
    if off[-1] > 2 ** 31 - 1:
        raise ValueError(f"the {len(vocab)} tables hold {off[-1]} rows in all; the sharded layout allows 2^31 - 1")
    return off


class DistExchange:
    """The collectives of the sharded DLRM step with one rank per process (torch.distributed: NCCL, or gloo on CPU).
    Every method takes lists with one entry, this rank's."""

    def __init__(self, group=None):
        self.group = group

    def all_to_all(self, outs, ins, out_splits, in_splits):
        for o, i, os_, is_ in zip(outs, ins, out_splits, in_splits):
            dist.all_to_all_single(o, i, output_split_sizes=os_, input_split_sizes=is_, group=self.group)

    def all_reduce(self, tensors):
        for t in tensors:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)


class LoopbackExchange:
    """The same collectives for R virtual ranks in this process (one entry per rank, all on one device): the 1-GPU
    test of the multi-GPU code path, same kernels.  The sum adds the ranks in rank order and hands every rank the same
    tensor, as an all-reduce does."""

    @staticmethod
    def all_to_all(outs, ins, out_splits, in_splits):
        R = len(ins)
        ioff = [np.concatenate([[0], np.cumsum(s)]).astype(np.int64) for s in in_splits]
        ooff = [np.concatenate([[0], np.cumsum(s)]).astype(np.int64) for s in out_splits]
        for q in range(R):
            for r in range(R):
                n = int(in_splits[q][r])
                if n != int(out_splits[r][q]):
                    raise ValueError("all_to_all: send and receive splits disagree")
                if n:
                    outs[r][ooff[r][q]:ooff[r][q] + n].copy_(ins[q][ioff[q][r]:ioff[q][r] + n])

    all_reduce = staticmethod(loopback_sum)


class DLRMShard:
    """One rank's part of a row-sharded DLRM.  The T tables are one row space (row_offsets); global row g lives on rank
    g % world at local row g // world of ``table`` ([max(rows, 1), dim]: a rank without rows keeps a 1-row dummy that
    is never read), with its optimizer slots ``slots`` (s0, s1, None when the optimizer has fewer).  ``bot`` / ``top``
    are this rank's Dense replicas as (kernel, bias or None, act) triples, ``dense_slots`` the (s0, s1) of every kernel
    and bias in that order (biases that are None skipped).  ``col_off`` ([T + 1], table k's bag = sparse columns
    col_off[k] .. col_off[k+1]) makes every feature multi-hot, pooled by a sum (``pooling`` 0) or a mean (1); None: one
    id per table.  ``cross``: the replicas of a DCN-v2 cross network in DLRMGraph's form (per layer [(kernel, bias or
    None)]), which replaces the dot interaction; their (s0, s1) follow the top MLP's in ``dense_slots``."""

    def __init__(self, eng, rank, world, vocab, dim, bot, top, table, slots, dense_slots, *, self_interaction=False,
                 mode="reference", loss_kind=0, clip=0.0, col_off=None, pooling=0, cross=None):
        from .tf2.mlp_ops import DLRMGraph
        self.eng, self.rank, self.world, self.D = eng, rank, world, int(dim)
        self.row_off = row_offsets(vocab)
        self.T, self.G = len(vocab), self.row_off[-1]
        if col_off is not None and len(col_off) != self.T + 1:
            raise ValueError("col_off needs T + 1 entries")
        self.col_off, self.pooling = (None, 0) if col_off is None else ([int(c) for c in col_off], int(pooling))
        self.C = self.T if col_off is None else self.col_off[-1]      # sparse columns per sample
        self.rows = shard_rows(self.G, rank, world)
        if tuple(table.shape) != (max(self.rows, 1), self.D):
            raise ValueError(f"shard shape {tuple(table.shape)} != {(max(self.rows, 1), self.D)}")
        self.table, self.slots = table, tuple(slots)
        self.bot, self.top, self.cross, self.dense_slots = bot, top, cross, list(dense_slots)
        if len(self.dense_slots) != len(self.dense_vars()):
            raise ValueError("dense_slots needs one (s0, s1) pair per Dense kernel and bias")
        self.graph = DLRMGraph([None] * self.T, bot, top, self.D, self_interaction, mode, loss_kind, clip, cross=cross)
        self.last = {}          # sizes of the last step: unique rows fetched, rows served to the other ranks

    def dense_vars(self):
        """The Dense kernels and biases, then the cross network's, in the order of dense_slots."""
        mlp = [t for w, b, _ in self.bot + self.top for t in (w, b) if t is not None]
        return mlp + [t for p in self.cross or [] for w, b in p for t in (w, b) if t is not None]

    # ---- global <-> shard (tests, checkpoints)
    def load_global(self, table):
        """table: the concatenated [G, D] tables (host or device); keeps this rank's rows."""
        self.table[:self.rows] = take_shard(table, self.rank, self.world)


# ---- the deduplicated row exchange of the sharded DLRM and GMF / WRMF steps
_Fetched = namedtuple("_Fetched", "bucket send recv req served got")


def _untimed(name):
    pass


def _bucket(part, lookups):
    return part.eng.lookup_bucket(lookups, part.row_off, part.world)


def _fold(part, d_rows, f):
    return part.eng.rows_segment_sum(d_rows, f.bucket[3], f.bucket[4], sum(f.send))


def _fetch_rows(parts, xchg, lookups, serve, width, equal_batches, timer=None, bucket=_bucket):
    """Fetch every part's unique rows from their owners.  parts[k] has .eng, .world and .row_off; lookups[k] is its
    int32 [B, T] lookups (B is the batch size that equal_batches compares); serve(part, req) is the owner's reply to
    the requested local rows req: the rows [len(req), width] first, then whatever the caller keeps.  bucket(part,
    lookups) is the part's orx_lookup_bucket call (default: over the part's row_off).  Runs the bucket, the (count, B)
    exchange with the step's one host sync (and, with equal_batches, the check that every rank passed the same B), the
    ids exchange, serve and the rows exchange.  -> per part a _Fetched: the lookup_bucket tuple, the send / receive
    counts per rank, req, serve's result and got [max(n, 1), width], whose first n = sum(send) rows are the unique rows
    in bucket order (never empty: orx_pointwise_grad_rows needs a rows pointer)."""
    timer = timer or _untimed
    R = parts[0].world
    n = len(parts)
    bk = [bucket(p, lk) for p, lk in zip(parts, lookups)]
    timer("bucket")
    send = [torch.stack([b[0], torch.full_like(b[0], lk.shape[0])], 1) for b, lk in zip(bk, lookups)]   # (count, B)
    recv = [torch.empty_like(x) for x in send]
    xchg.all_to_all(recv, send, [[1] * R] * n, [[1] * R] * n)
    host = torch.stack([torch.stack(send), torch.stack(recv)]).cpu()          # the step's one host sync
    sc = [host[0, k, :, 0].tolist() for k in range(n)]
    rc = [host[1, k, :, 0].tolist() for k in range(n)]
    if equal_batches and any(set(host[1, k, :, 1].tolist()) != {lookups[k].shape[0]} for k in range(n)):
        raise ValueError("every rank must pass the same local batch size to a sharded step "
                         f"(got {sorted(set(host[1, :, :, 1].reshape(-1).tolist()))})")
    timer("counts")
    dev = [lk.device for lk in lookups]
    req = [torch.empty(sum(r), dtype=torch.int32, device=d) for r, d in zip(rc, dev)]
    xchg.all_to_all(req, [b[1][:sum(s)] for b, s in zip(bk, sc)], rc, sc)
    timer("ids")
    served = [serve(p, q) for p, q in zip(parts, req)]
    timer("owner_serve")
    got = [torch.empty(max(sum(s), 1), width, dtype=torch.float32, device=d) for s, d in zip(sc, dev)]
    xchg.all_to_all([g[:sum(s)] for g, s in zip(got, sc)], [x[0] for x in served], sc, rc)
    timer("rows")
    return [_Fetched(*f) for f in zip(bk, sc, rc, req, served, got)]


def _return_grads(parts, xchg, fetched, d_rows, timer=None, fold=_fold):
    """Send the gradients of fetched rows back to their owners: fold(part, d_rows[k], fetched[k]) folds parts[k]'s
    gradients onto its unique rows in a fixed order (default: d_rows[k] holds the per-lookup gradient rows, row i for
    lookup i, summed by orx_rows_segment_sum), and one exchange takes those to the owners.  Sets each part's .last.
    -> per part the gradient rows [len(req), width] of the rows it served, in req's order."""
    timer = timer or _untimed
    g_uniq = [fold(p, d, f) for p, d, f in zip(parts, d_rows, fetched)]
    timer("segment_sum")
    g_rows = [torch.empty(sum(f.recv), g.shape[1], dtype=torch.float32, device=g.device)
              for f, g in zip(fetched, g_uniq)]
    xchg.all_to_all(g_rows, g_uniq, [f.recv for f in fetched], [f.send for f in fetched])
    timer("grad_xchg")
    for p, f in zip(parts, fetched):
        p.last = {"uniq": sum(f.send), "served": sum(f.recv)}
    return g_rows


def _bag_bucket(part, rows):
    return part.eng.lookup_bucket(rows.view(-1, 1), [0, part.G], part.world)


def _bag_fold(part, dZ, f):
    return part.eng.bag_segment_sum(dZ, part.col_off, part.pooling, f.bucket[2], f.bucket[3], f.bucket[4], sum(f.send))


def _dlrm_fetch(parts, xchg, sparses, equal_batches, timer=None):
    """The row fetch of the sharded DLRM step and inference: _fetch_rows with the owners gathering the requested rows
    of their shard, then Z = the fetched rows of every lookup, pooled per bag for a multi-hot model.  -> (Z [B, T, D]
    per part, the _Fetched per part).

    Multi-hot: orx_bag_shard_lookups maps the [B, C] bags to global rows (-1 for padding and bad ids), bucketed as
    [B*C, 1] lookups of one row space; orx_bag_gather then pools the fetched rows with slot as the bag ids, skipping
    slot -1, in column order -- the single-GPU pooling of bit copies of the same rows, so the same Z bit for bit."""
    serve = lambda p, req: (p.eng.gather(p.table, req),)
    if parts[0].col_off is None:
        fetched = _fetch_rows(parts, xchg, sparses, serve, parts[0].D, equal_batches, timer)
    else:
        rows = [p.eng.bag_shard_lookups(s, p.col_off, p.row_off) for p, s in zip(parts, sparses)]
        fetched = _fetch_rows(parts, xchg, rows, serve, parts[0].D, equal_batches, timer, bucket=_bag_bucket)
    Zs = []
    for p, f, s in zip(parts, fetched, sparses):
        B = s.shape[0]
        if p.col_off is not None:
            Z = torch.empty(B, p.T, p.D, dtype=torch.float32, device=s.device)
            p.eng.bag_gather([f.got] * p.T, f.bucket[2].view(B, p.C), p.col_off, p.pooling, Z.view(B, p.T * p.D))
            Zs.append(Z)
        elif sum(f.send):
            Zs.append(p.eng.gather(f.got, f.bucket[2]).view(B, p.T, p.D))     # slot -1 (a bad id) -> the zero row
        else:
            Zs.append(torch.zeros(B, p.T, p.D, dtype=torch.float32, device=s.device))
    return Zs, fetched


def dlrm_step_sharded(parts, xchg, batches, opt_args, c_loss=1.0, timer=None):
    """One synchronous training step of a row-sharded DLRM on the global batch (the union of every rank's batch; every
    rank passes the same local batch size).  parts: the DLRMShard of each rank this process drives; xchg: DistExchange
    or LoopbackExchange; batches[k] = (dense [B, n_dense] f32, sparse [B, T] int32 -- [B, C] bags for a multi-hot
    model --, label [B] f32) of parts[k];
    opt_args = (kind, lr, eps, beta1, beta2, step).  ``timer(name)``, when given, is called after each phase (the
    benchmark's per-phase split).  -> per part a [4] device tensor whose [0] is the GLOBAL loss, identical on every rank.

    The embedding rows of the batch are deduplicated before they travel (orx_lookup_bucket), the per-lookup gradient
    rows are folded onto those unique rows in a fixed order (orx_rows_segment_sum; orx_bag_segment_sum reads a
    multi-hot model's pooled gradient rows directly, divided by the bag's valid count for a mean) and each owner's
    orx_sparse_apply dedups across all ranks' requests -- Keras' sparse apply on the global batch.  The Dense gradients
    and the loss travel in one all-reduce; every replica then applies the same summed gradient."""
    timer = timer or _untimed
    R = parts[0].world
    for p, (dense, sparse, _) in zip(parts, batches):
        if sparse.dim() != 2 or sparse.shape[1] != p.C:
            raise ValueError(f"sparse features must be [B, {p.C}]")
        if sparse.shape[0] < 1 or dense.shape[0] != sparse.shape[0]:
            raise ValueError("the sharded DLRM step needs B >= 1 samples, with as many dense rows as sparse rows")
    Zs, fetched = _dlrm_fetch(parts, xchg, [b[1] for b in batches], True, timer)
    caches, grads = [], []
    for p, (dense, sparse, label), Z in zip(parts, batches, Zs):
        c = p.graph.forward(dense, sparse, label, want_grad=True, Z=Z)
        c["dpred"].mul_(c_loss / R)                         # Keras' MSE / BCE: a mean over the GLOBAL batch
        caches.append(c)
        grads.append(p.graph.backward(c))
    timer("fwd_bwd")
    if parts[0].col_off is None:
        g_rows = _return_grads(parts, xchg, fetched, [g[0].view(-1, p.D) for p, g in zip(parts, grads)], timer)
    else:
        g_rows = _return_grads(parts, xchg, fetched, [g[0] for g in grads], timer, fold=_bag_fold)
    for p, f, g in zip(parts, fetched, g_rows):
        o = p.eng.make_opt(*opt_args)
        p.eng.sparse_apply(p.eng.make_table(p.table, *p.slots), f.req, g, o)    # ADAM_DENSE: the owner sweeps its shard
    timer("owner_apply")
    flats = []
    for (_, bot_g, top_g, cross_g), c in zip(grads, caches):
        pairs = bot_g + top_g + [pair for layer in cross_g for pair in layer]
        flats.append(torch.cat([t.reshape(-1) for dw, db in pairs for t in (dw, db) if t is not None]
                               + [c["out4"][:1]]))
    xchg.all_reduce(flats)
    outs = []
    for p, flat, c in zip(parts, flats, caches):
        o, off = p.eng.make_opt(*opt_args), 0
        for var, (s0, s1) in zip(p.dense_vars(), p.dense_slots):
            p.eng.dense_apply(var, s0, s1, flat[off:off + var.numel()].view_as(var), o)
            off += var.numel()
        out = c["out4"].clone()
        out[0] = flat[-1] / R
        outs.append(out)
    timer("dense_allreduce")
    return outs


def dlrm_inference_sharded(parts, xchg, batches):
    """DLRM.inference of row-sharded tables, a collective call: batches[k] = (dense, sparse) of parts[k], any B >= 0
    per rank.  -> per part its predictions [B]."""
    for p, (dense, sparse) in zip(parts, batches):
        if sparse.dim() != 2 or sparse.shape[1] != p.C or dense.shape[0] != sparse.shape[0]:
            raise ValueError(f"sparse features must be [B, {p.C}] with as many dense rows")
    Zs = _dlrm_fetch(parts, xchg, [b[1] for b in batches], False)[0]
    out = []
    for p, (dense, sparse), Z in zip(parts, batches, Zs):
        if dense.shape[0] == 0:
            out.append(torch.empty(0, dtype=torch.float32, device=dense.device))
        else:
            out.append(p.graph.forward(dense, sparse, Z=Z)["pred"])
    return out


# ---------------------------------------------------------------------------------------
# row-sharded GMF / WRMF: user / item / bias rows on their owners, GMF's w replicated
# ---------------------------------------------------------------------------------------
class PointwiseShard:
    """One rank's part of a row-sharded GMF (kind ORX_POINT_GMF) / WRMF (ORX_POINT_WRMF).  Row r of the user table,
    the item table and the item bias lives on rank r % world at local row r // world: ``user`` [max(ru, 1), dim],
    ``item`` [max(ri, 1), dim], ``bias`` [max(ri, 1), 1] (a rank without rows keeps a 1-row dummy that is never read),
    with their optimizer slots (s0, s1 per table, None where the optimizer has fewer).  GMF: ``w`` is this rank's [dim, 1]
    replica of the Dense(1) kernel with its slots ``w_slots``.  (a, b, use_sigmoid): WRMF's PointwiseMSELoss.

    The exchange runs over one row space whose ownership matches that layout (orx.h, row-sharded GMF / WRMF): user u is
    global row u, item i is global row world * Lu + i with Lu = ceil(U / world), so one orx_lookup_bucket call over the
    [B, 2] (user, item) lookups gives every owner one request list."""

    def __init__(self, eng, rank, world, total_users, total_items, dim, kind, user, item, bias, slots, w=None,
                 w_slots=(None, None), a=1.0, b=1.0, use_sigmoid=False):
        from . import native as N
        self.eng, self.rank, self.world, self.kind = eng, rank, world, kind
        self.U, self.I, self.D = int(total_users), int(total_items), int(dim)
        self.W = self.D + 4                     # exchange row: D values, the item bias, 3 zeros (16-byte aligned rows)
        self.Lu = (self.U + world - 1) // world
        self.row_off = row_offsets([world * self.Lu, self.I])
        self.ru, self.ri = shard_rows(self.U, rank, world), shard_rows(self.I, rank, world)
        want = ((max(self.ru, 1), self.D), (max(self.ri, 1), self.D), (max(self.ri, 1), 1))
        if tuple(tuple(t.shape) for t in (user, item, bias)) != want:
            raise ValueError(f"shard shapes {[tuple(t.shape) for t in (user, item, bias)]} != {want}")
        if (kind == N.ORX_POINT_GMF) != (w is not None):
            raise ValueError("GMF needs its w replica, WRMF has none")
        self.user, self.item, self.bias = user, item, bias
        self.user_slots, self.item_slots, self.bias_slots = (tuple(x) for x in slots)
        self.w, self.w_slots = w, tuple(w_slots)
        self.a, self.b, self.use_sigmoid = float(a), float(b), bool(use_sigmoid)
        self.last = {}          # sizes of the last step: unique rows fetched, rows served to the other ranks

    def local_shards(self):
        return self.user[:self.ru], self.item[:self.ri], self.bias[:self.ri]

    def load_global(self, user, item, bias):
        """user [U, D], item [I, D], bias [I] or [I, 1] (host or device): keep this rank's rows."""
        for t, g in zip(self.local_shards(), (user, item, bias)):
            t.copy_(take_shard(g, self.rank, self.world).reshape(t.shape))


def pointwise_step_sharded(parts, xchg, batches, opt_args, c_loss=1.0, c_l2=1.0, timer=None):
    """One synchronous training step of a row-sharded GMF / WRMF on the global batch (the union of every rank's batch;
    every rank passes the same local batch size B >= 1).  parts: the PointwiseShard of each rank this process drives;
    xchg: DistExchange or LoopbackExchange; batches[k] = (uid int32 [B], iid int32 [B], label f32 [B]) of parts[k],
    global ids on the device; opt_args = (kind, lr, eps, beta1, beta2, step); (c_loss, c_l2) the coefficients of
    tape.gradient(c_loss * loss + c_l2 * l2_loss).  ``timer(name)``, when given, is called after each phase.
    -> per part a [2] device tensor = the GLOBAL (loss, l2_loss), identical on every rank.

    A sample with an id out of range is skipped whole (orx_pointwise_shard_lookups), as orx_pointwise_step skips it; GMF's
    loss is still the mean over the B * R samples of the global batch.  The batch's rows are deduplicated before they
    travel (orx_lookup_bucket), the owners pack user / item rows with the item bias in one exchange row
    (orx_pointwise_serve), the per-lookup gradient rows (orx_pointwise_grad_rows) are folded onto the unique rows in a
    fixed order (orx_rows_segment_sum), and each owner applies the optimizer to its user, item and bias shards once per
    row over ALL ranks' requests (orx_sparse_apply_strided; Keras Adam() sweeps each shard).  GMF's w gradient, the loss
    and l2 travel in one all-reduce, with c_l2 * w and 0.5 * |w|^2 contributed by rank 0 only; every replica then
    applies the same summed gradient."""
    from . import native as N
    timer = timer or _untimed
    R = parts[0].world
    for p, (uid, iid, label) in zip(parts, batches):
        if uid.dim() != 1 or uid.shape != iid.shape or label.shape != uid.shape:
            raise ValueError("uid, iid and label must be 1-D tensors of one length")
        if uid.numel() < 1:
            raise ValueError("the sharded pointwise step needs B >= 1 samples per rank")
    lks = [p.eng.pointwise_shard_lookups(uid, iid, p.U, p.I) for p, (uid, iid, _) in zip(parts, batches)]
    fetched = _fetch_rows(parts, xchg, lks,
                          lambda p, req: p.eng.pointwise_serve(p.user, p.item, p.bias, p.ru, p.ri, p.Lu, req, p.W),
                          parts[0].W, True, timer)
    grads = []
    for p, (_, _, label), f in zip(parts, batches, fetched):
        grads.append(p.eng.pointwise_grad_rows(p.kind, f.got, p.D, f.bucket[2], label, p.w, 1.0 / (label.numel() * R),
                                               p.a, p.b, p.use_sigmoid, c_loss, c_l2, add_w_terms=p.rank == 0))
    timer("grad_rows")
    g_rows = _return_grads(parts, xchg, fetched, [gr[0] for gr in grads], timer)
    for p, g, f in zip(parts, g_rows, fetched):
        _, ul, il = f.served
        o = p.eng.make_opt(*opt_args)
        D = p.D
        p.eng.sparse_apply_rows(p.eng.make_table(p.user, *p.user_slots), ul, g[:, :D], o)
        p.eng.sparse_apply_rows(p.eng.make_table(p.item, *p.item_slots), il, g[:, :D], o)
        p.eng.sparse_apply_rows(p.eng.make_table(p.bias, *p.bias_slots), il, g[:, D:D + 1], o)
    timer("owner_apply")
    gmf = parts[0].kind == N.ORX_POINT_GMF
    flats = [torch.cat([gr[1], gr[2]]) if gmf else gr[2].clone() for gr in grads]
    xchg.all_reduce(flats)
    outs = []
    for p, flat in zip(parts, flats):
        if gmf:
            p.eng.dense_apply(p.w, *p.w_slots, flat[:p.D].view_as(p.w), p.eng.make_opt(*opt_args))
        outs.append(flat[-2:].clone())
    timer("dense_allreduce")
    return outs


class _PeerBuf:
    """A cudaMalloc'd, IPC-exportable device buffer viewed as a torch tensor (orx_peer_alloc)."""

    def __init__(self, eng, n_elems, dtype):
        self.eng = eng
        n = max(int(n_elems), 4)
        self.bytes = n * 4
        ptr = C.c_void_p()
        handle = C.create_string_buffer(64)
        _lib.check(eng.lib.orx_peer_alloc(eng.h, self.bytes, C.byref(ptr), handle), "orx_peer_alloc")
        self.ptr, self.handle = ptr.value, handle.raw
        typestr = {torch.float32: "<f4", torch.int32: "<i4"}[dtype]
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (self.ptr, False),
                                         "version": 2, "strides": None}
        self.t = torch.as_tensor(self, device=eng.device)     # zero-copy view of our own allocation

    def free(self):
        if self.ptr:
            self.t = None
            self.eng.lib.orx_peer_free(self.eng.h, C.c_void_p(self.ptr))
            self.ptr = 0


_MAILBOX_DTYPES = (torch.int32, torch.int32, torch.float32, torch.float32, torch.float32, torch.float32, torch.int32,
                   torch.int32)   # tripbox idbox got gotb gin ginb meta flags
_SHARD_ERRORS = {1: "a peer rank never arrived (flag wait timed out)",
                 2: "more triplets were routed to this rank than home_cap: rebuild with a larger home_cap",
                 3: "one owner received more requests than req_cap", 4: "gradient inbox overflow: rebuild with a larger gin_cap"}


class HomeRoutedPairwise:
    """Row-sharded BPR (kind 0) / UCML (kind 1) step, "home-routed" (csrc/orx_shard.cu): row r of the user and item
    tables lives on rank ``r % R``; a triplet is computed on the rank that owns its USER row, so only the two item rows
    travel in and the two item gradient rows travel out, as peer stores of aligned rows into IPC-mapped mailboxes.  One
    C call per step (six launches, flag words in peer memory instead of barriers, no collective, no host sync).
    ``torch.distributed`` is used once, to swap the 64-byte IPC handles.

    ``peers=None``: the R ranks are R processes (one per GPU) and the mailboxes are exchanged over ``torch.distributed``.
    ``peers=<LoopbackGroup>``: R virtual ranks share one device and one stream (1-GPU parity test of the same kernels).
    """

    def __init__(self, eng, rank, world, total_users, total_items, dim, batch, *, kind=0, opt_kind=1, lr=0.05, eps=1e-7,
                 beta1=0.9, beta2=0.999, margin=0.5, seed=0, init=True, home_cap=None, gin_cap=None, timeout_ms=20000,
                 peers=None, tables=None, slots=None):
        if dim % 4 or dim > 512:
            raise ValueError("the sharded step needs dim % 4 == 0 and dim <= 512")
        if opt_kind not in (0, 1, 2, 6, 8):
            raise ValueError("the sharded step supports SGD, Adagrad and row-sparse Adam, and SGD with (Nesterov) "
                             "momentum")
        self.eng, self.rank, self.world = eng, rank, world
        self.U, self.I, self.D, self.B = total_users, total_items, dim, batch
        self.kind, self.opt_kind, self.lr, self.eps, self.b1, self.b2, self.margin = kind, opt_kind, lr, eps, beta1, beta2, margin
        self.iterations = 0
        dev = eng.device
        self.ru, self.ri = shard_rows(total_users, rank, world), shard_rows(total_items, rank, world)
        if tables is not None:          # shards owned by the caller (openrec.tf2.recommenders.ShardedBPR: keras variables)
            self.user, self.item, self.bias = tables
            want = ((max(self.ru, 1), dim), (max(self.ri, 1), dim), (max(self.ri, 1), 1))
            if tuple(tuple(t.shape) for t in tables) != want:
                raise ValueError(f"shard shapes {[tuple(t.shape) for t in tables]} != {want}")
        else:
            self.user = torch.zeros(max(self.ru, 1), dim, dtype=torch.float32, device=dev)
            self.item = torch.zeros(max(self.ri, 1), dim, dtype=torch.float32, device=dev)
            self.bias = torch.zeros(max(self.ri, 1), 1, dtype=torch.float32, device=dev)
            if init:
                for k, t in enumerate((self.user, self.item, self.bias)):
                    eng.fill_uniform(t, -0.05, 0.05, seed * 1000003 + rank * 17 + k)
        n_slots = {0: 0, 1: 1, 2: 2, 6: 1, 8: 1}[opt_kind]           # 6 / 8: momentum, beta1 = its coefficient
        fill = 0.1 if opt_kind == 1 else 0.0
        mk = lambda t: [torch.full_like(t, fill) for _ in range(n_slots)] + [None] * (2 - n_slots)
        if slots is not None:           # optimizer slots owned by the caller (the keras optimizer's slot tensors)
            self.user_slots, self.item_slots, self.bias_slots = (list(x) for x in slots)
        else:
            self.user_slots, self.item_slots, self.bias_slots = mk(self.user), mk(self.item), mk(self.bias)
        # capacities: worst case for small problems (tests), 2x the expected load for big ones (errors are sticky flags)
        small = world * batch <= (1 << 16)
        self.home_cap = int(home_cap or (world * batch if small else 2 * batch))
        self.req_cap = 2 * self.home_cap
        self.gin_cap = int(gin_cap or (world * (2 * self.home_cap + 32) if small else 4 * batch + 32 * world))
        self.gin_cap = (self.gin_cap + 31) // 32 * 32
        self._x = _lib.OrxShard(world, rank, dim, batch, self.home_cap, self.req_cap, self.gin_cap, timeout_ms,
                                0, 0, 0, 0, 0, 0, 0, 0)
        sizes = (C.c_int64 * 8)()
        _lib.check(eng.lib.orx_shard_sizes(C.byref(self._x), sizes), "orx_shard_sizes")
        self._loop = peers
        self._opened = []
        if peers is None:
            self._bufs = [_PeerBuf(eng, sizes[k], _MAILBOX_DTYPES[k]) for k in range(8)]
            mine = [b.ptr for b in self._bufs]
            torch.cuda.synchronize()
            everyone = [None] * world
            dist.all_gather_object(everyone, [b.handle for b in self._bufs])
            ptrs = np.zeros((8, world), dtype=np.int64)
            for r in range(world):
                for k in range(8):
                    if r == rank:
                        ptrs[k, r] = mine[k]
                    else:
                        p = C.c_void_p()
                        _lib.check(eng.lib.orx_peer_open(eng.h, everyone[r][k], C.byref(p)), "orx_peer_open")
                        self._opened.append(p.value)
                        ptrs[k, r] = p.value
            self._set_pointers(ptrs)
            dist.barrier()
        else:                    # loopback: plain device memory, the group wires the pointer tables
            self._bufs = None
            self._tensors = [torch.zeros(max(int(sizes[k]), 4), dtype=_MAILBOX_DTYPES[k], device=dev) for k in range(8)]
            peers._register(self)
        self._out = torch.zeros(16, 4, dtype=torch.float32, device=dev)     # ring of step outputs
        self._tabs = (eng.make_table(self.user, *self.user_slots), eng.make_table(self.item, *self.item_slots),
                      eng.make_table(self.bias, *self.bias_slots))
        self.launches_per_step = 6      # 4 when every step announces the next batch (step(next_ids=...))
        self._announced = None

    def _set_pointers(self, ptrs):
        self._ptrs = torch.from_numpy(np.ascontiguousarray(ptrs)).to(self.eng.device)
        base = self._ptrs.data_ptr()
        for k, name in enumerate(("tripbox", "idbox", "got", "gotb", "gin", "ginb", "meta", "flags")):
            setattr(self._x, name, base + 8 * self.world * k)

    def _flags(self):
        return self._bufs[7].t if self._bufs is not None else self._tensors[7]

    def _call(self, uid, pid, nid, c_loss, c_l2, lo, hi, nxt=None, epoch=None):
        eng = self.eng
        B = uid.numel()
        if B > self.B:
            raise ValueError("batch larger than the mailboxes this model was built for")
        epoch = self.iterations if epoch is None else epoch
        out4 = self._out[epoch % 16]
        o = eng.make_opt(self.opt_kind, self.lr, self.eps, self.b1, self.b2, epoch)
        vp = lambda t: C.c_void_p(t.data_ptr())
        nx = (vp(nxt[0]), vp(nxt[1]), vp(nxt[2]), nxt[0].numel()) if nxt is not None else (None, None, None, 0)
        _lib.check(eng.lib.orx_shard_step(eng.h, self.kind, C.byref(self._x), C.byref(self._tabs[0]), C.byref(self._tabs[1]),
                                          C.byref(self._tabs[2]), vp(uid), vp(pid), vp(nid), B, *nx, self.U, self.I, self.margin,
                                          c_loss, c_l2, 1.0 / (B * self.world), C.byref(o), epoch, lo, hi, vp(out4),
                                          eng.stream()), "orx_shard_step")
        return out4

    def step(self, uid, pid, nid, c_loss=1.0, c_l2=1.0, reduce_loss=True, next_ids=None):
        """uid/pid/nid: this rank's int32 GLOBAL ids on the device (every rank must pass the same batch size).
        Returns a [2] device tensor = the GLOBAL (loss, l2_loss): the partials ride the meta mailboxes.

        ``next_ids=(uid, pid, nid)`` announces the batch of the NEXT step (device tensors; the next call must pass these
        very tensors): its routing and request phases -- two of the four cross-rank handoffs of a step -- then run inside
        this step's apply launch, and the next step is four launches instead of six.  All ranks announce, or none."""
        if self._loop is not None:
            raise RuntimeError("loopback ranks are stepped by their LoopbackGroup")
        if self._announced is not None and any(a.data_ptr() != b.data_ptr() for a, b in zip(self._announced, (uid, pid, nid))):
            raise ValueError("this batch is not the one announced with next_ids= in the previous step")
        self.iterations += 1
        out = self._call(uid, pid, nid, c_loss, c_l2, 0, 5, nxt=next_ids)[:2]
        self._announced = tuple(next_ids) if next_ids is not None else None     # also keeps the tensors alive
        return out

    def censor_vec(self, uid, pid, nid):
        """UCML.censor_vec (ucml.py:44-48) on this model's shards, a collective call (censor_vec_sharded).  Safe after
        a step that announced the next batch: the announced route / request read no table row, and every later read of
        a row runs on its owner's stream, behind the owner's censor."""
        if self._loop is not None:
            raise RuntimeError("loopback ranks are censored by their LoopbackGroup")
        censor_vec_sharded(self.eng, self.user, self.item, self.U, self.I, self.world, self.rank, uid, pid, nid)

    def check(self):
        """Raise if a flag wait timed out or a mailbox overflowed (sticky device word; one tiny D2H read)."""
        code = int(self._flags()[4 * 64].item())
        if code:
            raise RuntimeError("sharded step: " + _SHARD_ERRORS.get(code, f"error {code}"))

    # ---- global <-> shard (tests, checkpoints)
    def load_global(self, user, item, bias):
        for t, g in zip(self.local_shards(), (user, item, bias)):
            t.copy_(take_shard(g, self.rank, self.world).reshape(t.shape))

    def local_shards(self):
        return self.user[:self.ru], self.item[:self.ri], self.bias[:self.ri]

    def gather_global(self):
        """-> (user, item, bias) full tables on every rank (test helper; sizes must be small)."""
        return [gather_shards(t, total, self.world) for t, total in zip(self.local_shards(), (self.U, self.I, self.I))]

    # ---- per-rank shard checkpoint (SURVEY 8f N4 for tables that only exist sharded)
    def save_shard(self, path):
        """Write this rank's rows + optimizer slots + step count to ``path`` (one .npz per rank)."""
        arrs = {"meta": np.array([self.rank, self.world, self.U, self.I, self.D, self.kind, self.opt_kind, self.iterations],
                                 dtype=np.int64)}
        for name, t, slots in (("user", self.user[:self.ru], self.user_slots), ("item", self.item[:self.ri], self.item_slots),
                               ("bias", self.bias[:self.ri], self.bias_slots)):
            arrs[name] = t.cpu().numpy()
            for k, s in enumerate(slots):
                if s is not None:
                    arrs[f"{name}_s{k}"] = s[:t.shape[0]].cpu().numpy()
        np.savez(path, **arrs)

    def load_shard(self, path):
        z = np.load(path)
        meta = z["meta"].tolist()
        want = [self.rank, self.world, self.U, self.I, self.D, self.kind, self.opt_kind]
        if meta[:7] != want:
            raise ValueError(f"shard checkpoint {path} was written for (rank, world, U, I, D, kind, opt) = {meta[:7]}, "
                             f"this model is {want}")
        dev = self.eng.device
        for name, t, slots in (("user", self.user[:self.ru], self.user_slots), ("item", self.item[:self.ri], self.item_slots),
                               ("bias", self.bias[:self.ri], self.bias_slots)):
            t.copy_(torch.from_numpy(z[name]).to(dev))
            for k, s in enumerate(slots):
                if s is not None:
                    s[:t.shape[0]].copy_(torch.from_numpy(z[f"{name}_s{k}"]).to(dev))
        self.iterations = int(meta[7])

    def close(self):
        torch.cuda.synchronize()
        if self._bufs is None:
            return
        dist.barrier()
        for p in self._opened:
            self.eng.lib.orx_peer_close(self.eng.h, C.c_void_p(p))
        self._opened = []
        dist.barrier()
        for b in self._bufs:
            b.free()
        self._bufs = None


class LoopbackGroup:
    """R virtual ranks of HomeRoutedPairwise on ONE device and ONE stream: every rank has its own liborx handle, tables
    and mailboxes (plain device memory); a step issues phase k of the six launches for every rank before phase k + 1,
    so every flag a kernel waits for is already set.  Same kernels, same peer-pointer tables as the multi-GPU step."""

    def __init__(self, world, total_users, total_items, dim, batch, device=None, **kw):
        from . import native
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.world = world
        self.ranks = []
        self._announced = None
        self._engines = [native.Engine(dev.index or 0) for _ in range(world)]
        for r in range(world):
            HomeRoutedPairwise(self._engines[r], r, world, total_users, total_items, dim, batch, peers=self, **kw)
        ptrs = np.zeros((8, world), dtype=np.int64)
        for r, m in enumerate(self.ranks):
            for k in range(8):
                ptrs[k, r] = m._tensors[k].data_ptr()
        for m in self.ranks:
            m._set_pointers(ptrs)
        torch.cuda.synchronize()

    def _register(self, m):
        self.ranks.append(m)

    def step(self, batches, c_loss=1.0, c_l2=1.0, next_batches=None):
        """batches[r] = (uid, pid, nid) of rank r.  Returns the [2] global (loss, l2_loss) tensor of every rank.
        ``next_batches`` announces the next step's batches: their route / request phases are issued between compute and
        apply of this step -- where the multi-GPU step runs them (inside the apply launch; fused roles of R virtual ranks
        on one stream would wait for each other, so the loopback issues the stand-alone kernels at that point)."""
        if self._announced is not None:
            for b, a in zip(batches, self._announced):
                if any(x.data_ptr() != y.data_ptr() for x, y in zip(b, a)):
                    raise ValueError("these batches are not the ones announced in the previous step")
        for m in self.ranks:
            m.iterations += 1
        outs = [None] * self.world
        for ph in range(6):       # phases 0 / 1 of an announced batch were issued a step ago: the C call skips them
            fused = ph == 4 and next_batches is not None and self.world == 1    # one rank: the real fused launch
            if ph == 4 and next_batches is not None and not fused:
                self._issue_early(next_batches, c_loss, c_l2)
            for r, m in enumerate(self.ranks):
                outs[r] = m._call(*batches[r], c_loss, c_l2, ph, ph, nxt=next_batches[r] if fused else None)
        self._announced = [tuple(b) for b in next_batches] if next_batches is not None else None
        return [o[:2] for o in outs]

    def _issue_early(self, next_batches, c_loss, c_l2):
        """Route (phase 0) of the announced batches for every rank, then request (phase 1)."""
        for r, m in enumerate(self.ranks):
            m._call(*next_batches[r], c_loss, c_l2, 0, 0, epoch=m.iterations + 1)
        for r, m in enumerate(self.ranks):
            m._call(*next_batches[r], c_loss, c_l2, 1, 1, epoch=m.iterations + 1)

    def censor_vec(self, batches):
        """UCML.censor_vec of the global batch, batches[r] = (uid, pid, nid) of rank r (the same B for every rank): the
        [R][3][B] block an all-gather would give, built on the device, then each rank's three orx_censor_shard calls
        on its own engine and shards -- the kernels of HomeRoutedPairwise.censor_vec."""
        B = batches[0][0].numel()
        if any(x.numel() != B for b in batches for x in b):
            raise ValueError("every rank passes uid, pid and nid of one length B")
        if B == 0:
            return
        ids = torch.cat([torch.stack([x.reshape(-1) for x in b]).to(torch.int32).reshape(-1) for b in batches])
        for m in self.ranks:
            censor_gathered(m.eng, m.user, m.item, m.U, m.I, self.world, m.rank, ids, B)

    def load_global(self, user, item, bias):
        for m in self.ranks:
            m.load_global(user, item, bias)

    def gather_global(self):
        R = self.world
        outs = []
        for k, total in enumerate((self.ranks[0].U, self.ranks[0].I, self.ranks[0].I)):
            shards = [m.local_shards()[k] for m in self.ranks]
            full = torch.zeros(total, shards[0].shape[1], dtype=torch.float32, device=shards[0].device)
            for r in range(R):
                full[r::R] = shards[r]
            outs.append(full)
        return outs

    def check(self):
        for m in self.ranks:
            m.check()

    def close(self):
        torch.cuda.synchronize()
        for e in self._engines:
            e.close()


# ---------------------------------------------------------------------------------------
# bench.py's N>1 leg
# ---------------------------------------------------------------------------------------
def bench(args, rank, world, eng, barrier, clocks=None):
    import bench as B
    from . import native as N
    K, W = args.steps, max(3, args.warmup)
    dev = eng.device
    U, I, D, Bsz = B.U, 12_500_000 * world, B.D, B.B      # BASELINE configs[4]: 100M items x 128 over 8 GPUs
    # Default: the home-routed peer-store exchange (csrc/orx_shard.cu); ORX_SHARDED=nccl selects the NCCL all-to-all form
    mode = os.environ.get("ORX_SHARDED", "home")
    if mode == "home":
        model = HomeRoutedPairwise(eng, rank, world, U, I, D, Bsz, kind=0, opt_kind=N.ORX_OPT_ADAGRAD, lr=B.LR, seed=1)
    else:
        model = ShardedPairwise(eng, rank, world, U, I, D, kind=0, opt_kind=N.ORX_OPT_ADAGRAD, lr=B.LR, seed=1)
    g = torch.Generator(device="cpu").manual_seed(100 + rank)
    host_ids = [tuple(torch.randint(0, n, (Bsz,), generator=g, dtype=torch.int32).pin_memory() for n in (U, I, I))
                for _ in range(B.N_BATCHES)]
    dev_ids = [tuple(x.to(dev) for x in b) for b in host_ids]

    # Every step announces the next batch (HomeRoutedPairwise.step(next_ids=...)): a training loop knows it -- the data
    # pipeline is a step ahead -- and the routing + request phases of step t+1 then hide under the apply phase of step t.
    # ORX_SHARD_ANNOUNCE=0 measures the six-launch step without it.
    announce = mode == "home" and os.environ.get("ORX_SHARD_ANNOUNCE", "1") != "0"
    NB = B.N_BATCHES
    cnt = {"k": 0}

    def step(i):
        k = cnt["k"]
        cnt["k"] = k + 1
        if announce:
            model.step(*dev_ids[k % NB], reduce_loss=False, next_ids=dev_ids[(k + 1) % NB])
        else:
            model.step(*dev_ids[k % NB], reduce_loss=False)

    def drain():            # the batch announced by the last step of a loop is stepped outside the timed region
        if announce and model._announced is not None:
            model.step(*model._announced)
            cnt["k"] += 1

    for i in range(W):
        step(i)
    seconds = B._timed(step, K, barrier, torch, clocks)
    drain()
    # e2e: pinned host ids in, global loss out to the host, every step (read one step behind, so the copy overlaps).
    # The ids of batch k+2 are uploaded on a side stream during step k into a 4-deep ring of device buffers.
    pinned = [torch.zeros(2).pin_memory() for _ in range(2)]
    state = {"prev": None, "last": None}
    ring = [tuple(torch.empty(Bsz, dtype=torch.int32, device=dev) for _ in range(3)) for _ in range(4)]
    up_ev, done_ev = [None] * 4, [None] * 4
    side = torch.cuda.Stream(device=dev)
    e2e = {"k": 0}

    def upload(k):
        if done_ev[k % 4] is not None:
            side.wait_event(done_ev[k % 4])          # the step that last read this ring slot (batch k - 4) has finished
        with torch.cuda.stream(side):
            for dst, src in zip(ring[k % 4], host_ids[k % NB]):
                dst.copy_(src, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
        up_ev[k % 4] = ev

    def e2e_step(i):
        k = e2e["k"]
        e2e["k"] = k + 1
        if k == 0:
            upload(0)
            upload(1)
        cur = torch.cuda.current_stream(dev)
        cur.wait_event(up_ev[k % 4])
        cur.wait_event(up_ev[(k + 1) % 4])
        out = model.step(*ring[k % 4], next_ids=ring[(k + 1) % 4]) if announce else model.step(*ring[k % 4])   # global (loss, l2)
        d = torch.cuda.Event()
        d.record()
        done_ev[k % 4] = d
        upload(k + 2)
        pinned[i & 1].copy_(out, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        if state["prev"] is not None:
            state["prev"][0].synchronize()
            state["last"] = state["prev"][1].clone()
        state["prev"] = (ev, pinned[i & 1])

    for i in range(W):
        e2e_step(i)
    e2e_seconds = B._timed(e2e_step, K, barrier, torch, clocks)
    drain()
    state["prev"][0].synchronize()
    last = state["prev"][1].clone()
    if hasattr(model, "check"):
        model.check()
    checked = None
    if getattr(args, "check", False):
        # parity at the full table shape (BASELINE configs[4]); the oracle stays under tests/ (test infrastructure)
        tests_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests")
        if tests_dir not in sys.path:
            sys.path.insert(0, tests_dir)
        import shard_check
        access = shard_check.HomeRoutedAccess(model) if mode == "home" else shard_check.CombinedAccess(model)
        checked = shard_check.run(model, access, rank, world, U, I, D, Bsz, kind=0, opt_kind=1, lr=B.LR)
    # NVLink-bound exchange (SURVEY 8e): bytes per GPU per direction per step: rows out as owner + gradient rows out as home
    rows_each_way = 2 if mode == "home" else 3
    link_bytes = 2.0 * (world - 1) / world * rows_each_way * (D + 1) * 4 * Bsz
    nvlink_peak = 450.0
    ms = seconds / K * 1e3
    roofline = {"bound": "nvlink", "kernel": "k_sh_serve + k_sh_compute (peer stores)" if mode == "home" else "NCCL all-to-all",
                "achieved": link_bytes / (seconds / K) / 1e9, "peak": nvlink_peak, "unit": "GB/s",
                "frac": link_bytes / (seconds / K) / 1e9 / nvlink_peak, "traffic": None,
                "peak_source": "H100 SXM datasheet: NVLink 4, 450 GB/s per direction per GPU",
                "algorithmic_bytes_per_launch": link_bytes,
                "note": f"per-GPU per-direction NVLink bytes of the item-row + gradient-row exchange ({rows_each_way} rows each way "
                        f"per triplet, (N-1)/N of them remote) over the WHOLE step time ({ms:.3f} ms): the step also does the local "
                        "HBM work of the single-GPU step; the N = 1 line carries the HBM roofline of the fused kernel"}
    per_step = 4 if announce else model.launches_per_step
    return {"seconds": seconds, "e2e_seconds": e2e_seconds, "launches": per_step * K * world,
            "units_per_step": Bsz, "h2d": 3 * 4 * Bsz, "d2h": 8, "roofline": roofline,
            "e2e_api": f"openrec_b200.sharded.{type(model).__name__}.step; pinned host ids in, global loss to host each step",
            "extra": {"last_loss": [float(x) for x in last], "total_items": I, "total_users": U, "check": checked,
                      "exchange": {"home": "home-routed: triplets computed on the user row's owner; item rows / gradient rows "
                                           "as peer stores into IPC-mapped mailboxes over NVLink, flag words instead of "
                                           "barriers, no collective, no host sync",
                                   }.get(mode, "NCCL all-to-all (counts, ids, rows, gradient rows)")}}
