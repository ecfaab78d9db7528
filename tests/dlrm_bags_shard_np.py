"""TEST INFRASTRUCTURE: numpy restatements of orx_bag_shard_lookups and orx_bag_segment_sum (the multi-hot form of the
row-sharded DLRM step), and ``install(FakeEngine)``, which gives the oracle-backed engine of tests/fake_engine.py these
two entry points, orx_bag_gather and the one-hot sharded entry points of tests/dlrm_shard_np.py, so the multi-hot
sharded DLRM step runs on CPU over gloo."""
from __future__ import annotations

import numpy as np
import torch

import dlrm_bags_np as NB
import dlrm_shard_np


def bag_shard_lookups_np(sparse, col_off, row_off):
    """sparse int [B, C] -> int32 [B, C]: row_off[k] + id for a valid id of a column of table k's bag, else -1."""
    s = np.asarray(sparse, np.int64)
    co, ro = np.asarray(col_off, np.int64), np.asarray(row_off, np.int64)
    k = np.repeat(np.arange(len(co) - 1), np.diff(co))               # the table of each column
    ok = (s >= 0) & (s < (ro[1:] - ro[:-1])[k][None, :])
    return np.where(ok, ro[:-1][k][None, :] + s, -1).astype(np.int32)


def bag_scale(slot, col_off, B, mean):
    """-> (k [C] the table of each column, div [B, C] float32: the valid count of lookup (b, c)'s bag for a mean, else
    1)."""
    co = np.asarray(col_off, np.int64)
    k = np.repeat(np.arange(len(co) - 1), np.diff(co))
    sl = np.asarray(slot).reshape(B, -1)
    div = np.ones(sl.shape, np.float32)
    if mean:
        n = np.stack([(sl[:, co[t]:co[t + 1]] >= 0).sum(1) for t in range(len(co) - 1)], 1)
        div = np.maximum(n[:, k], 1).astype(np.float32)
    return k, div


def bag_segment_sum_np(dz, col_off, mean, slot, grp_off, grp_idx, n_uniq, dtype=np.float32):
    """dz [B, T, D] -> [n_uniq, D]: row j = the sum over p in grp_off[j] .. grp_off[j+1] of lookup grp_idx[p]'s row
    dz[b, k(c)] (/ its bag's valid count for a mean, before the add), added in that order in ``dtype``."""
    dz = np.asarray(dz)
    B, C = dz.shape[0], int(col_off[-1])
    k, div = bag_scale(slot, col_off, B, mean)
    out = np.zeros((int(n_uniq), dz.shape[2]), dtype)
    for j in range(int(n_uniq)):
        acc = np.zeros(dz.shape[2], dtype)
        for p in range(grp_off[j], grp_off[j + 1]):
            b, c = divmod(int(grp_idx[p]), C)
            v = dz[b, k[c]].astype(dtype)
            acc = acc + (v / dtype(div[b, c]) if mean else v)
        out[j] = acc
    return out


def _bag_shard_lookups(self, sparse, col_off, row_off):
    return torch.from_numpy(bag_shard_lookups_np(sparse.numpy(), col_off, row_off))


def _bag_segment_sum(self, dz3d, col_off, mode, slot, grp_off, grp_idx, n_uniq, out=None):
    res = torch.from_numpy(bag_segment_sum_np(dz3d.numpy(), col_off, mode == 1, slot.numpy(), grp_off.numpy(),
                                              grp_idx.numpy(), n_uniq))
    if out is None:
        return res
    out.copy_(res)
    return out


def _bag_gather(self, tabs, sparse, col_off, mode, out2d, n_bad=None):
    B, T = sparse.shape[0], len(tabs)
    Z, _, _ = NB.pool_f32([t.numpy() for t in tabs], sparse.numpy(), col_off, mode == 1)
    out2d[:, :T * tabs[0].shape[1]].copy_(torch.from_numpy(Z.reshape(B, -1)))


def install(engine_cls):
    """Add the sharded DLRM entry points, one-hot and multi-hot, to the oracle-backed engine class (tests only)."""
    dlrm_shard_np.install(engine_cls)
    engine_cls.bag_shard_lookups = _bag_shard_lookups
    engine_cls.bag_segment_sum = _bag_segment_sum
    engine_cls.bag_gather = _bag_gather
