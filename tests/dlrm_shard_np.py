"""TEST INFRASTRUCTURE: numpy restatements of orx_lookup_bucket and orx_rows_segment_sum (the row-sharded DLRM step's two
kernels), and ``install(FakeEngine)``, which gives the oracle-backed engine of tests/fake_engine.py these two entry points
and orx_gather's contract for an out-of-range id (a zero row), so the sharded DLRM step runs on CPU over gloo."""
from __future__ import annotations

import numpy as np
import torch


def lookup_bucket_np(sparse, row_off, world):
    """sparse int [B, T], row_off [T + 1] -> (counts, send_local [n_uniq], slot [B*T], grp_off [n_uniq + 1],
    grp_idx [n_valid]) as orx_lookup_bucket defines them (the unspecified tails left off)."""
    s = np.asarray(sparse, np.int64)
    off = np.asarray(row_off, np.int64)
    ok = (s >= 0) & (s < np.diff(off)[None, :])
    g = np.where(ok, off[:-1][None, :] + s, -1).reshape(-1)
    valid = np.flatnonzero(g >= 0)
    G = int(off[-1])
    L = max((G + world - 1) // world, 1)
    gv = g[valid]
    uniq, inv = np.unique((gv % world) * L + gv // world, return_inverse=True)
    slot = np.full(g.size, -1, np.int32)
    slot[valid] = inv
    counts = np.bincount(uniq // L, minlength=world).astype(np.int32)
    grp_off = np.concatenate([[0], np.cumsum(np.bincount(inv, minlength=uniq.size))]).astype(np.int32)
    grp_idx = valid[np.argsort(inv, kind="stable")].astype(np.int32)
    return counts, (uniq % L).astype(np.int32), slot, grp_off, grp_idx


def _lookup_bucket(self, sparse, row_off, world):
    counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(sparse.numpy(), row_off, world)
    n = slot.size
    pad = lambda a, m: torch.from_numpy(np.concatenate([a, np.zeros(m - a.size, np.int32)]))
    return torch.from_numpy(counts), pad(send_local, n), torch.from_numpy(slot), pad(grp_off, n + 1), pad(grp_idx, n)


def _rows_segment_sum(self, src, grp_off, grp_idx, n_uniq, out=None):
    s, off, idx = src.numpy(), grp_off.numpy(), grp_idx.numpy()
    res = np.zeros((int(n_uniq), s.shape[1]), np.float32)
    for j in range(int(n_uniq)):
        for p in range(off[j], off[j + 1]):
            res[j] += s[idx[p]]
    if out is None:
        return torch.from_numpy(res)
    out.copy_(torch.from_numpy(res))
    return out


def _gather(self, tab, ids, n_bad=None):
    ids = ids.long().reshape(-1)
    ok = ((ids >= 0) & (ids < tab.shape[0])).reshape(-1, 1)
    return torch.where(ok, tab[ids.clamp(0, tab.shape[0] - 1)], torch.zeros((), dtype=tab.dtype))


def install(engine_cls):
    """Add the sharded DLRM entry points to the oracle-backed engine class (tests only)."""
    engine_cls.lookup_bucket = _lookup_bucket
    engine_cls.rows_segment_sum = _rows_segment_sum
    engine_cls.gather = _gather
