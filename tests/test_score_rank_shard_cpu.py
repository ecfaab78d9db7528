"""CPU, world size 2 and 3 over gloo: RankingEvaluator.evaluate on a ShardedBPR / ShardedUCML runs the four phases of
the sharded evaluation on every rank with an all-reduce between them, and the result equals the oracle's AUC / NDCG /
Recall on the gathered tables.  The engine is the oracle-backed one of tests/fake_engine.py with a test-local
score_rank_shard that restates the phases in numpy (each rank counts over its own item rows only), so this checks the
counting decomposition and the collective plumbing; the kernels are checked in tests/test_gpu_score_rank_shard.py."""
import os

import numpy as np
import pytest
import torch
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _scores(kind, urow, items, bias):
    """float32 scores of one user row against item rows, each computed in float64 and rounded once."""
    u, it = urow.astype(np.float64)[None, :], items.astype(np.float64)
    s = (u * it).sum(-1) if kind == 0 else -((u - it) ** 2).sum(-1)
    if bias is not None:
        s = s + bias.astype(np.float64)
    return s.astype(F32)


def _lists(u, U, I, po, pi, eo, ei):
    if not 0 <= u < U:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), 0
    p = pi[po[u]:po[u + 1]].astype(np.int64)
    e = ei[eo[u]:eo[u + 1]].astype(np.int64) if eo is not None else np.zeros(0, np.int64)
    return p[(p >= 0) & (p < I)], e[(e >= 0) & (e < I)], len(p)


def _score_rank_shard(self, kind, phase, g, user, item, bias, uid, pos_off, pos_items, excl_off, excl_items, max_pos,
                      xrows, xpred, xcnt, at=()):
    R, r, U, I = g.world, g.rank, g.total_users, g.total_items
    uid = uid.numpy().astype(np.int64)
    Bu, D, P = len(uid), user.shape[1], max_pos + 1
    po, pi = pos_off.numpy(), pos_items.numpy()
    eo, ei = (excl_off.numpy(), excl_items.numpy()) if excl_off is not None else (None, None)
    rows = xrows.numpy().view(F32).reshape(Bu, D)
    bias_np = None if bias is None else bias.numpy()
    item_np = item.numpy()
    if phase == 0:                   # this rank's user rows, 0 elsewhere
        out = np.zeros((Bu, D), F32)
        for b, u in enumerate(uid):
            if 0 <= u < U and u % R == r:
                out[b] = user.numpy()[u // R]
        xrows.copy_(torch.from_numpy(out.view(np.int32).reshape(-1)))
        return None
    if phase == 1:                   # this rank's positives' scores, 0 elsewhere
        out = np.zeros((Bu, P), F32)
        for b, u in enumerate(uid):
            p, _, raw = _lists(u, U, I, po, pi, eo, ei)
            if raw > max_pos:
                continue
            for q, i in enumerate(p):
                if i % R == r:
                    out[b, q] = _scores(kind, rows[b], item_np[i // R][None], None if bias_np is None else
                                        bias_np[i // R:i // R + 1])[0]
        xpred.copy_(torch.from_numpy(out.view(np.int32).reshape(-1)))
        return None
    if phase == 2:                   # counts over this rank's item rows: AUC terms of its eval items, rank hits of
        pred = xpred.numpy().view(F32).reshape(Bu, P)   # its items that are not excluded
        cnt = np.zeros((Bu, P), np.int64)
        mine = np.arange(g.local_items, dtype=np.int64) * R + r
        for b, u in enumerate(uid):
            p, e, raw = _lists(u, U, I, po, pi, eo, ei)
            if raw > max_pos or not len(p):
                continue
            n = len(p)
            pp = pred[b, :n]
            with np.errstate(all="ignore"):
                sp = np.exp(pp) * (~np.isin(p, e)).astype(F32)
            sp = np.where(np.isnan(sp), F32(np.inf), sp)
            s = _scores(kind, rows[b], item_np[:g.local_items], None if bias_np is None else bias_np[:g.local_items])
            ev = ~np.isin(mine, p) & ~np.isin(mine, e)
            cnt[b, 0] = int(np.count_nonzero(pp[None, :] >= s[ev][:, None]))
            with np.errstate(all="ignore"):
                j = np.count_nonzero(np.sort(sp)[None, :] < np.exp(s[~np.isin(mine, e)])[:, None], axis=1)
            cnt[b, 1:n + 1] = np.bincount(j, minlength=n + 1)[1:n + 1]
        xcnt.copy_(torch.from_numpy(cnt.reshape(-1)))
        return None
    cnt = xcnt.numpy().reshape(Bu, P)  # phase 3: the metrics from the summed counts
    auc, ndcg, rec = (np.full(Bu, np.nan, F32), np.full((Bu, len(at)), np.nan, F32),
                      np.full((Bu, len(at)), np.nan, F32))
    for b, u in enumerate(uid):
        p, e, raw = _lists(u, U, I, po, pi, eo, ei)
        if raw > max_pos:
            continue
        n, extra = len(p), len(set(e.tolist()) - set(p.tolist()))
        ranks = np.array([cnt[b, q + 1:n + 1].sum() for q in range(n)], np.int64).astype(F32)
        with np.errstate(all="ignore"):
            auc[b] = F32(cnt[b, 0]) / F32(n * (I - n - extra))
            w = (F32(1) / (np.log(ranks + 2) / np.log(F32(2.0)))).astype(F32)
            for k, a in enumerate(at):
                ndcg[b, k] = (w * (ranks < a)).sum(dtype=F32)
                rec[b, k] = F32(np.count_nonzero(ranks < a)) / F32(n)
    return torch.from_numpy(auc), torch.from_numpy(ndcg), torch.from_numpy(rec)


def _sizes(Bu, dim, max_pos):
    return Bu * dim, Bu * (max_pos + 1), Bu * (max_pos + 1)


def _worker(world, ucml):
    """One rank: sharded model, evaluate, gather, compare on rank 0 with the oracle on the global tables."""
    import torch.distributed as dist
    import fake_engine
    from oracle import openrec_oracle as O
    fake_engine.FakeEngine.score_rank_shard = _score_rank_shard
    fake_engine.FakeEngine.score_rank_shard_sizes = staticmethod(_sizes)
    fake_engine.install()
    from openrec.tf2.data import Dataset
    from openrec.tf2.metrics import RankingEvaluator
    from openrec.tf2.recommenders import ShardedBPR, ShardedUCML
    rank = int(os.environ["RANK"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(17)
    U, I, D = 23, 61, 6                            # U, I not multiples of the world size
    va, tr = [], []
    for u in range(U):
        items = rng.choice(I, 12, replace=False)
        if u % 5:
            va += [(u, int(i)) for i in items[:1 + u % 4]]
        tr += [(u, int(i)) for i in items[4:4 + int(rng.integers(0, 8))]]
    tr += [(3, int(va[0][1]))]                    # a validation positive that is also excluded

    def mk(pairs):
        raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = np.array(pairs).T
        return Dataset(raw_data=raw, total_users=U, total_items=I)
    val, train = mk(va), mk(tr)
    model = (ShardedUCML if ucml else ShardedBPR)(D, D, U, I, seed=2)
    at = [1, 5, 20]
    ev = RankingEvaluator(val, excl_datasets=[train], at=at, batch_size=7)
    res = ev.evaluate(model)
    got = [res[k].numpy() for k in ("AUC", "NDCG", "Recall")]
    tabs = []
    for v, total in zip(model.variables, (U, I, I)):      # row r of the global table = local row r // R of rank r % R
        t = v.t
        per = (total + world - 1) // world
        pad = torch.zeros(per, t.shape[1])
        pad[:min(t.shape[0], (total - rank + world - 1) // world)] = t[:(total - rank + world - 1) // world]
        parts = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(parts, pad)
        tabs.append(torch.stack(parts, 1).reshape(per * world, -1)[:total].numpy())
    everyone = [None] * world
    dist.all_gather_object(everyone, got)
    if rank == 0:
        for theirs in everyone:
            for x, y in zip(got, theirs):
                np.testing.assert_array_equal(x.view(np.int32), y.view(np.int32))
        user, item, bias = tabs
        kind = 1 if ucml else 0
        users = ev.warm_users
        pred = np.stack([_scores(kind, user[u], item, bias[:, 0]) for u in users])
        pos, excl = np.zeros((len(users), I), bool), np.zeros((len(users), I), bool)
        for b, u in enumerate(users):
            pos[b, ev.pos_items[ev.pos_off[u]:ev.pos_off[u + 1]]] = True
            excl[b, ev.excl_items[ev.excl_off[u]:ev.excl_off[u + 1]]] = True
        with np.errstate(all="ignore"):
            want = O.auc(pos, pred, excl), O.ndcg(pos, pred, excl, tuple(at)), O.recall(pos, pred, excl, tuple(at))
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_allclose(got[1], want[1], rtol=1e-6)
        np.testing.assert_array_equal(got[2], want[2])
        assert len(users) > 14 and np.isfinite(got[0]).sum() > 10
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("ucml", [False, True], ids=["bpr", "ucml"])
def test_sharded_evaluation_equals_oracle(world, ucml):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_score_rank_shard_cpu as t\nt._worker({world}, {ucml})\nprint('rank ok')\n")
    for rc, out in run_ranks(world, code, f"score_rank_shard_cpu {ucml}"):
        assert rc == 0 and "rank ok" in out, out
