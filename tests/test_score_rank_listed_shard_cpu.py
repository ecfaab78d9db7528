"""CPU, world size 2 and 3 over gloo: CandidateEvaluator.evaluate on a ShardedBPR / ShardedUCML runs the four phases
of the sharded listed-candidate evaluation on every rank with an all-reduce between them, and the result equals the
oracle's AUC / NDCG / Recall on the gathered tables with the masks of Dataset.evaluation.  The engine is the
oracle-backed one of tests/fake_engine.py with a test-local score_rank_listed_shard that restates the phases in numpy
(each rank counts over the listed items and positives it owns), so this checks the count decomposition and the
collective plumbing; the kernels are checked in tests/test_gpu_score_rank_listed_shard.py."""
import os

import numpy as np
import pytest
import torch
from _ranks import run_ranks
from test_score_rank_shard_cpu import _score_rank_shard, _scores, _sizes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _row(u, U, I, off, items):
    if off is None or not 0 <= u < U:
        return np.zeros(0, np.int64), 0
    r = items[off[u]:off[u + 1]].astype(np.int64)
    return r[(r >= 0) & (r < I)], len(r)


def _score_rank_listed_shard(self, kind, phase, g, user, item, bias, uid, pos_off, pos_items, neg_off, neg_items,
                             excl_off, excl_items, max_pos, xrows, xpred, xcnt, at=()):
    if phase < 2:                    # phases 0 and 1 are those of the catalogue evaluation
        return _score_rank_shard(self, kind, phase, g, user, item, bias, uid, pos_off, pos_items, excl_off,
                                 excl_items, max_pos, xrows, xpred, xcnt, at=at)
    R, r, U, I = g.world, g.rank, g.total_users, g.total_items
    uid = uid.numpy().astype(np.int64)
    Bu, D, P = len(uid), user.shape[1], max_pos + 1
    lists = [(o.numpy(), it.numpy()) if o is not None else (None, None)
             for o, it in ((pos_off, pos_items), (neg_off, neg_items), (excl_off, excl_items))]
    rows = xrows.numpy().view(F32).reshape(Bu, D)
    bias_np = None if bias is None else bias.numpy()
    item_np = item.numpy()

    def score(b, i):                 # an item this rank owns
        return _scores(kind, rows[b], item_np[i // R][None], None if bias_np is None else
                       bias_np[i // R:i // R + 1])[0]

    def parts(u):
        (p, raw), (n, _), (e, _) = (_row(u, U, I, *l) for l in lists)
        return p, n[~np.isin(n, p) & ~np.isin(n, e)], e, raw
    if phase == 2:                   # counts over the eval items and non-excluded positives this rank owns
        pred = xpred.numpy().view(F32).reshape(Bu, P)
        cnt = np.zeros((Bu, P), np.int64)
        for b, u in enumerate(uid):
            p, ev, e, raw = parts(u)
            if raw > max_pos or not len(p):
                continue
            n = len(p)
            pp = pred[b, :n]
            with np.errstate(all="ignore"):
                sp = np.exp(pp) * (~np.isin(p, e)).astype(F32)
            sp = np.where(np.isnan(sp), F32(np.inf), sp)
            s_ev = np.array([score(b, i) for i in ev if i % R == r], F32)
            s_pos = np.array([score(b, i) for i in p if i % R == r and i not in set(e.tolist())], F32)
            cnt[b, 0] = int(np.count_nonzero(pp[None, :] >= s_ev[:, None]))
            with np.errstate(all="ignore"):
                hits = np.exp(np.concatenate([s_ev, s_pos]))
                j = np.count_nonzero(np.sort(sp)[None, :] < hits[:, None], axis=1)
            cnt[b, 1:n + 1] = np.bincount(j, minlength=n + 1)[1:n + 1]
        xcnt.copy_(torch.from_numpy(cnt.reshape(-1)))
        return None
    cnt = xcnt.numpy().reshape(Bu, P)  # phase 3: the metrics from the summed counts, n_eval from the lists
    auc, ndcg, rec = (np.full(Bu, np.nan, F32), np.full((Bu, len(at)), np.nan, F32),
                      np.full((Bu, len(at)), np.nan, F32))
    for b, u in enumerate(uid):
        p, ev, _, raw = parts(u)
        if raw > max_pos:
            continue
        n = len(p)
        ranks = np.array([cnt[b, q + 1:n + 1].sum() for q in range(n)], np.int64).astype(F32)
        with np.errstate(all="ignore"):
            auc[b] = F32(cnt[b, 0]) / F32(n * len(ev))
            w = (F32(1) / (np.log(ranks + 2) / np.log(F32(2.0)))).astype(F32)
            for k, a in enumerate(at):
                ndcg[b, k] = (w * (ranks < a)).sum(dtype=F32)
                rec[b, k] = F32(np.count_nonzero(ranks < a)) / F32(n)
    return torch.from_numpy(auc), torch.from_numpy(ndcg), torch.from_numpy(rec)


def _worker(world, ucml):
    """One rank: sharded model, evaluate, gather, compare on rank 0 with the oracle on the global tables."""
    import torch.distributed as dist
    import fake_engine
    from oracle import openrec_oracle as O
    fake_engine.FakeEngine.score_rank_listed_shard = _score_rank_listed_shard
    fake_engine.FakeEngine.score_rank_shard_sizes = staticmethod(_sizes)
    fake_engine.install()
    from openrec.tf2.data import Dataset
    from openrec.tf2.metrics import CandidateEvaluator
    from openrec.tf2.recommenders import ShardedBPR, ShardedUCML
    from openrec_b200.tf2.data.dataset import _Streams
    rank = int(os.environ["RANK"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(17)
    U, I, D = 23, 61, 6                            # U, I not multiples of the world size
    va, tr = [], []
    for u in range(U):
        items = rng.choice(I, 30, replace=False)
        if u % 5:
            va += [(u, int(i), 1.0) for i in items[:1 + u % 4]]
            va += [(u, int(i), 0.0) for i in items[10:10 + int(rng.integers(0, 15))]]
        tr += [(u, int(i), 1.0) for i in items[4:4 + int(rng.integers(0, 12))]]   # some listed items excluded
    va.append((va[0][0], va[0][1], 0.0))           # a pair both positive and listed

    def mk(recs, **kw):
        raw = np.empty(len(recs), dtype=[("user_id", np.int32), ("item_id", np.int32), ("label", np.float32)])
        raw["user_id"], raw["item_id"], raw["label"] = np.array(recs, dtype=np.float64).T
        return Dataset(raw_data=raw, total_users=U, total_items=I, **kw)
    val, train = mk(va, implicit_negative=False), mk(tr)
    model = (ShardedUCML if ucml else ShardedBPR)(D, D, U, I, seed=2)
    at = [1, 5, 20]
    ev = CandidateEvaluator(val, excl_datasets=[train], at=at, batch_size=7)
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
        rows = list(_Streams.evaluation(val.datastore, [train]))
        users = np.array([r["user_id"] for r in rows])
        assert users.tolist() == ev.warm_users.tolist()
        pred = np.stack([_scores(kind, user[u], item, bias[:, 0]) for u in users])
        pos, excl = np.stack([r["pos_mask"] for r in rows]), np.stack([r["excl_mask"] for r in rows])
        with np.errstate(all="ignore"):
            want = O.auc(pos, pred, excl), O.ndcg(pos, pred, excl, tuple(at)), O.recall(pos, pred, excl, tuple(at))
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_allclose(got[1], want[1], rtol=1e-6)
        np.testing.assert_array_equal(got[2], want[2])
        assert len(users) > 14 and np.isfinite(got[0]).sum() > 8
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("ucml", [False, True], ids=["bpr", "ucml"])
def test_sharded_listed_evaluation_equals_oracle(world, ucml):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_score_rank_listed_shard_cpu as t\nt._worker({world}, {ucml})\nprint('rank ok')\n")
    for rc, out in run_ranks(world, code, f"score_rank_listed_shard_cpu {ucml}"):
        assert rc == 0 and "rank ok" in out, out
