"""CPU, world size 2 and 3 over gloo: Retriever.recommend on a ShardedBPR / ShardedUCML runs the three phases of the
sharded top-K retrieval on every rank with an all-reduce between them, and the result equals the oracle top-K
(tests/topk_oracle.py) on the gathered tables.  The engine is the oracle-backed one of tests/fake_engine.py with a
test-local score_topk_shard that restates the phases in numpy (each rank keeps the k best keys of its own item rows,
the merge takes the k best non-zero keys of the summed lists), so this checks the decomposition and the collective
plumbing; the kernels are checked in tests/test_gpu_score_topk_shard.py."""
import os

import numpy as np
import pytest
import torch
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
M32 = np.uint64(0xFFFFFFFF)


def _scores(kind, urow, items, bias):
    """float32 scores of one user row against item rows, each computed in float64 and rounded once."""
    u, it = urow.astype(np.float64)[None, :], items.astype(np.float64)
    s = (u * it).sum(-1) if kind == 0 else -((u - it) ** 2).sum(-1)
    if bias is not None:
        s = s + bias.astype(np.float64)
    return s.astype(F32)


def _keys(s, ids):
    """The kernels' 64-bit keys: order-preserving score bits (-0.0 as +0.0) high, ~id low; '>' = the top-K order."""
    u = np.where(s == 0, F32(0), s).astype(F32).view(np.uint32).astype(np.uint64)
    u = np.where(u & np.uint64(0x80000000), ~u & M32, u | np.uint64(0x80000000))
    return (u << np.uint64(32)) | (~ids.astype(np.uint64) & M32)


def _decode(keys, k):
    items, scores = np.full(k, -1, np.int32), np.full(k, -np.inf, F32)
    n = len(keys)
    u = (keys >> np.uint64(32)).astype(np.uint32)
    scores[:n] = np.where(u & np.uint32(0x80000000), u & np.uint32(0x7FFFFFFF), ~u).view(F32)
    items[:n] = (~(keys & M32)).astype(np.uint32).view(np.int32)
    return items, scores


def _score_topk_shard(self, kind, phase, g, user, item, bias, uid, excl_off, excl_items, k, xrows, xkeys):
    R, r, U, I = g.world, g.rank, g.total_users, g.total_items
    uid = uid.numpy().astype(np.int64)
    Bu, D = len(uid), user.shape[1]
    keys = xkeys.numpy().view(np.uint64).reshape(Bu, R, k)
    if phase == 0:                   # this rank's user rows, 0 elsewhere
        out = np.zeros((Bu, D), F32)
        for b, u in enumerate(uid):
            if 0 <= u < U and u % R == r:
                out[b] = user.numpy()[u // R]
        xrows.copy_(torch.from_numpy(out.view(np.int32).reshape(-1)))
        return None
    if phase == 1:                   # this rank's k best keys in slot [b, r], 0 elsewhere
        rows = xrows.numpy().view(F32).reshape(Bu, D)
        mine = np.arange(g.local_items, dtype=np.int64) * R + r
        out = np.zeros((Bu, R, k), np.uint64)
        for b, u in enumerate(uid):
            s = _scores(kind, rows[b], item.numpy()[:g.local_items], None if bias is None else
                        bias.numpy()[:g.local_items])
            ok = ~np.isnan(s)
            if excl_off is not None and 0 <= u < U:
                eo = excl_off.numpy()
                ok &= ~np.isin(mine, excl_items.numpy()[eo[u]:eo[u + 1]])
            best = np.sort(_keys(s[ok], mine[ok]))[::-1][:k]
            out[b, r, :len(best)] = best
        keys[:] = out
        return None
    items, scores = np.empty((Bu, k), np.int32), np.empty((Bu, k), F32)   # phase 2: merge the ranks' lists
    for b in range(Bu):
        x = keys[b].reshape(-1)
        items[b], scores[b] = _decode(np.sort(x[x != 0])[::-1][:k], k)
    return torch.from_numpy(items), torch.from_numpy(scores)


def _worker(world, ucml):
    """One rank: sharded model, recommend, gather, compare on rank 0 with the oracle on the global tables; then ranks
    passing different numbers of ids all raise ValueError."""
    import torch.distributed as dist
    import fake_engine
    import topk_oracle as T
    fake_engine.FakeEngine.score_topk_shard = _score_topk_shard
    fake_engine.install()
    from openrec.tf2.data import Dataset
    from openrec.tf2.recommenders import Retriever, ShardedBPR, ShardedUCML
    rank = int(os.environ["RANK"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(19)
    U, I, D = 23, 61, 6                            # U, I not multiples of the world size
    tr = [(u, int(i)) for u in range(U) for i in rng.choice(I, int(rng.integers(0, 12)), replace=False)]
    tr += [(4, i) for i in range(I) if i % 9]      # a user with fewer than k eligible items
    raw = np.empty(len(tr), dtype=[("user_id", np.int32), ("item_id", np.int32)])
    raw["user_id"], raw["item_id"] = np.array(tr).T
    train = Dataset(raw_data=raw, total_users=U, total_items=I)
    model = (ShardedUCML if ucml else ShardedBPR)(D, D, U, I, seed=2)
    users = np.array(list(range(U)) + [4, 0, 4], np.int64)
    k = 10
    ret = Retriever(excl_datasets=[train], k=k, batch_size=7)
    items, scores = ret.recommend(model, users)
    got = [items.numpy(), scores.numpy().view(np.int32)]
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
                np.testing.assert_array_equal(x, y)
        user, item, bias = tabs
        kind = 1 if ucml else 0
        pred = np.stack([_scores(kind, user[u], item, bias[:, 0]) for u in users])
        excl = np.zeros((len(users), I), bool)
        for b, u in enumerate(users):
            excl[b, ret.excl_items[ret.excl_off[u]:ret.excl_off[u + 1]]] = True
        want = T.topk(pred, excl, k)
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1].view(np.int32))
        assert (got[0][4] == -1).any()              # user 4: at most 7 items left
    with pytest.raises(ValueError):
        ret.recommend(model, users[:5 + rank])
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("ucml", [False, True], ids=["bpr", "ucml"])
def test_sharded_retrieval_equals_oracle(world, ucml):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_score_topk_shard_cpu as t\nt._worker({world}, {ucml})\nprint('rank ok')\n")
    for rc, out in run_ranks(world, code, f"score_topk_shard_cpu {ucml}"):
        assert rc == 0 and "rank ok" in out, out
