"""CPU: RankingEvaluator's host side -- the CSR lists it builds, the users and batches it evaluates, and what it refuses
-- on the oracle-backed engine of tests/fake_engine.py, with a test-local score_rank that scatters the CSR rows into
dense masks and calls the oracle's metrics.  The kernel itself is checked on the GPU (tests/test_gpu_score_rank.py).
Each check runs in a subprocess because tests/fake_engine.install() re-routes the engine process-wide."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dense(uid, U, I, off, items):
    m = np.zeros((len(uid), I), bool)
    if off is None:
        return m
    off, items = off.numpy(), items.numpy()
    for b, u in enumerate(uid):
        if 0 <= u < U:
            r = items[off[u]:off[u + 1]]
            m[b, r[(r >= 0) & (r < I)]] = True
    return m


def _score_rank(self, kind, user_tab, uid, item_tab, item_bias, pos_off, pos_items, excl_off, excl_items, max_pos,
                at=(), scale=None):
    self.calls.append((uid.numpy().copy(), int(max_pos)))
    from oracle import openrec_oracle as O
    uid_np = uid.numpy().astype(np.int64)
    U, I = user_tab.shape[0], item_tab.shape[0]
    pred = self.score_all(kind, user_tab, uid, item_tab, item_bias, scale=scale).numpy()
    pos, excl = _dense(uid_np, U, I, pos_off, pos_items), _dense(uid_np, U, I, excl_off, excl_items)
    with np.errstate(all="ignore"):
        return (torch.from_numpy(O.auc(pos, pred, excl).astype(np.float32)),
                torch.from_numpy(O.ndcg(pos, pred, excl, tuple(at)).astype(np.float32)),
                torch.from_numpy(O.recall(pos, pred, excl, tuple(at)).astype(np.float32)))


def _install():
    import fake_engine
    eng = fake_engine.install()
    fake_engine.FakeEngine.score_rank = _score_rank
    eng.calls = []
    return eng


def _in_subprocess(check):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_evaluator_cpu as t\nt.{check}(t._install())\nprint('check ok')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "check ok" in r.stdout, r.stdout + r.stderr


def _dataset(pairs, U, I, **kw):
    from openrec_b200.tf2.data import Dataset
    raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
    if pairs:
        raw["user_id"], raw["item_id"] = np.array(pairs).T
    return Dataset(raw_data=raw, total_users=U, total_items=I, **kw)


def _rows(off, items):
    return [items[off[u]:off[u + 1]].tolist() for u in range(len(off) - 1)]


def test_csr_sorted_unique_union():
    _in_subprocess("_check_csr_sorted_unique_union")


def _check_csr_sorted_unique_union(fake):
    """Positives: sorted and unique per user, duplicated records counted once, users absent from the dataset empty.
    Exclusions: the union of several datasets' positives, sorted and unique; max_pos the longest positive row."""
    from openrec.tf2.metrics import RankingEvaluator
    U, I = 6, 20
    val = _dataset([(3, 9), (1, 4), (3, 2), (3, 9), (1, 0), (5, 19)], U, I)
    tr1 = _dataset([(1, 7), (3, 2), (0, 5)], U, I)
    tr2 = _dataset([(1, 4), (1, 7), (1, 1), (4, 3)], U, I)
    ev = RankingEvaluator(val, excl_datasets=[tr1, tr2], at=[5])
    assert _rows(ev.pos_off, ev.pos_items) == [[], [0, 4], [], [2, 9], [], [19]]
    assert _rows(ev.excl_off, ev.excl_items) == [[5], [1, 4, 7], [], [2], [3], []]
    assert ev.pos_off.dtype == np.int64 and ev.pos_items.dtype == np.int32 and ev.excl_off.dtype == np.int64
    assert ev.max_pos == 2
    assert ev.warm_users.tolist() == [3, 1, 5]                    # first appearance in the records


def test_warm_order_batches_and_metrics():
    _in_subprocess("_check_warm_order_batches_and_metrics")


def _check_warm_order_batches_and_metrics(fake):
    """evaluate() walks warm_users() in order, in batches of batch_size with a short last batch and the batch's own
    max_pos, and its per-user results equal the reference loop (evaluation stream masks + inference + AUC / NDCG /
    Recall)."""
    from openrec.tf2.metrics import AUC, NDCG, RankingEvaluator, Recall
    from openrec.tf2.recommenders import BPR
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(7)
    U, I, D = 40, 60, 8
    val_pairs = [(int(u), int(i)) for u in rng.permutation(U)[:23] for i in rng.choice(I, 1 + u % 4, replace=False)]
    tr_pairs = [(int(u), int(i)) for u in range(U) for i in rng.choice(I, 5, replace=False)]
    val, tr = _dataset(val_pairs, U, I), _dataset(tr_pairs, U, I)
    model = BPR(D, D, U, I)
    ev = RankingEvaluator(val, excl_datasets=[tr], at=[3, 10], batch_size=5)
    fake.calls.clear()
    res = ev.evaluate(model)
    warm = val.datastore.warm_users()
    assert len(warm) == 23
    assert [c[0].tolist() for c in fake.calls] == [warm[b:b + 5] for b in range(0, 23, 5)]
    lens = {u: len(val.datastore.get_positive_items(u)) for u in warm}
    assert [c[1] for c in fake.calls] == [max(lens[u] for u in warm[b:b + 5]) for b in range(0, 23, 5)]
    rows = list(_Streams.evaluation(val.datastore, [tr]))
    users = np.array([r["user_id"] for r in rows], np.int32)
    pos, excl = np.stack([r["pos_mask"] for r in rows]), np.stack([r["excl_mask"] for r in rows])
    pred = model.inference(users)
    np.testing.assert_array_equal(res["AUC"].numpy(), AUC(pos_mask=pos, pred=pred, excl_mask=excl).numpy())
    np.testing.assert_array_equal(res["NDCG"].numpy(),
                                  NDCG(pos_mask=pos, pred=pred, excl_mask=excl, at=[3, 10]).numpy())
    np.testing.assert_array_equal(res["Recall"].numpy(),
                                  Recall(pos_mask=pos, pred=pred, excl_mask=excl, at=[3, 10]).numpy())
    assert res["AUC"].numpy().shape == (23,) and res["NDCG"].numpy().shape == (23, 2)


def test_refusals():
    _in_subprocess("_check_refusals")


def _check_refusals(fake):
    """A dataset with explicit negatives ranks against its listed items only: NotImplementedError.  More than eight
    cut-offs: ValueError.  A model without full-catalogue operands (row-sharded): NotImplementedError."""
    from openrec.tf2.metrics import RankingEvaluator
    U, I = 5, 10
    with pytest.raises(NotImplementedError):
        RankingEvaluator(_dataset([(0, 1), (1, 2)], U, I, num_negatives=3))
    val = _dataset([(0, 1), (1, 2)], U, I)
    with pytest.raises(ValueError):
        RankingEvaluator(val, at=list(range(1, 10)))

    class NoOperands:
        pass
    with pytest.raises(NotImplementedError):
        RankingEvaluator(val).evaluate(NoOperands())


def test_engine_score_rank_signature():
    """Engine.score_rank's arguments, in the order the evaluator passes them."""
    from openrec_b200 import native as N
    params = list(inspect.signature(N.Engine.score_rank).parameters)
    assert params == ["self", "kind", "user_tab", "uid", "item_tab", "item_bias", "pos_off", "pos_items", "excl_off",
                      "excl_items", "max_pos", "at", "scale"]
