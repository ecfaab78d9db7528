"""CPU: CandidateEvaluator's host side -- the CSR lists it builds, the users and batches it evaluates, and what it
refuses -- on the oracle-backed engine of tests/fake_engine.py, with a test-local score_rank_listed that restates the
contract of orx_score_rank_listed in numpy (the masks pos = P, excl = ~(P u L) u E, then the oracle's metrics).  The
kernel itself is checked on the GPU (tests/test_gpu_score_rank_listed.py).  Each check runs in a subprocess because
tests/fake_engine.install() re-routes the engine process-wide."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _row(u, U, I, off, items):
    if off is None or not 0 <= u < U:
        return np.zeros(0, np.int64)
    r = items.numpy()[off.numpy()[u]:off.numpy()[u + 1]].astype(np.int64)
    return r[(r >= 0) & (r < I)]


def _score_rank_listed(self, kind, user_tab, uid, item_tab, item_bias, pos_off, pos_items, neg_off, neg_items,
                       excl_off, excl_items, max_pos, at=(), scale=None):
    self.calls.append((uid.numpy().copy(), int(max_pos)))
    from oracle import openrec_oracle as O
    uid_np = uid.numpy().astype(np.int64)
    U, I = user_tab.shape[0], item_tab.shape[0]
    pred = self.score_all(kind, user_tab, uid, item_tab, item_bias, scale=scale).numpy()
    pos, excl = np.zeros((len(uid_np), I), bool), np.ones((len(uid_np), I), bool)
    for b, u in enumerate(uid_np):
        p, n, e = (_row(u, U, I, o, it) for o, it in ((pos_off, pos_items), (neg_off, neg_items),
                                                       (excl_off, excl_items)))
        pos[b, p] = True
        excl[b, p] = excl[b, n] = False
        excl[b, e] = True
    with np.errstate(all="ignore"):
        return (torch.from_numpy(O.auc(pos, pred, excl).astype(np.float32)),
                torch.from_numpy(O.ndcg(pos, pred, excl, tuple(at)).astype(np.float32)),
                torch.from_numpy(O.recall(pos, pred, excl, tuple(at)).astype(np.float32)))


def _install():
    import fake_engine
    eng = fake_engine.install()
    fake_engine.FakeEngine.score_rank_listed = _score_rank_listed
    eng.calls = []
    return eng


def _in_subprocess(check):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_candidate_evaluator_cpu as t\nt.{check}(t._install())\nprint('check ok')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "check ok" in r.stdout, r.stdout + r.stderr


def _dataset(recs, U, I, **kw):
    from openrec_b200.tf2.data import Dataset
    raw = np.empty(len(recs), dtype=[("user_id", np.int32), ("item_id", np.int32), ("label", np.float32)])
    if recs:
        raw["user_id"], raw["item_id"], raw["label"] = np.array(recs, dtype=np.float64).T
    return Dataset(raw_data=raw, total_users=U, total_items=I, **kw)


def _rows(off, items):
    return [items[off[u]:off[u + 1]].tolist() for u in range(len(off) - 1)]


def _check_against_reference_loop(fake, labelled):
    from openrec.tf2.metrics import AUC, NDCG, CandidateEvaluator, Recall
    from openrec.tf2.recommenders import BPR
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(7)
    U, I, D = 40, 60, 8
    val_recs = []
    for u in rng.permutation(U)[:23]:
        items = rng.choice(I, 20, replace=False)
        val_recs += [(int(u), int(i), 1.0) for i in items[:1 + u % 4]]
        if labelled:
            val_recs += [(int(u), int(i), 0.0) for i in items[5:5 + int(rng.integers(0, 12))]]
    if labelled:
        val_recs.append((val_recs[0][0], val_recs[0][1], 0.0))     # one pair both positive and negative
    tr = _dataset([(int(u), int(i), 1.0) for u in range(U) for i in rng.choice(I, 5, replace=False)], U, I)
    np.random.seed(3)
    val = (_dataset(val_recs, U, I, implicit_negative=False) if labelled
           else _dataset(val_recs, U, I, num_negatives=10))
    model = BPR(D, D, U, I)
    ev = CandidateEvaluator(val, excl_datasets=[tr], at=[3, 10], batch_size=5)
    fake.calls.clear()
    res = ev.evaluate(model)
    store = val.datastore
    warm = store.warm_users()
    assert len(warm) == 23 and ev.warm_users.tolist() == warm
    assert [c[0].tolist() for c in fake.calls] == [warm[b:b + 5] for b in range(0, 23, 5)]
    lens = {u: len(store.get_positive_items(u)) for u in warm}
    assert [c[1] for c in fake.calls] == [max(lens[u] for u in warm[b:b + 5]) for b in range(0, 23, 5)]
    listed = _rows(ev.neg_off, ev.neg_items)
    for u in range(U):
        assert listed[u] == (sorted(set(store.get_negative_items(u))) if u in set(warm) else [])
    if labelled:
        u, i = val_recs[0][0], val_recs[0][1]
        assert i in listed[u] and i in _rows(ev.pos_off, ev.pos_items)[u]
    rows = list(_Streams.evaluation(store, [tr]))
    users = np.array([r["user_id"] for r in rows], np.int32)
    pos, excl = np.stack([r["pos_mask"] for r in rows]), np.stack([r["excl_mask"] for r in rows])
    pred = model.inference(users)
    np.testing.assert_array_equal(res["AUC"].numpy(), AUC(pos_mask=pos, pred=pred, excl_mask=excl).numpy())
    np.testing.assert_array_equal(res["NDCG"].numpy(),
                                  NDCG(pos_mask=pos, pred=pred, excl_mask=excl, at=[3, 10]).numpy())
    np.testing.assert_array_equal(res["Recall"].numpy(),
                                  Recall(pos_mask=pos, pred=pred, excl_mask=excl, at=[3, 10]).numpy())
    assert res["AUC"].numpy().shape == (23,) and res["NDCG"].numpy().shape == (23, 2)
    assert np.isfinite(res["AUC"].numpy()).sum() > 15


def _check_num_negatives(fake):
    _check_against_reference_loop(fake, labelled=False)


def _check_labelled(fake):
    _check_against_reference_loop(fake, labelled=True)


@pytest.mark.parametrize("check", ["_check_num_negatives", "_check_labelled"])
def test_warm_order_batches_and_metrics(check):
    """evaluate() walks warm_users() in order, in batches of batch_size with a short last batch and the batch's own
    max_pos; the listed CSR is get_negative_items of the warm users; the results equal the reference loop (evaluation
    stream masks + inference + AUC / NDCG / Recall), for drawn negatives and for labelled ones with a pair that is
    both positive and negative."""
    _in_subprocess(check)


def test_refusals():
    _in_subprocess("_check_refusals")


def _check_refusals(fake):
    """No listed negatives: ValueError naming RankingEvaluator.  More than eight cut-offs: ValueError.  A model
    without operands: NotImplementedError.  RankingEvaluator still refuses explicit negatives."""
    from openrec.tf2.metrics import CandidateEvaluator, RankingEvaluator
    U, I = 5, 10
    with pytest.raises(ValueError, match="RankingEvaluator"):
        CandidateEvaluator(_dataset([(0, 1, 1.0), (1, 2, 1.0)], U, I))
    val = _dataset([(0, 1, 1.0), (1, 2, 1.0)], U, I, num_negatives=3)
    with pytest.raises(ValueError):
        CandidateEvaluator(val, at=list(range(1, 10)))
    with pytest.raises(NotImplementedError, match="CandidateEvaluator"):
        RankingEvaluator(val)

    class NoOperands:
        pass
    with pytest.raises(NotImplementedError):
        CandidateEvaluator(val).evaluate(NoOperands())


def test_engine_score_rank_listed_signature():
    """Engine.score_rank_listed's arguments, in the order the evaluator passes them."""
    from openrec_b200 import native as N
    params = list(inspect.signature(N.Engine.score_rank_listed).parameters)
    assert params == ["self", "kind", "user_tab", "uid", "item_tab", "item_bias", "pos_off", "pos_items", "neg_off",
                      "neg_items", "excl_off", "excl_items", "max_pos", "at", "scale"]
    shard = list(inspect.signature(N.Engine.score_rank_listed_shard).parameters)
    assert shard == ["self", "kind", "phase", "g", "user_shard", "item_shard", "bias_shard", "uid", "pos_off",
                     "pos_items", "neg_off", "neg_items", "excl_off", "excl_items", "max_pos", "xrows", "xpred",
                     "xcnt", "at"]
