"""CPU: the top-K oracle on hand-made cases, and Retriever's host side -- the exclusion CSR it builds, the chunks it
sends, what it refuses -- on the oracle-backed engine of tests/fake_engine.py, with a test-local score_topk that
scatters the CSR rows into a dense mask and calls the oracle.  The kernel itself is checked on the GPU
(tests/test_gpu_score_topk.py).  Engine checks run in a subprocess because tests/fake_engine.install() re-routes the
engine process-wide."""
import inspect
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import topk_oracle as T  # noqa: E402

F32 = np.float32


# ---- the oracle -------------------------------------------------------------------------------------------------------
def test_oracle_ties_by_ascending_id():
    pred = np.array([[1, 3, 3, 2, 3]], F32)
    items, scores = T.topk(pred, None, 4)
    assert items.tolist() == [[1, 2, 4, 3]]
    assert scores.tolist() == [[3, 3, 3, 2]]


def test_oracle_nan_never_returned_and_signed_zero_ties():
    pred = np.array([[np.nan, 0.0, -0.0, np.nan, -np.inf, -0.0]], F32)
    items, scores = T.topk(pred, None, 6)
    assert items.tolist() == [[1, 2, 5, 4, -1, -1]]          # -0.0 == +0.0: ascending id; -inf is a valid score
    assert np.signbit(scores[0, 1]) and not np.signbit(scores[0, 0])
    assert np.isneginf(scores[0, 3:]).all()


def test_oracle_exclusions_padding_and_k_above_I():
    pred = np.array([[5, 4, 3], [1, 2, 3]], F32)
    excl = np.array([[1, 0, 1], [0, 0, 0]], bool)
    items, scores = T.topk(pred, excl, 5)
    assert items.tolist() == [[1, -1, -1, -1, -1], [2, 1, 0, -1, -1]]
    assert scores[0, 0] == 4 and np.isneginf(scores[0, 1:]).all() and np.isneginf(scores[1, 3:]).all()
    assert scores.dtype == np.float32 and items.dtype == np.int32


def test_oracle_k1_is_argmax_with_lowest_id():
    rng = np.random.default_rng(3)
    pred = rng.integers(0, 4, (50, 30)).astype(F32)
    items, _ = T.topk(pred, None, 1)
    np.testing.assert_array_equal(items[:, 0], pred.argmax(1))   # argmax returns the first maximum


# ---- Retriever's host logic on the oracle-backed engine ---------------------------------------------------------------
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


def _score_topk(self, kind, user_tab, uid, item_tab, item_bias, excl_off, excl_items, k, scale=None):
    self.calls.append((uid.numpy().copy(), int(k)))
    uid_np = uid.numpy().astype(np.int64)
    U, I = user_tab.shape[0], item_tab.shape[0]
    pred = self.score_all(kind, user_tab, uid, item_tab, item_bias, scale=scale).numpy()
    items, scores = T.topk(pred, _dense(uid_np, U, I, excl_off, excl_items), k)
    return torch.from_numpy(items), torch.from_numpy(scores)


def _install():
    import fake_engine
    eng = fake_engine.install()
    fake_engine.FakeEngine.score_topk = _score_topk
    eng.calls = []
    return eng


def _in_subprocess(check):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_retriever_cpu as t\nt.{check}(t._install())\nprint('check ok')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "check ok" in r.stdout, r.stdout + r.stderr


def _dataset(pairs, U, I):
    from openrec_b200.tf2.data import Dataset
    raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
    if pairs:
        raw["user_id"], raw["item_id"] = np.array(pairs).T
    return Dataset(raw_data=raw, total_users=U, total_items=I)


def _rows(off, items):
    return [items[off[u]:off[u + 1]].tolist() for u in range(len(off) - 1)]


def test_exclusion_csr_is_union_of_positives():
    _in_subprocess("_check_exclusion_csr")


def _check_exclusion_csr(fake):
    """The union of several datasets' positives, sorted and unique per user, duplicated records counted once, users
    absent everywhere empty; no datasets: nothing excluded."""
    from openrec.tf2.recommenders import Retriever
    U, I = 6, 20
    tr1 = _dataset([(1, 7), (3, 2), (0, 5), (3, 2)], U, I)
    tr2 = _dataset([(1, 4), (1, 7), (1, 1), (4, 3)], U, I)
    r = Retriever(excl_datasets=[tr1, tr2], k=3)
    assert _rows(r.excl_off, r.excl_items) == [[5], [1, 4, 7], [], [2], [3], []]
    assert r.excl_off.dtype == np.int64 and r.excl_items.dtype == np.int32
    none = Retriever(k=3)
    assert none.excl_off is None and none.excl_items is None


def test_chunks_and_results():
    _in_subprocess("_check_chunks_and_results")


def _check_chunks_and_results(fake):
    """recommend() flattens user_id (any shape, host or tensor), sends chunks of batch_size with a short last chunk,
    and its results equal model.inference plus the oracle top-K on the evaluation stream's exclusion masks."""
    from openrec.tf2.recommenders import BPR, Retriever
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(11)
    U, I, D = 30, 50, 8
    tr = _dataset([(int(u), int(i)) for u in range(U) for i in rng.choice(I, 1 + u % 7, replace=False)], U, I)
    model = BPR(D, D, U, I)
    r = Retriever(excl_datasets=[tr], k=7, batch_size=4)
    users = rng.integers(0, U, (3, 6)).astype(np.int64)
    fake.calls.clear()
    items, scores = r.recommend(model, users)
    flat = users.reshape(-1)
    assert [c[0].tolist() for c in fake.calls] == [flat[b:b + 4].tolist() for b in range(0, 18, 4)]
    assert all(c[1] == 7 for c in fake.calls)
    assert items.numpy().shape == (18, 7) and scores.numpy().shape == (18, 7)
    excl = {row["user_id"]: row["excl_mask"] for row in _Streams.evaluation(tr.datastore, [tr])}
    pred = model.inference(flat.astype(np.int32)).numpy()
    want_i, want_s = T.topk(pred, np.stack([excl[int(u)] for u in flat]), 7)
    np.testing.assert_array_equal(items.numpy(), want_i)
    np.testing.assert_array_equal(scores.numpy(), want_s)
    fake.calls.clear()
    again = r.recommend(model, torch.from_numpy(flat))
    np.testing.assert_array_equal(again[0].numpy(), want_i)
    assert len(fake.calls) == 5
    e_items, e_scores = r.recommend(model, np.zeros(0, np.int64))
    assert e_items.numpy().shape == (0, 7) and e_scores.numpy().shape == (0, 7)


def test_refusals():
    _in_subprocess("_check_refusals")


def _check_refusals(fake):
    """k outside [1, ORX_MAX_TOPK] and a non-positive batch size: ValueError.  Datasets with different total_users:
    ValueError.  DLRM and models without whole-table operands: NotImplementedError."""
    from openrec.tf2.recommenders import DLRM, Retriever
    from openrec_b200._lib import ORX_MAX_TOPK
    U, I = 5, 10
    for k in (0, -1, ORX_MAX_TOPK + 1):
        with pytest.raises(ValueError):
            Retriever(k=k)
    Retriever(k=ORX_MAX_TOPK)
    with pytest.raises(ValueError):
        Retriever(batch_size=0)
    with pytest.raises(ValueError):
        Retriever(excl_datasets=[_dataset([(0, 1)], U, I), _dataset([(0, 1)], U + 1, I)])
    r = Retriever(excl_datasets=[_dataset([(0, 1)], U, I)])
    with pytest.raises(NotImplementedError):
        r.recommend(DLRM.__new__(DLRM), [0])

    class NoOperands:
        pass
    with pytest.raises(NotImplementedError):
        r.recommend(NoOperands(), [0])


def test_engine_score_topk_signature():
    """Engine.score_topk's arguments, in the order Retriever passes them."""
    from openrec_b200 import native as N
    params = list(inspect.signature(N.Engine.score_topk).parameters)
    assert params == ["self", "kind", "user_tab", "uid", "item_tab", "item_bias", "excl_off", "excl_items", "k",
                      "scale"]
