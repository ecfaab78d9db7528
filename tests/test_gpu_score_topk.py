"""GPU parity of the fused catalogue top-K retrieval (orx_score_topk, openrec_b200/csrc/orx_eval.cu) and of
openrec.tf2.recommenders.Retriever.

The reference throughout is orx_score_all on the same inputs followed by the numpy top-K of tests/topk_oracle.py on the
dense exclusion masks the CSR rows describe.  The fused kernel computes every score by the chain of k_score_all, so the
items must be equal and the scores bit-equal (a -0.0 may come back as +0.0)."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import topk_oracle as T  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
KINDS = [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST]


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


class Problem:
    """Tables, per-user exclusion CSR rows (sorted, unique, possibly with the ignored entries -1 and I; None: no lists)
    and a batch of uids."""

    def __init__(self, kind, user, item, bias, scale, excl_rows, uid):
        self.kind, self.U, self.I, self.D = kind, len(user), len(item), item.shape[1]
        self.user, self.item = dev(user), dev(item)
        self.bias = None if bias is None else dev(bias)
        self.scale = None if scale is None else dev(scale)
        self.excl_rows = excl_rows
        self.uid = np.asarray(uid, np.int64)
        self.excl_off, self.excl_items = self._csr(excl_rows) if excl_rows is not None else (None, None)

    def _csr(self, rows):
        lens = np.array([len(rows.get(u, ())) for u in range(self.U)], np.int64)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        items = np.concatenate([np.asarray(rows.get(u, ()), np.int64) for u in range(self.U)] + [np.zeros(0)])
        return dev(off, torch.int64), dev(items.astype(np.int32), torch.int32)

    def mask(self, uid=None):
        uid = self.uid if uid is None else uid
        m = np.zeros((len(uid), self.I), bool)
        for b, u in enumerate(uid):
            if self.excl_rows is not None and 0 <= u < self.U:
                r = np.asarray(self.excl_rows.get(int(u), ()), np.int64)
                m[b, r[(r >= 0) & (r < self.I)]] = True
        return m

    def fused(self, eng, k, uid=None):
        uid = self.uid if uid is None else uid
        it, sc = eng.score_topk(self.kind, self.user, dev(uid, torch.int32), self.item, self.bias, self.excl_off,
                                self.excl_items, k, scale=self.scale)
        return it.cpu().numpy(), sc.cpu().numpy()

    def reference(self, eng, k, uid=None):
        uid = self.uid if uid is None else uid
        pred = eng.score_all(self.kind, self.user, dev(uid, torch.int32), self.item, self.bias, scale=self.scale)
        return T.topk(pred.cpu().numpy(), self.mask(uid), k)


def bits(s):
    s = np.where(s == 0, F32(0), s).astype(F32)      # -0.0 and +0.0 compare equal
    return s.view(np.int32)


def check(got, want, what=""):
    np.testing.assert_array_equal(got[0], want[0], err_msg=f"items {what}")
    np.testing.assert_array_equal(bits(got[1]), bits(want[1]), err_msg=f"score bits {what}")


def check_prefix(got, want, k, what=""):
    """want computed at a k' >= k: its first k columns are the answer at k."""
    check(got, (want[0][:, :k], want[1][:, :k]), f"k={k} {what}")


def last_dispatch(eng, pb, k, Bu=None):
    rec = [r for r in eng.debug_dispatch_log() if r.op == L.ORX_OP_SCORE_TOPK]
    assert rec, "no orx_score_topk record"
    r = rec[-1]
    assert r.variant == L.ORX_VARIANT_TOPK and r.ta == pb.kind and r.tb == k
    assert (r.m, r.n, r.k) == (len(pb.uid) if Bu is None else Bu, pb.I, pb.D) and r.s >= 1
    return r


def make_problem(rng, kind, Bu, I, D, scaled=False, biased=True, maxe=60, U=None, ties=True):
    """Random tables; users get up to maxe exclusions, a few rows carry the ignored entries -1 and I.  With ties: item
    rows (and biases) copied from other items -- exact ties that must resolve by ascending id -- some one ulp away."""
    U = U or max(3, Bu // 2 + 2)
    user = rng.uniform(-1, 1, (U, D)).astype(F32)
    item = rng.uniform(-1, 1, (I, D)).astype(F32)
    bias = rng.uniform(-1, 1, I).astype(F32)
    scale = rng.uniform(-2, 2, D).astype(F32) if scaled else None
    excl_rows = {}
    for u in range(U):
        e = set(rng.choice(I, min(I, int(rng.integers(0, maxe + 1))), replace=False).tolist())
        if rng.random() < 0.2:
            e |= {-1, I}
        excl_rows[u] = sorted(e)
    if ties and I > 4:
        n = max(1, min(I // 4, 2000))
        for j, s in zip(rng.choice(I, n, replace=False), rng.choice(I, n)):
            if j == s:
                continue
            item[j], bias[j] = item[s], bias[s]
            if rng.random() < 0.3:
                c = rng.integers(0, D)
                item[j, c] = np.nextafter(item[j, c], F32(np.inf) if rng.random() < 0.5 else F32(-np.inf))
    uid = rng.integers(0, U, Bu)
    where = rng.permutation(Bu)[:4]
    uid[where] = np.array([-1, U, 0, 0])[:len(where)]        # bad uids and a duplicate
    return Problem(kind, user, item, bias if biased else None, scale, excl_rows, uid)


def ks_for(I):
    return sorted({k for k in (1, 10, 100, L.ORX_MAX_TOPK, I, I + 5) if 1 <= k <= L.ORX_MAX_TOPK})


# (Bu, I, D): tile edges at 128 users / 128 items, D below, at and above the chunk of 8, item splits that do not divide
# the tile count (I = 100 003: 782 item tiles)
SHAPES = [(1, 1, 1), (127, 129, 7), (129, 16980, 50), (129, 100003, 128), (1000, 127, 1)]
VARIANTS = [(False, True), (True, True), (False, False), (True, False)]   # (scale, bias)


@pytest.mark.parametrize("Bu,I,D", SHAPES)
@pytest.mark.parametrize("scaled,biased", VARIANTS, ids=["plain", "scale", "nobias", "scale-nobias"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_topk_equals_score_all_oracle(eng, kind, scaled, biased, Bu, I, D):
    """Items equal, scores bit-equal, at k = 1, 10, 100, ORX_MAX_TOPK, I and I + 5 (where <= ORX_MAX_TOPK), with exact
    ties, one-ulp neighbours, bad uids, a duplicate uid and ignored list entries."""
    rng = np.random.default_rng(seed_of(kind, scaled, biased, Bu, I, D))
    pb = make_problem(rng, kind, Bu, I, D, scaled=scaled, biased=biased)
    ks = ks_for(I)
    want = pb.reference(eng, max(ks))
    for k in ks:
        check_prefix(pb.fused(eng, k), want, k)
        last_dispatch(eng, pb, k)


@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_special_values_and_exclusions(eng, kind):
    """NaN biases (never returned), +-inf biases, zero scores of both signs, exclusion rows that leave fewer than k
    items (padding), list entries -1 and I, duplicate uids, uids -1 and U; then the same users with excl_off = NULL."""
    rng = np.random.default_rng(seed_of("special", kind))
    U, I, D = 8, 300, 16
    user = rng.uniform(-1, 1, (U, D)).astype(F32)
    item = rng.uniform(-1, 1, (I, D)).astype(F32)
    bias = rng.uniform(-1, 1, I).astype(F32)
    bias[rng.choice(I, 30, replace=False)] = np.nan
    bias[rng.choice(I, 10, replace=False)] = np.inf
    bias[rng.choice(I, 10, replace=False)] = -np.inf
    zero = rng.choice(I, 40, replace=False)
    item[zero] = 0.0
    bias[zero] = np.where(np.arange(40) % 2, F32(-0.0), F32(0.0))
    user[3] = 0.0                                             # with DOT: exact zeros of both bias signs
    allI = list(range(I))
    excl = {0: allI[5:], 1: [-1] + allI[:290] + [I], 2: [], 3: [-1, 5, 6, I], 4: allI, 5: [7]}
    uid = [0, 1, 2, 3, 4, 4, -1, U, 1, 2, 5, 6, 3]
    pb = Problem(kind, user, item, bias, None, excl, uid)
    for k in (1, 7, 50, 400):
        got, want = pb.fused(eng, k), pb.reference(eng, k)
        check(got, want, f"k={k}")
        last_dispatch(eng, pb, k)
        assert not np.isnan(got[1]).any()
        assert (got[0][4] == -1).all() and np.isneginf(got[1][4]).all()          # everything excluded
    got = pb.fused(eng, 400)
    assert (got[0][0][5 - int(np.isnan(bias[:5]).sum()):] == -1).all()         # 5 items at most
    pb_noex = Problem(kind, user, item, bias, None, None, uid)
    for k in (10, 400):
        check(pb_noex.fused(eng, k), pb_noex.reference(eng, k), f"no exclusions k={k}")


def test_bad_uid_dot_without_bias_is_first_k_items(eng):
    """A uid outside [0, U) under DOT without bias scores 0 everywhere: the answer is items 0 .. k-1 (ties by id)."""
    rng = np.random.default_rng(seed_of("zero"))
    pb = Problem(N.ORX_SCORE_DOT, rng.uniform(-1, 1, (4, 32)).astype(F32), rng.uniform(-1, 1, (5000, 32)).astype(F32),
                 None, None, None, [-1, 4, 7])
    for k in (1, 100, L.ORX_MAX_TOPK):
        items, scores = pb.fused(eng, k)
        assert (items == np.arange(k)).all() and (scores == 0).all()
        check((items, scores), pb.reference(eng, k))


@pytest.mark.parametrize("order", ["rising", "falling"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_adversarial_orders(eng, kind, order):
    """Scores rising with item id (every item beats the threshold, every tile compacts every row) and falling (the
    first tile fills the lists, later ones append nothing)."""
    rng = np.random.default_rng(seed_of("order", kind, order))
    U, I, D, Bu = 200, 100003, 32, 129
    user = rng.uniform(-1e-3, 1e-3, (U, D)).astype(F32)
    item = rng.uniform(-1e-3, 1e-3, (I, D)).astype(F32)
    ramp = np.arange(I, dtype=F32) * F32(1e-2)
    bias = ramp if order == "rising" else ramp[::-1].copy()
    excl = {u: sorted(rng.choice(I, 50, replace=False).tolist()) for u in range(U)}
    pb = Problem(kind, user, item, bias, None, excl, rng.integers(0, U, Bu))
    want = pb.reference(eng, L.ORX_MAX_TOPK)
    for k in (1, 100, L.ORX_MAX_TOPK):
        check_prefix(pb.fused(eng, k), want, k, order)
        last_dispatch(eng, pb, k)


def test_independent_of_splits_batch_and_handle(eng):
    """A row computed alone (Bu = 1: many item splits) equals the same row inside Bu = 1000 (few splits); two calls on
    one handle and one on a fresh handle give identical bits; a large call followed by a small one is correct."""
    rng = np.random.default_rng(seed_of("independence"))
    pb = make_problem(rng, N.ORX_SCORE_DOT, 1000, 100003, 64)
    k = 100
    big = pb.fused(eng, k)
    splits_big = last_dispatch(eng, pb, k).s
    want = pb.reference(eng, k)
    check(big, want, "Bu=1000")
    for b in (0, 1, 517, 999):
        alone = pb.fused(eng, k, uid=pb.uid[b:b + 1])
        r = last_dispatch(eng, pb, k, Bu=1)
        assert r.s > splits_big
        np.testing.assert_array_equal(alone[0], big[0][b:b + 1])
        np.testing.assert_array_equal(alone[1].view(np.int32), big[1][b:b + 1].view(np.int32))
    again = pb.fused(eng, k)
    assert np.array_equal(again[0], big[0]) and np.array_equal(again[1].view(np.int32), big[1].view(np.int32))
    small = make_problem(rng, N.ORX_SCORE_NEG_SQDIST, 130, 3000, 24, scaled=True)
    first = small.fused(eng, 33)
    check(first, small.reference(eng, 33), "small after large")
    fresh = N.Engine(torch.cuda.current_device())
    try:
        for p, kk, ref in ((small, 33, first), (pb, k, big)):
            it, sc = fresh.score_topk(p.kind, p.user, dev(p.uid, torch.int32), p.item, p.bias, p.excl_off,
                                      p.excl_items, kk, scale=p.scale)
            torch.cuda.synchronize()
            assert np.array_equal(it.cpu().numpy(), ref[0])
            assert np.array_equal(sc.cpu().numpy().view(np.int32), ref[1].view(np.int32))
    finally:
        torch.cuda.synchronize()
        fresh.close()


def test_scores_may_be_null(eng):
    """top_scores = NULL through the C-ABI: the items are those of the full call."""
    import ctypes as C
    rng = np.random.default_rng(seed_of("null-scores"))
    pb = make_problem(rng, N.ORX_SCORE_DOT, 40, 2000, 16)
    k = 25
    want = pb.fused(eng, k)
    uid = dev(pb.uid, torch.int32)
    items = torch.full((40, k), -7, dtype=torch.int32, device="cuda")
    L.check(eng.lib.orx_score_topk(eng.h, pb.kind, C.c_void_p(pb.user.data_ptr()), pb.U, C.c_void_p(uid.data_ptr()),
                                   40, None, C.c_void_p(pb.item.data_ptr()), C.c_void_p(pb.bias.data_ptr()), pb.I,
                                   pb.D, C.c_void_p(pb.excl_off.data_ptr()), C.c_void_p(pb.excl_items.data_ptr()), k,
                                   C.c_void_p(items.data_ptr()), None, eng.stream()))
    np.testing.assert_array_equal(items.cpu().numpy(), want[0])
    for bad_k in (0, L.ORX_MAX_TOPK + 1):
        with pytest.raises(ValueError):
            eng.score_topk(pb.kind, pb.user, uid, pb.item, pb.bias, pb.excl_off, pb.excl_items, bad_k)
    empty = eng.score_topk(pb.kind, pb.user, uid[:0], pb.item, pb.bias, pb.excl_off, pb.excl_items, k)
    assert empty[0].shape == (0, k)


def test_retrieval_between_prefetch_and_step(eng):
    """An orx_score_topk call (which grows the evaluation scratch on first use) issued between orx_pairwise_prefetch and
    the step that consumes the prefetch: the step still uses the prefetched index and its tables and outputs are
    bit-identical to the same sequence without the retrieval.  Every row appears once in the batch, so the step itself
    has no float atomics and is bit-reproducible."""
    rng = np.random.default_rng(seed_of("prefetch"))
    U, I, D, B = 5000, 10000, 64, 2048
    init = [rng.uniform(-0.1, 0.1, s).astype(F32) for s in ((U, D), (I, D), (I, 1))]
    items = rng.permutation(I)[:2 * B].astype(np.int32)
    ids = [rng.permutation(U)[:B].astype(np.int32), items[:B], items[B:]]
    pb = make_problem(rng, N.ORX_SCORE_DOT, 700, 40000, 64)

    def run(with_topk, e):
        tabs = [dev(a) for a in init]
        acc = [torch.full_like(t, 0.1) for t in tabs]
        tt = [N.table(t, s) for t, s in zip(tabs, acc)]
        d = [dev(x, torch.int32) for x in ids]
        out4 = torch.zeros(4, device="cuda")
        torch.cuda.synchronize()
        e.debug_dispatch_log()
        e.pairwise_prefetch(tt[0], tt[1], *d, L.ORX_OPT_ADAGRAD, ids_ready=True)
        if with_topk:
            pb.fused(e, L.ORX_MAX_TOPK)
        e.pairwise_step(N.ORX_PAIR_BPR, *tt, *d, N.opt(L.ORX_OPT_ADAGRAD, 0.05), out4)
        rec = [r for r in e.debug_dispatch_log() if r.op == L.ORX_OP_PAIRWISE_STEP]
        assert len(rec) == 1 and rec[0].s in (1, 2), rec
        torch.cuda.synchronize()
        return [t.cpu().numpy().view(np.int32) for t in tabs + acc + [out4]]

    fresh = N.Engine(torch.cuda.current_device())
    try:
        want = run(False, fresh)
        got = run(True, fresh)
    finally:
        torch.cuda.synchronize()
        fresh.close()
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_bench_shape(eng):
    """I = 1 000 000, D = 128, Bu = 256, k = 100, exclusions ~ Poisson(100) per user."""
    rng = np.random.default_rng(seed_of("bench"))
    I, D, Bu, U = 1_000_000, 128, 256, 256
    user = rng.uniform(-0.1, 0.1, (U, D)).astype(F32)
    item = rng.uniform(-0.1, 0.1, (I, D)).astype(F32)
    bias = rng.uniform(-0.1, 0.1, I).astype(F32)
    excl = {u: sorted(rng.choice(I, rng.poisson(100), replace=False).tolist()) for u in range(U)}
    pb = Problem(N.ORX_SCORE_DOT, user, item, bias, None, excl, rng.permutation(U)[:Bu])
    check(pb.fused(eng, 100), pb.reference(eng, 100))
    last_dispatch(eng, pb, 100)


# ---- end to end through openrec.tf2 -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


@pytest.mark.parametrize("model_name", ["bpr", "ucml", "gmf", "wrmf"])
def test_retriever_end_to_end(tf, model_name):
    """Retriever.recommend(model, users) at the example's shape (U = 1 200, I = 16 980, D = 50, the train dataset
    excluded, weights on a dyadic grid so that ties are common) against model.inference plus the oracle top-K on the
    exclusion masks of the evaluation stream."""
    from openrec.tf2.data import Dataset
    from openrec.tf2.recommenders import BPR, GMF, UCML, WRMF, Retriever
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(seed_of("e2e-retriever", model_name))
    U, I, D = 1200, 16980, 50
    pairs = [(u, int(i)) for u in range(U) if u % 11 for i in rng.choice(I, int(rng.integers(1, 41)), replace=False)]
    raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
    raw["user_id"], raw["item_id"] = np.array(pairs).T
    train = Dataset(raw_data=raw, total_users=U, total_items=I)
    cls = {"bpr": BPR, "ucml": UCML, "gmf": GMF, "wrmf": WRMF}[model_name]
    model = cls(D, D, U, I)
    model.user_latent_factor.embeddings.assign((rng.integers(-2, 3, (U, D)) / 8).astype(F32))
    model.item_latent_factor.embeddings.assign((rng.integers(-2, 3, (I, D)) / 8).astype(F32))
    model.item_bias.embeddings.assign((rng.integers(-64, 65, (I, 1)) / 64).astype(F32))
    if model_name == "gmf":
        model.mlp.layers[0].kernel.assign((rng.integers(-8, 9, (D, 1)) / 8).astype(F32))
    k = 100
    ret = Retriever(excl_datasets=[train], k=k, batch_size=256)
    rows = list(_Streams.evaluation(train.datastore, [train]))
    users = np.array([r["user_id"] for r in rows], np.int32)
    items, scores = ret.recommend(model, users.astype(np.int64)[:, None])          # host ids, flattened
    items, scores = items.numpy(), scores.numpy()
    assert items.shape == (len(users), k)
    pred = model.inference(users).numpy()
    want = T.topk(pred, np.stack([r["excl_mask"] for r in rows]), k)
    check((items, scores), want, model_name)
    seen = {u: set(train.datastore.get_positive_items(u)) for u in users[:50].tolist()}
    assert all(not seen[u] & set(items[b].tolist()) for b, u in enumerate(users[:50].tolist()))
