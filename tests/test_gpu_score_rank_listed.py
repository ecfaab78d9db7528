"""GPU parity of the listed-candidate evaluation (orx_score_rank_listed, openrec_b200/csrc/orx_eval.cu) and of
openrec.tf2.metrics.CandidateEvaluator.

Each batch row is ranked against its listed items only.  The references are the paths a user has without the new call,
on the same inputs: orx_score_all, then orx_rank_metrics on the dense masks Dataset.evaluation builds for a dataset
with explicit negatives (pos = P, excl = ~(P u L) u E); and orx_score_rank with the complement exclusion rows
~(P u L) u E.  Every score comes from the chain of k_score_all, so AUC and Recall must be bit-identical; NDCG within one
float32 ulp (float64 sums in another order), the bar of tests/test_gpu_score_rank.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N
from test_gpu_score_rank import Problem, check_equal, dev, make_problem, seed_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
KINDS = [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST]


@pytest.fixture(scope="module")
def eng():
    return N.engine()


class Listed(Problem):
    """A Problem with listed items: neg_rows, per user, sorted and unique (may hold -1 and I)."""

    def __init__(self, kind, user, item, bias, scale, pos_rows, neg_rows, excl_rows, uid):
        super().__init__(kind, user, item, bias, scale, pos_rows, excl_rows, uid)
        self.neg_rows = neg_rows
        self.neg_off, self.neg_items = self._csr(neg_rows)

    def tables(self):
        return (self.user.cpu().numpy(), self.item.cpu().numpy(), None if self.bias is None else self.bias.cpu().numpy(),
                None if self.scale is None else self.scale.cpu().numpy())

    def listed(self, eng, at, max_pos=None, item=None):
        return eng.score_rank_listed(self.kind, self.user, dev(self.uid, torch.int32),
                                     self.item if item is None else item, self.bias, self.pos_off, self.pos_items,
                                     self.neg_off, self.neg_items, self.excl_off, self.excl_items,
                                     self.max_pos() if max_pos is None else max_pos, at=at, scale=self.scale)

    def _row(self, rows, u):
        r = np.asarray((rows or {}).get(int(u), ()), np.int64)
        return set(r[(r >= 0) & (r < self.I)].tolist())

    def complement_rows(self):
        """Per user: ~(P u L) u E within [0, I)."""
        every = set(range(self.I))
        return {u: sorted((every - self._row(self.pos_rows, u) - self._row(self.neg_rows, u))
                          | self._row(self.excl_rows, u)) for u in range(self.U)}

    def reference(self, eng, at):
        """orx_score_all + orx_rank_metrics on the masks of Dataset.evaluation."""
        pred = eng.score_all(self.kind, self.user, dev(self.uid, torch.int32), self.item, self.bias, scale=self.scale)
        Bu = len(self.uid)
        pos, excl = np.zeros((Bu, self.I), bool), np.ones((Bu, self.I), bool)
        for b, u in enumerate(self.uid):
            if not 0 <= u < self.U:
                continue
            p, n, e = (sorted(self._row(r, u)) for r in (self.pos_rows, self.neg_rows, self.excl_rows))
            pos[b, p] = True
            excl[b, p] = excl[b, n] = False
            excl[b, e] = True
        return eng.rank_metrics(pred, dev(pos, torch.uint8), dev(excl, torch.uint8), at=at)

    def complement(self, eng, at, max_pos=None):
        """orx_score_rank with the exclusion rows ~(P u L) u E."""
        u, i, b, s = self.tables()
        pb = Problem(self.kind, u, i, b, s, self.pos_rows, self.complement_rows(), self.uid)
        return pb.fused(eng, at, max_pos=max_pos)


def with_lists(pb, rng, n_neg=100, overlap=0.1):
    """Listed items for every user of a make_problem: up to n_neg items, about `overlap` of them also positives and as
    many also excluded, on some rows the ignored entries -1 and I."""
    neg_rows = {}
    for u in range(pb.U):
        k = min(pb.I, int(rng.integers(0, n_neg + 1)))
        s = set(rng.choice(pb.I, k, replace=False).tolist())
        p = [i for i in pb.pos_rows.get(u, ()) if 0 <= i < pb.I]
        e = [i for i in pb.excl_rows.get(u, ()) if 0 <= i < pb.I]
        for src in (p, e):
            if src:
                s |= set(rng.choice(src, max(1, int(overlap * len(src))), replace=False).tolist())
        if rng.random() < 0.2:
            s |= {-1, pb.I}
        neg_rows[u] = sorted(s)
    return neg_rows


def make_listed(rng, kind, Bu, I, D, scaled=False, biased=True, **kw):
    pb = make_problem(rng, kind, Bu, I, D, scaled=scaled, biased=biased, **kw)
    u, i, b, s = (None if t is None else t.cpu().numpy() for t in (pb.user, pb.item, pb.bias, pb.scale))
    return Listed(kind, u, i, b, s, pb.pos_rows, with_lists(pb, rng), pb.excl_rows, pb.uid)


def check_both(eng, pb, at, what=""):
    got = pb.listed(eng, at)
    check_equal(got, pb.reference(eng, at), f"masks {what}")
    check_equal(got, pb.complement(eng, at), f"complement {what}")
    return got


# ---- parity ----------------------------------------------------------------------------------------------------------
# (Bu, I, D): Bu in {1, 37, 1000}, I in {1, 129, 16980}, D in {1, 33, 50, 128} (below, at and past one 32-column slab)
SHAPES = [(1, 1, 1), (37, 129, 33), (1000, 16980, 50), (37, 16980, 128), (1000, 129, 1), (1, 16980, 128),
          (37, 1, 50), (1000, 129, 33)]
VARIANTS = [(False, True), (True, True), (False, False), (True, False)]   # (scale, bias)


@pytest.mark.parametrize("Bu,I,D", SHAPES)
@pytest.mark.parametrize("scaled,biased", VARIANTS, ids=["plain", "scale", "nobias", "scale-nobias"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_listed_equals_mask_and_complement_paths(eng, kind, scaled, biased, Bu, I, D):
    """Cut-offs none, one and eight (one past I); exact ties and one-ulp neighbours, overflowing / underflowing expf,
    excluded positives, listed items that are positives or excluded, bad uids and ignored entries."""
    rng = np.random.default_rng(seed_of("listed", kind, scaled, biased, Bu, I, D))
    pb = make_listed(rng, kind, Bu, I, D, scaled=scaled, biased=biased)
    for at in ((), (1,), (1, 2, 3, 5, 10, 50, 100, I + 7)):
        check_both(eng, pb, at, f"at={at}")


@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_special_rows(eng, kind):
    """Bad uids, a positive row longer than max_pos (NaN outputs, the other rows unchanged), no listed items (NaN AUC),
    listed items that are positives or excluded, excluded positives, entries -1 and I, and crafted item rows whose
    scores tie exactly, are NaN or +-inf; no exclusion lists at all on the same users."""
    rng = np.random.default_rng(seed_of("listed-special", kind))
    U, I, D = 9, 300, 16
    user = rng.uniform(-1, 1, (U, D)).astype(F32)
    item = rng.uniform(-1, 1, (I, D)).astype(F32)
    bias = rng.uniform(-1, 1, I).astype(F32)
    item[10], item[11, 3], item[12, 5], item[13, 0] = item[20], np.nan, np.inf, -np.inf
    bias[14], bias[15] = np.inf, -np.inf
    item[16], bias[16] = item[21], bias[21]                 # 16 ties 21 exactly, bias included
    pos = {0: [3, 7], 1: sorted(rng.choice(I, 40, replace=False).tolist()), 2: [4, 5], 3: [1, 2, 3, 30],
           4: [6, 8, 9], 5: [-1, 5, I], 6: [20, 21, 11], 7: [12, 13], 8: []}
    neg = {0: [50, 60], 1: sorted(rng.choice(I, 30, replace=False).tolist()), 2: [], 3: [1, 2, 40, 41, 42],
           4: [50, 51, 52], 5: [-1, 6, 7, I], 6: [10, 16, 14, 15, 12, 13, 70], 7: [10, 11, 14, 15, 16, 20],
           8: [1, 2, 3]}
    neg = {u: sorted(r) for u, r in neg.items()}
    pos = {u: sorted(r) for u, r in pos.items()}
    excl = {0: [], 1: [], 2: [], 3: [2, 40, 99], 4: [6, 8, 51], 5: [-1, 7, I], 6: [70], 7: [], 8: [1]}
    uid = [0, 1, 2, 3, 4, 5, 6, 7, 8, -1, U, 3, 6]
    pb = Listed(kind, user, item, bias, None, pos, neg, excl, uid)
    at = (1, 3, 10, I + 1)
    got = check_both(eng, pb, at)
    a, n, r = (t.cpu().numpy() for t in got)
    assert np.isnan(a[2]) and not np.isnan(r[2]).any()      # no listed items: no eval item, Recall still defined
    assert np.isnan(a[8]) and np.isnan(r[8]).all()          # no positives
    assert np.isnan(a[9]) and np.isnan(a[10]) and not n[9].any()
    a2, n2, r2 = (t.cpu().numpy() for t in pb.listed(eng, at, max_pos=39))   # user 1's 40 positives: NaN everywhere
    long_rows = np.asarray(uid) == 1
    assert np.isnan(a2[long_rows]).all() and np.isnan(n2[long_rows]).all() and np.isnan(r2[long_rows]).all()
    np.testing.assert_array_equal(a2[~long_rows].view(np.int32), a[~long_rows].view(np.int32))
    np.testing.assert_array_equal(r2[~long_rows].view(np.int32), r[~long_rows].view(np.int32))
    check_equal(pb.listed(eng, at, max_pos=39), pb.complement(eng, at, max_pos=39), "max_pos = 39")
    noex = Listed(kind, user, item, bias, None, pos, neg, None, uid)
    check_both(eng, noex, at, "no exclusions")


# ---- limits and handle behaviour -------------------------------------------------------------------------------------
def test_empty_batch_and_refusals(eng):
    """Bu = 0 is a no-op; each bad argument returns ORX_ERR_INVALID and leaves the outputs untouched."""
    rng = np.random.default_rng(seed_of("listed-refuse"))
    pb = make_listed(rng, N.ORX_SCORE_DOT, 16, 100, 8, U=20)
    lib = L.lib()
    Bu, mp = 16, pb.max_pos()
    uid = dev(pb.uid, torch.int32)
    auc = torch.full((Bu,), 7.0, device="cuda")
    ndcg = torch.full((Bu * 8,), 7.0, device="cuda")
    at = (C.c_int32 * 8)(*range(1, 9))
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731

    def call(kind=0, user=pb.user, U=20, uid=uid, Bu=Bu, item=pb.item, I=100, dim=8, pos_off=pb.pos_off,
             neg_off=pb.neg_off, max_pos=mp, at=at, n_at=8):
        return lib.orx_score_rank_listed(eng.h, kind, p(user), U, p(uid), Bu, None, p(item), p(pb.bias), I, dim,
                                         p(pos_off), p(pb.pos_items), p(neg_off), p(pb.neg_items), p(pb.excl_off),
                                         p(pb.excl_items), max_pos, at, n_at, p(auc), p(ndcg), None, eng.stream())

    bad = {"kind": dict(kind=2), "null user": dict(user=None), "null uid": dict(uid=None), "null item": dict(item=None),
           "null pos_off": dict(pos_off=None), "null neg_off": dict(neg_off=None), "U 0": dict(U=0), "I 0": dict(I=0),
           "I > 2^31 - 1": dict(I=1 << 31), "dim 0": dict(dim=0), "Bu < 0": dict(Bu=-1), "max_pos < 0": dict(max_pos=-1),
           "n_at 9": dict(n_at=9), "null cut-offs": dict(at=None), "Bu * P": dict(Bu=1 << 20, max_pos=4096)}
    for name, kw in bad.items():
        assert call(**kw) == -1, name   # ORX_ERR_INVALID
        assert L.last_error(), name
    torch.cuda.synchronize()
    assert (auc == 7.0).all() and (ndcg == 7.0).all()
    assert call(Bu=0) == 0
    torch.cuda.synchronize()
    assert (auc == 7.0).all()
    with pytest.raises(ValueError):
        eng.score_rank_listed(N.ORX_SCORE_DOT, pb.user, uid, pb.item, pb.bias, pb.pos_off, pb.pos_items, None, None,
                              None, None, mp)


def test_workspace_reuse_and_fresh_handle(eng):
    """A large call, then a small one on the same handle, then the small one on a fresh handle: identical bits."""
    rng = np.random.default_rng(seed_of("listed-ws"))
    big = make_listed(rng, N.ORX_SCORE_DOT, 1000, 16980, 50, maxp=200)
    small = make_listed(rng, N.ORX_SCORE_NEG_SQDIST, 129, 3000, 24)
    at = (5, 50)
    check_equal(big.listed(eng, at), big.reference(eng, at), "big")
    first = small.listed(eng, at)
    check_equal(first, small.reference(eng, at), "small")
    fresh = N.Engine(torch.cuda.current_device())
    try:
        again = small.listed(fresh, at)
        torch.cuda.synchronize()
        for x, y in zip(first, again):
            assert np.array_equal(x.cpu().numpy().view(np.int32), y.cpu().numpy().view(np.int32))
    finally:
        torch.cuda.synchronize()
        fresh.close()


def test_evaluation_between_prefetch_and_step(eng):
    """An orx_score_rank_listed call (growing its scratch on a fresh handle) between orx_pairwise_prefetch and the
    step that consumes the prefetch: the step still uses the prefetched index, and its tables and outputs are
    bit-identical to the same sequence without the evaluation."""
    rng = np.random.default_rng(seed_of("listed-prefetch"))
    U, I, D, B = 5000, 10000, 64, 2048
    init = [rng.uniform(-0.1, 0.1, s).astype(F32) for s in ((U, D), (I, D), (I, 1))]
    items = rng.permutation(I)[:2 * B].astype(np.int32)
    ids = [rng.permutation(U)[:B].astype(np.int32), items[:B], items[B:]]
    pb = make_listed(rng, N.ORX_SCORE_DOT, 700, 40000, 64, maxp=400)

    def run(with_eval, e):
        tabs = [dev(a) for a in init]
        acc = [torch.full_like(t, 0.1) for t in tabs]
        tt = [N.table(t, s) for t, s in zip(tabs, acc)]
        d = [dev(x, torch.int32) for x in ids]
        out4 = torch.zeros(4, device="cuda")
        torch.cuda.synchronize()
        e.debug_dispatch_log()
        e.pairwise_prefetch(tt[0], tt[1], *d, L.ORX_OPT_ADAGRAD, ids_ready=True)
        if with_eval:
            pb.listed(e, (10,))
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


def test_far_item_table(eng):
    """An item table past 2^32 elements (2^25 + 2^22 + 64 rows at D = 128), users listing low rows and rows at or
    above 2^32 / D: bit-equal to the same lists on the touched rows alone (a truncated row address would read the
    row's low alias, planted with other values)."""
    D = 128
    rows = -(-((1 << 32) + (1 << 29)) // D) + 64
    need = rows * D * 4 + rows * 4
    free = torch.cuda.mem_get_info()[0]
    if free < need + (2 << 30):
        pytest.skip(f"needs {(need + (2 << 30)) / 2**30:.1f} GB free on the device, {free / 2**30:.1f} GB are")
    rng = np.random.default_rng(seed_of("listed-far"))
    U, Bu = 64, 64
    far0 = (1 << 32) // D
    item = torch.empty((rows, D), device="cuda")
    bias = torch.empty(rows, device="cuda")
    try:
        item.uniform_(-1, 1)
        bias.uniform_(-1, 1)
        far = np.sort(rng.choice(np.arange(far0, rows), 3000, replace=False))
        low = np.sort(np.concatenate([far - far0, rng.choice(1 << 20, 500, replace=False)]))   # aliases and others
        item[torch.from_numpy(far).cuda()] = torch.from_numpy(rng.uniform(5, 6, (len(far), D)).astype(F32)).cuda()
        pool = np.unique(np.concatenate([far, low]))
        user = rng.uniform(-1, 1, (U, D)).astype(F32)
        pos, neg, excl = {}, {}, {}
        for u in range(U):
            c = rng.choice(pool, 150, replace=False)
            pos[u], neg[u], excl[u] = sorted(c[:20].tolist()), sorted(c[20:140].tolist()), sorted(c[130:150].tolist())
        uid = rng.integers(0, U, Bu)
        at = (5, 50)
        big = Listed(N.ORX_SCORE_DOT, user, np.zeros((1, D), F32), None, None, pos, neg, excl, uid)
        big.item, big.bias, big.I = item, bias, rows
        got = big.listed(eng, at)
        touched = np.unique(np.concatenate([np.asarray(r, np.int64) for d in (pos, neg, excl) for r in d.values()]))
        sel = torch.from_numpy(touched).cuda()
        ren = {int(i): k for k, i in enumerate(touched)}
        m = lambda d: {u: [ren[i] for i in r] for u, r in d.items()}   # noqa: E731
        small = Listed(N.ORX_SCORE_DOT, user, item[sel].cpu().numpy(), bias[sel].cpu().numpy(), None, m(pos), m(neg),
                       m(excl), uid)
        want = small.listed(eng, at)
        torch.cuda.synchronize()
        for x, y in zip(got, want):
            np.testing.assert_array_equal(x.cpu().numpy().view(np.int32), y.cpu().numpy().view(np.int32))
        assert np.isfinite(got[0].cpu().numpy()).all()
    finally:
        del item, bias
        torch.cuda.empty_cache()


@pytest.mark.parametrize("off", [1, 2, 3])
def test_unaligned_item_table(eng, off):
    """An item table (and bias) that starts `off` floats past a 16-byte boundary: bit-equal to the aligned call."""
    rng = np.random.default_rng(seed_of("listed-unaligned", off))
    pb = make_listed(rng, N.ORX_SCORE_NEG_SQDIST, 200, 3000, 128)
    at = (10, 100)
    want = pb.listed(eng, at)
    buf = torch.full((pb.I * 128 + 8,), float("nan"), device="cuda")
    view = buf[off:off + pb.I * 128].view(pb.I, 128)
    view.copy_(pb.item)
    bbuf = torch.full((pb.I + 8,), float("nan"), device="cuda")
    bview = bbuf[off:off + pb.I]
    bview.copy_(pb.bias)
    assert view.data_ptr() % 16 and bview.data_ptr() % 16
    saved = pb.bias
    pb.bias = bview
    try:
        got = pb.listed(eng, at, item=view)
    finally:
        pb.bias = saved
    for x, y in zip(got, want):
        np.testing.assert_array_equal(x.cpu().numpy().view(np.int32), y.cpu().numpy().view(np.int32))


# ---- end to end through openrec.tf2 -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def listed_datasets(rng, U, I, n_warm, labelled):
    """train / validation Datasets; the validation set lists explicit negatives: 100 per user drawn by the Dataset
    (num_negatives), or labelled records (implicit_negative=False) with one pair both positive and negative."""
    from openrec.tf2.data import Dataset
    tr, va = [], []
    warm = set(rng.choice(U, n_warm, replace=False).tolist())
    for u in range(U):
        items = rng.choice(I, 145, replace=False)
        if u in warm:
            va += [(u, int(i), 1.0) for i in items[:1 + u % 5]]
            if labelled:
                va += [(u, int(i), 0.0) for i in items[45:45 + int(rng.integers(0, 100))]]
        if u % 11:
            tr += [(u, int(i), 1.0) for i in items[5:5 + int(rng.integers(1, 41))]]
    if labelled:
        va.append((va[0][0], va[0][1], 0.0))                 # a pair both positive and listed negative
    rng.shuffle(va)

    def mk(recs, **kw):
        raw = np.empty(len(recs), dtype=[("user_id", np.int32), ("item_id", np.int32), ("label", np.float32)])
        raw["user_id"], raw["item_id"], raw["label"] = np.array(recs).T
        return Dataset(raw_data=raw, total_users=U, total_items=I, **kw)
    np.random.seed(11)
    return mk(tr), (mk(va, implicit_negative=False) if labelled else mk(va, num_negatives=100))


@pytest.mark.parametrize("labelled", [False, True], ids=["num_negatives", "labelled"])
@pytest.mark.parametrize("model_name", ["bpr", "ucml", "gmf", "wrmf"])
def test_candidate_evaluator_end_to_end(tf, model_name, labelled):
    """CandidateEvaluator.evaluate(model) against the reference example's loop (the evaluation stream's masks +
    model.inference + AUC / NDCG / Recall), per user, at the example's shape (I = 16 980, D = 50, 1 000 warm users)."""
    from openrec.tf2.metrics import AUC, NDCG, CandidateEvaluator, Recall
    from openrec.tf2.recommenders import BPR, GMF, UCML, WRMF
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(seed_of("e2e-candidate", model_name, labelled))
    U, I, D = 1200, 16980, 50
    train, val = listed_datasets(rng, U, I, 1000, labelled)
    model = {"bpr": BPR, "ucml": UCML, "gmf": GMF, "wrmf": WRMF}[model_name](D, D, U, I)
    model.user_latent_factor.embeddings.assign((rng.integers(-2, 3, (U, D)) / 8).astype(F32))
    model.item_latent_factor.embeddings.assign((rng.integers(-2, 3, (I, D)) / 8).astype(F32))
    model.item_bias.embeddings.assign((rng.integers(-64, 65, (I, 1)) / 64).astype(F32))
    if model_name == "gmf":
        model.mlp.layers[0].kernel.assign((rng.integers(-8, 9, (D, 1)) / 8).astype(F32))
    at = [10, 50]
    ev = CandidateEvaluator(val, excl_datasets=[train], at=at, batch_size=256)
    res = ev.evaluate(model)
    rows = list(_Streams.evaluation(val.datastore, [train]))
    assert [r["user_id"] for r in rows] == ev.warm_users.tolist()
    ref = {"AUC": [], "NDCG": [], "Recall": []}
    for b0 in range(0, len(rows), 300):
        chunk = rows[b0:b0 + 300]
        users = np.array([r["user_id"] for r in chunk], np.int32)
        pos, excl = np.stack([r["pos_mask"] for r in chunk]), np.stack([r["excl_mask"] for r in chunk])
        pred = model.inference(users)
        ref["AUC"].append(AUC(pos_mask=pos, pred=pred, excl_mask=excl).numpy())
        ref["NDCG"].append(NDCG(pos_mask=pos, pred=pred, excl_mask=excl, at=at).numpy())
        ref["Recall"].append(Recall(pos_mask=pos, pred=pred, excl_mask=excl, at=at).numpy())
    want = [torch.from_numpy(np.concatenate(ref[k])) for k in ("AUC", "NDCG", "Recall")]
    got = [torch.from_numpy(res[k].numpy()) for k in ("AUC", "NDCG", "Recall")]
    check_equal(got, want, model_name)
    assert 0.2 < np.nanmean(got[0].numpy()) < 0.8
