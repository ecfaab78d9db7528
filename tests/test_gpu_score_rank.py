"""GPU parity of the fused catalogue evaluation (orx_score_rank, openrec_b200/csrc/orx_eval.cu) and of
openrec.tf2.metrics.RankingEvaluator.

The reference throughout is the existing two-kernel path on the same inputs: orx_score_all, then orx_rank_metrics on
dense masks scattered from the same CSR rows.  Every metric is an integer count over comparisons of float32 scores and
the fused kernel computes each score by the same FFMA chain, so AUC and Recall must be bit-identical; NDCG within one
float32 ulp (both kernels sum float64 terms, in different orders)."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


# ---- problems --------------------------------------------------------------------------------------------------------
class Problem:
    """Tables, per-user CSR lists (sorted, unique, possibly with the ignored entries -1 and I) and a batch of uids."""

    def __init__(self, kind, user, item, bias, scale, pos_rows, excl_rows, uid):
        self.kind, self.U, self.I = kind, len(user), len(item)
        self.user, self.item = dev(user), dev(item)
        self.bias = None if bias is None else dev(bias)
        self.scale = None if scale is None else dev(scale)
        self.pos_rows, self.excl_rows = pos_rows, excl_rows
        self.uid = np.asarray(uid, np.int64)
        self.pos_off, self.pos_items = self._csr(pos_rows)
        self.excl_off, self.excl_items = self._csr(excl_rows) if excl_rows is not None else (None, None)

    def _csr(self, rows):
        lens = np.array([len(rows.get(u, ())) for u in range(self.U)], np.int64)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        items = np.concatenate([np.asarray(rows.get(u, ()), np.int64) for u in range(self.U)] + [np.zeros(0)])
        return dev(off, torch.int64), dev(items.astype(np.int32), torch.int32)

    def max_pos(self):
        lens = [len(self.pos_rows.get(int(u), ())) if 0 <= u < self.U else 0 for u in self.uid]
        return max(lens) if lens else 0

    def masks(self):
        Bu = len(self.uid)
        pos, excl = np.zeros((Bu, self.I), bool), np.zeros((Bu, self.I), bool)
        for b, u in enumerate(self.uid):
            if not 0 <= u < self.U:
                continue
            for rows, m in ((self.pos_rows, pos), (self.excl_rows or {}, excl)):
                r = np.asarray(rows.get(int(u), ()), np.int64)
                m[b, r[(r >= 0) & (r < self.I)]] = True
        return pos, excl

    def fused(self, eng, at, max_pos=None):
        return eng.score_rank(self.kind, self.user, dev(self.uid, torch.int32), self.item, self.bias, self.pos_off,
                              self.pos_items, self.excl_off, self.excl_items,
                              self.max_pos() if max_pos is None else max_pos, at=at, scale=self.scale)

    def reference(self, eng, at):
        pred = eng.score_all(self.kind, self.user, dev(self.uid, torch.int32), self.item, self.bias, scale=self.scale)
        pos, excl = self.masks()
        return eng.rank_metrics(pred, dev(pos, torch.uint8), dev(excl, torch.uint8), at=at)


def make_problem(rng, kind, Bu, I, D, scaled=False, biased=True, maxp=30, maxe=60, U=None, ties=True):
    """Random tables; users get up to maxp positives and maxe exclusions, one positive in ten also excluded, and a few
    rows carry the ignored entries -1 and I.  With ties: item rows copied from positives (exact ties: the <= and >
    rules), rows one ulp away from a positive, and biases 89, 100, -110, -1e4 (expf overflows and underflows)."""
    U = U or max(3, Bu // 2 + 2)
    user = rng.uniform(-1, 1, (U, D)).astype(F32)
    item = rng.uniform(-1, 1, (I, D)).astype(F32)
    bias = rng.uniform(-1, 1, I).astype(F32)
    scale = rng.uniform(-2, 2, D).astype(F32) if scaled else None
    pos_rows, excl_rows = {}, {}
    for u in range(U):
        k = min(I, int(rng.integers(0, maxp + 1)) + int(rng.integers(0, maxe + 1)))
        chosen = rng.choice(I, k, replace=False)
        n_pos = min(k, int(rng.integers(0, maxp + 1)))
        pos, ex = chosen[:n_pos], chosen[n_pos:]
        both = pos[rng.random(len(pos)) < 0.1]
        p, e = set(pos.tolist()), set(ex.tolist()) | set(both.tolist())
        if rng.random() < 0.2:
            p |= {-1, I}
        if rng.random() < 0.2:
            e |= {-1, I}
        pos_rows[u], excl_rows[u] = sorted(p), sorted(e)
    if ties and I > 4:
        src = [i for u in range(U) for i in pos_rows[u] if 0 <= i < I]
        if src:
            n = max(1, min(I // 8, 400))
            for j, s in zip(rng.choice(I, n, replace=False), rng.choice(src, n)):
                if j == s:
                    continue
                item[j], bias[j] = item[s], bias[s]
                if rng.random() < 0.5:                      # one ulp away in one coordinate
                    c = rng.integers(0, D)
                    item[j, c] = np.nextafter(item[j, c], F32(np.inf) if rng.random() < 0.5 else F32(-np.inf))
        ext = rng.choice(I, max(1, I // 50), replace=False)
        bias[ext] = rng.choice(np.array([89, 100, -110, -1e4], F32), len(ext))
    uid = rng.integers(0, U, Bu)
    where = rng.permutation(Bu)[:4]
    uid[where] = np.array([-1, U, 0, 0])[:len(where)]        # bad uids and a duplicate
    return Problem(kind, user, item, bias if biased else None, scale, pos_rows, excl_rows, uid)


def check_equal(got, want, what=""):
    (ga, gn, gr), (wa, wn, wr) = ([t.cpu().numpy() for t in x] for x in (got, want))
    np.testing.assert_array_equal(ga.view(np.int32), wa.view(np.int32), err_msg=f"AUC bits {what}")
    np.testing.assert_array_equal(gr.view(np.int32), wr.view(np.int32), err_msg=f"Recall bits {what}")
    assert gn.shape == wn.shape, what
    assert np.array_equal(np.isnan(gn), np.isnan(wn)), what
    ok = ~np.isnan(wn)
    np.testing.assert_array_max_ulp(gn[ok], wn[ok], maxulp=1)


def last_dispatch(eng):
    rec = [r for r in eng.debug_dispatch_log() if r.op == L.ORX_OP_SCORE_RANK]
    assert rec, "no orx_score_rank record"
    return rec[-1]


# (Bu, I, D): tile edges at 128 users / 128 items, D below, at and above the chunk of 8, item splits that do not divide
# the tile count (I = 100 003: 782 item tiles)
SHAPES = [(1, 1, 1), (127, 129, 7), (128, 127, 16), (129, 16980, 50), (1000, 16980, 50), (129, 100003, 128),
          (128, 1000, 256), (1000, 127, 1)]
VARIANTS = [(False, True), (True, True), (False, False), (True, False)]   # (scale, bias)


@pytest.mark.parametrize("Bu,I,D", SHAPES)
@pytest.mark.parametrize("scaled,biased", VARIANTS, ids=["plain", "scale", "nobias", "scale-nobias"])
@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_score_rank_equals_two_kernel_path(eng, kind, scaled, biased, Bu, I, D):
    """AUC and Recall bit-identical, NDCG within 1 ulp, for cut-offs none, one and eight (one larger than I), with exact
    ties, one-ulp neighbours, overflowing / underflowing expf, excluded positives, bad uids and ignored list entries."""
    rng = np.random.default_rng(seed_of(kind, scaled, biased, Bu, I, D))
    pb = make_problem(rng, kind, Bu, I, D, scaled=scaled, biased=biased)
    eight = (1, 2, 3, 5, 10, 50, 100, I + 7)
    for at in ((), (1,), eight):
        check_equal(pb.fused(eng, at), pb.reference(eng, at), f"at={at}")
        assert last_dispatch(eng).variant == L.ORX_VARIANT_RANK_SMEM


@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_special_rows(eng, kind):
    """No positives (NaN AUC and Recall, NDCG 0), no eval items (NaN AUC), every item positive, duplicate uids, uids
    -1 and U, list entries -1 and I, and a row longer than max_pos (NaN outputs; the other rows unchanged).  No
    exclusion lists at all (excl_off = NULL) is checked on the same users."""
    rng = np.random.default_rng(seed_of("special", kind))
    U, I, D = 8, 300, 16
    pb = make_problem(rng, kind, 1, I, D, U=U, maxp=5, maxe=5)
    allI = list(range(I))
    pb.pos_rows.update({0: [], 1: [3, 7, 11], 2: allI, 3: [-1, 5, I], 4: sorted(rng.choice(I, 40, replace=False))})
    pb.excl_rows.update({0: [1, 2], 1: [i for i in allI if i not in (3, 7, 11)], 2: [], 3: [-1, 5, 6, I], 4: [0]})
    uid = [0, 1, 2, 3, 4, 4, -1, U, 1, 2, 5, 6]
    pb = Problem(kind, pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy(), None, pb.pos_rows,
                 pb.excl_rows, uid)
    at = (1, 10, 100, I + 1)
    got, want = pb.fused(eng, at), pb.reference(eng, at)
    check_equal(got, want)
    a, n, r = (t.cpu().numpy() for t in got)
    assert np.isnan(a[0]) and np.isnan(r[0]).all() and not n[0].any()
    assert np.isnan(a[1]) and np.isnan(a[2]) and (r[2] > 0).all()
    assert np.isnan(a[6]) and np.isnan(a[7]) and not n[6].any()
    # max_pos = 39: the rows of user 2 (all I items) and user 4 (40 items) are longer and give NaN everywhere, the
    # other rows are unchanged
    a2, n2, r2 = (t.cpu().numpy() for t in pb.fused(eng, at, max_pos=39))
    long_rows = np.isin(pb.uid, [2, 4])
    assert np.isnan(a2[long_rows]).all() and np.isnan(n2[long_rows]).all() and np.isnan(r2[long_rows]).all()
    np.testing.assert_array_equal(a2[~long_rows].view(np.int32), a[~long_rows].view(np.int32))
    np.testing.assert_array_equal(r2[~long_rows].view(np.int32), r[~long_rows].view(np.int32))
    # without exclusion lists
    pb_noex = Problem(kind, pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy(), None, pb.pos_rows,
                      None, uid)
    check_equal(pb_noex.fused(eng, at), pb_noex.reference(eng, at), "no exclusions")


@pytest.mark.parametrize("case", ["one_long_user", "tiles_jointly"])
def test_global_path(eng, case):
    """RANK_GLOBAL: one user with 30 000 positives at I = 100 003, and 128 users of ~300 positives each (each row
    alone is small, the tile's thresholds and histograms together exceed shared memory).  RANK_SMEM for a small
    max_pos on the same handle.  All equal the two-kernel path."""
    rng = np.random.default_rng(seed_of("global", case))
    kind = N.ORX_SCORE_DOT
    if case == "one_long_user":
        pb = make_problem(rng, kind, 1, 100003, 64, U=2, maxp=5, maxe=100)
        pb.pos_rows[0] = sorted(rng.choice(100003, 30000, replace=False).tolist())
        pb = Problem(kind, pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy(), None, pb.pos_rows,
                     pb.excl_rows, [0])
    else:
        pb = make_problem(rng, kind, 128, 20000, 32, U=200, maxp=5, maxe=50)
        for u in range(200):
            pb.pos_rows[u] = sorted(rng.choice(20000, int(rng.integers(250, 320)), replace=False).tolist())
        pb = Problem(kind, pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy(), None, pb.pos_rows,
                     pb.excl_rows, rng.integers(0, 200, 128))
    at = (10, 100, 1000)
    check_equal(pb.fused(eng, at), pb.reference(eng, at), case)
    assert last_dispatch(eng).variant == L.ORX_VARIANT_RANK_GLOBAL
    small = make_problem(rng, kind, 64, 5000, 32)
    check_equal(small.fused(eng, at), small.reference(eng, at), "small after global")
    assert last_dispatch(eng).variant == L.ORX_VARIANT_RANK_SMEM


def test_workspace_reuse_and_fresh_handle(eng):
    """A large call then a small one on the same handle (the scratch is reused, not reinitialised by size), and the
    small one again on a fresh handle: identical bits."""
    rng = np.random.default_rng(seed_of("ws"))
    big = make_problem(rng, N.ORX_SCORE_DOT, 1000, 16980, 50, maxp=200)
    small = make_problem(rng, N.ORX_SCORE_NEG_SQDIST, 129, 3000, 24)
    at = (5, 50)
    check_equal(big.fused(eng, at), big.reference(eng, at), "big")
    first = small.fused(eng, at)
    check_equal(first, small.reference(eng, at), "small")
    fresh = N.Engine(torch.cuda.current_device())
    try:
        again = small.fused(fresh, at)
        torch.cuda.synchronize()
        for x, y in zip(first, again):
            assert np.array_equal(x.cpu().numpy().view(np.int32), y.cpu().numpy().view(np.int32))
    finally:
        torch.cuda.synchronize()
        fresh.close()


def test_evaluation_between_prefetch_and_step(eng):
    """An orx_score_rank call (which grows its scratch on first use) issued between orx_pairwise_prefetch and the step
    that consumes the prefetch: the step still uses the prefetched index and its tables and outputs are bit-identical
    to the same sequence without the evaluation.  Every row appears once in the batch, so the step itself has no
    float atomics and is bit-reproducible."""
    rng = np.random.default_rng(seed_of("prefetch"))
    U, I, D, B = 5000, 10000, 64, 2048
    init = [rng.uniform(-0.1, 0.1, s).astype(F32) for s in ((U, D), (I, D), (I, 1))]
    items = rng.permutation(I)[:2 * B].astype(np.int32)
    ids = [rng.permutation(U)[:B].astype(np.int32), items[:B], items[B:]]
    pb = make_problem(rng, N.ORX_SCORE_DOT, 700, 40000, 64, maxp=400)

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
            pb.fused(e, (10,))
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
    """I = 1 000 000, D = 128, Bu = 256, positives ~ Poisson(20), exclusions ~ Poisson(100), against the two-kernel
    path."""
    rng = np.random.default_rng(seed_of("bench"))
    I, D, Bu, U = 1_000_000, 128, 256, 256
    user = rng.uniform(-0.1, 0.1, (U, D)).astype(F32)
    item = rng.uniform(-0.1, 0.1, (I, D)).astype(F32)
    bias = rng.uniform(-0.1, 0.1, I).astype(F32)
    pos_rows, excl_rows = {}, {}
    for u in range(U):
        n_p, n_e = rng.poisson(20), rng.poisson(100)
        c = rng.choice(I, n_p + n_e, replace=False)
        pos_rows[u], excl_rows[u] = sorted(c[:n_p].tolist()), sorted(c[n_p:].tolist())
    pb = Problem(N.ORX_SCORE_DOT, user, item, bias, None, pos_rows, excl_rows, rng.permutation(U)[:Bu])
    at = (50, 100)
    check_equal(pb.fused(eng, at), pb.reference(eng, at))


# ---- end to end through openrec.tf2 -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def _datasets(rng, U, I, n_warm):
    """train / validation Datasets: n_warm validation users with 1..5 held-out items, everyone with up to 40 training
    items (some users absent from one of them)."""
    from openrec.tf2.data import Dataset
    tr, va = [], []
    warm = rng.choice(U, n_warm, replace=False)
    for u in range(U):
        items = rng.choice(I, 45, replace=False)
        if u in set(warm.tolist()):
            va += [(u, i) for i in items[:1 + u % 5]]
        if u % 11:
            tr += [(u, i) for i in items[5:5 + int(rng.integers(1, 41))]]
    rng.shuffle(va)                                          # warm-user order = first appearance, not sorted

    def mk(pairs):
        raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = np.array(pairs).T
        return Dataset(raw_data=raw, total_users=U, total_items=I)
    return mk(tr), mk(va)


@pytest.mark.parametrize("model_name", ["bpr", "ucml", "gmf", "wrmf"])
def test_evaluator_end_to_end(tf, model_name):
    """RankingEvaluator.evaluate(model) against the reference example's loop (the evaluation stream's masks +
    model.inference + AUC / NDCG / Recall), per user, at the example's shape: 1 000 warm users, I = 16 980, D = 50,
    weights on a dyadic grid.  AUC / Recall bit-identical, NDCG within 1 ulp, the DictMean results within 1e-6, and
    inference unchanged by the _score_operands refactor (equal to score_all on the same operands)."""
    from openrec.tf2.metrics import AUC, NDCG, DictMean, RankingEvaluator, Recall
    from openrec.tf2.recommenders import BPR, GMF, UCML, WRMF
    from openrec_b200.tf2.data.dataset import _Streams
    rng = np.random.default_rng(seed_of("e2e-evaluator", model_name))
    U, I, D = 1200, 16980, 50
    train, val = _datasets(rng, U, I, 1000)
    cls = {"bpr": BPR, "ucml": UCML, "gmf": GMF, "wrmf": WRMF}[model_name]
    model = cls(D, D, U, I)
    model.user_latent_factor.embeddings.assign((rng.integers(-2, 3, (U, D)) / 8).astype(F32))
    model.item_latent_factor.embeddings.assign((rng.integers(-2, 3, (I, D)) / 8).astype(F32))
    model.item_bias.embeddings.assign((rng.integers(-64, 65, (I, 1)) / 64).astype(F32))
    if model_name == "gmf":
        model.mlp.layers[0].kernel.assign((rng.integers(-8, 9, (D, 1)) / 8).astype(F32))
    at = [50, 100]
    ev = RankingEvaluator(val, excl_datasets=[train], at=at, batch_size=256)
    res = ev.evaluate(model)
    shapes = {"AUC": [], "NDCG": [len(at)], "Recall": [len(at)]}
    fused_mean, ref_mean = DictMean(shapes), DictMean(shapes)
    fused_mean.update_state(res)
    rows = list(_Streams.evaluation(val.datastore, [train]))
    assert [r["user_id"] for r in rows] == ev.warm_users.tolist()
    ref = {"AUC": [], "NDCG": [], "Recall": []}
    kind, user, item, bias, scale = model._score_operands()
    for b0 in range(0, len(rows), 300):                    # the reference loop, in its own batch size
        chunk = rows[b0:b0 + 300]
        users = np.array([r["user_id"] for r in chunk], np.int32)
        pos = np.stack([r["pos_mask"] for r in chunk])
        excl = np.stack([r["excl_mask"] for r in chunk])
        pred = model.inference(users)
        direct = N.engine().score_all(kind, user, dev(users, torch.int32), item, bias, scale=scale)
        assert np.array_equal(pred.numpy().view(np.int32), direct.cpu().numpy().view(np.int32))
        batch = {"AUC": AUC(pos_mask=pos, pred=pred, excl_mask=excl),
                 "NDCG": NDCG(pos_mask=pos, pred=pred, excl_mask=excl, at=at),
                 "Recall": Recall(pos_mask=pos, pred=pred, excl_mask=excl, at=at)}
        ref_mean.update_state(batch)
        for k in ref:
            ref[k].append(batch[k].numpy())
    ref = [np.concatenate(ref[k]) for k in ("AUC", "NDCG", "Recall")]
    got = [res[k].numpy() for k in ("AUC", "NDCG", "Recall")]
    check_equal([torch.from_numpy(x) for x in got], [torch.from_numpy(x) for x in ref], model_name)
    fm, rm = fused_mean.result(), ref_mean.result()
    for k in shapes:
        np.testing.assert_allclose(fm[k].numpy(), rm[k].numpy(), atol=1e-6, rtol=0, err_msg=k)
    assert 0.3 < got[0].mean() < 0.7 and got[2][:, 1].max() > 0
