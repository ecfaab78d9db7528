"""GPU parity of the kernels outside the training step (orx_misc.cu, orx_dlrm.cu's strided gather, orx_sampler.cu):
fill, gather, censor, dense apply, full-catalogue scoring, ranking metrics and the three device samplers, on every
path they take and at the reference example's evaluation shape.

Copies, integer outputs and the samplers are compared bit for bit; arithmetic against the float64 oracle
(oracle/openrec_oracle.py) with the bound stated at each test; the samplers and the fill stream against the numpy
restatement of their counter-based draws (oracle/device_samplers.py)."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle import device_samplers as S
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- path rules ------------------------------------------------------------------------------------------------------
# The branch each kernel takes and how many rows / ids / elements its first grid pass covers (the launchers cap the
# grid at a multiple of the SM count; beyond that a grid-stride loop runs).
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gather_vec(D):                      # k_gather: float4 rows
    return D % 4 == 0


def gather_strided_vec(D, out_ld):      # k_gather_strided: float4 rows only if every output row stays 16-byte aligned
    return D % 4 == 0 and out_ld % 4 == 0


def censor_vec(D):                      # k_censor: one float4 per lane, 8 rows in flight per warp
    return D % 4 == 0 and D <= 128


def gather_cap():                       # 32 blocks per SM, 8 warps, one row per warp
    return 32 * _sms() * 8


def censor_cap():                       # 8 blocks per SM, 8 warps x 8 ids
    return 8 * _sms() * 64


def dense_cap():                        # k_dense_apply and k_fill_uniform: 16 blocks per SM x 256 threads
    return 16 * _sms() * 256


SCORE_T, SCORE_KC = 64, 16              # k_score_all: 64 users x 64 items per block, D in chunks of 16


GATHER_D = (1, 3, 4, 50, 128, 256)
# (D, out_ld, first column, features F = id stride): vector path; scalar with D % 4 != 0; scalar with D % 4 == 0 but a
# leading dimension that is not (base still 16-byte aligned); id strides 1 and F
STRIDED = [(128, 384, 128, 3), (64, 64, 0, 1), (50, 150, 50, 3), (8, 13, 0, 1), (1, 5, 3, 4)]
CENSOR_D = (1, 3, 12, 50, 128, 129, 256)
CENSOR_BIG = (300000, 100000)           # ids, rows
CENSOR_BIG_D = (50, 128)
DENSE_N = (1, 257, 2000003)
FILL_N = 3000001
SCORE_SHAPES = [(1, 1, 1), (64, 64, 16), (65, 65, 17), (130, 1000, 33), (1000, 16980, 50), (70, 300, 256)]
RANK_I = (1, 1023, 1024, 1025, 3072, 16980)


def _gather_ns():
    return (0, 1, 777, gather_cap() + 333)


def test_misc_path_coverage():
    """The parametrisations below reach both sides of every branch predicate and at least one grid-stride case per
    kernel."""
    assert {gather_vec(D) for D in GATHER_D} == {True, False}
    assert max(_gather_ns()) > gather_cap()
    assert {(D % 4 == 0, gather_strided_vec(D, ld)) for D, ld, _, _ in STRIDED} == {(True, True), (False, False),
                                                                                  (True, False)}
    assert {F == 1 for *_, F in STRIDED} == {True, False}
    assert {censor_vec(D) for D in CENSOR_D} == {True, False}
    assert any(D % 4 == 0 and not censor_vec(D) for D in CENSOR_D) and any(D % 4 for D in CENSOR_D)
    assert CENSOR_BIG[0] > censor_cap()
    assert max(DENSE_N) > dense_cap() and FILL_N > dense_cap() and min(DENSE_N) == 1
    tiles = {(Bu + SCORE_T - 1) // SCORE_T for Bu, _, _ in SCORE_SHAPES}
    assert min(tiles) == 1 and max(tiles) > 2
    assert any(D > SCORE_KC and D % SCORE_KC for _, _, D in SCORE_SHAPES)
    assert any(D % SCORE_KC == 0 for _, _, D in SCORE_SHAPES)
    assert any(I > SCORE_T and I % SCORE_T for _, I, _ in SCORE_SHAPES)
    assert {I % 1024 for I in RANK_I} >= {0, 1, 1023} and max(RANK_I) > 1024


# ---- helpers ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    return N.engine()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())   # hash() is randomised per process


def vp(t):
    return C.c_void_p(t.data_ptr())


def close(t, ref, atol, rtol, what=""):
    got = t.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(t) else np.asarray(t, np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol,
                               err_msg=what)


def bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


SENTINEL = 0x7FC0DEAD                   # a quiet NaN whose payload no kernel writes


def sentinel_buffer(n_floats, pad=64):
    """float32 buffer of n_floats between two pads of `pad` floats (256 bytes: the base stays 16-byte aligned), all
    set to the NaN SENTINEL.  -> (whole buffer, address of the first float after the front pad)."""
    buf = torch.full((n_floats + 2 * pad,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    return buf, C.c_void_p(buf.data_ptr() + 4 * pad)


# ---- score_all -------------------------------------------------------------------------------------------------------
def _score_ref(kind, user, item, uid, w):
    """float64 oracle with a zero bias; an out-of-range uid scores as a zero user row (an appended zero row)."""
    U = len(user)
    ue = np.vstack([user, np.zeros((1, user.shape[1]))])
    ids = np.where((uid >= 0) & (uid < U), uid, U)
    zero = np.zeros((len(item), 1))
    if kind == N.ORX_SCORE_DOT:
        return O.gmf_inference(ue, item, zero, w, ids) if w is not None else O.dot_inference(ue, item, zero, ids)
    if w is not None:
        ue = ue * w.reshape(1, -1)
    return np.concatenate([O.ucml_inference(ue, item, zero, ids[c:c + 25]) for c in range(0, len(ids), 25)])


@pytest.mark.parametrize("Bu,I,D", SCORE_SHAPES)
@pytest.mark.parametrize("scaled", [False, True], ids=["plain", "scale"])
@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_score_all(eng, kind, scaled, Bu, I, D):
    """Full-catalogue scores against O.dot_inference / O.gmf_inference (DOT, scale = GMF's w) and O.ucml_inference
    (NEG_SQDIST, with scale: of u * w), each with the item bias and with a NULL bias.  The uids hold duplicates, 0,
    U - 1, -1 and U; out-of-range uids score as a zero user row.  Bound: |got - ref| <= 1e-5 * max(1, M) + 1e-5 |ref|,
    M = D * max|u'| * max|i| (DOT) or D * (max|u'| + max|i|)^2 (NEG_SQDIST), u' = u (* w): float32 sums of D terms of
    at most that size."""
    rng = np.random.default_rng(seed_of(Bu, I, D, kind, scaled))
    U = max(3, Bu // 2)                                       # duplicates come naturally
    user, item = rng.uniform(-1, 1, (U, D)), rng.uniform(-1, 1, (I, D))
    bias, w = rng.uniform(-1, 1, (I, 1)), (rng.uniform(-2, 2, (D, 1)) if scaled else None)
    uid = rng.integers(0, U, Bu)
    where = rng.permutation(Bu)[:5]
    uid[where] = np.array([U - 1, 0, -1, U, U - 1])[:len(where)]     # the last one duplicates the first
    tu, ti, tb, tw = dev(user), dev(item), dev(bias), dev(w.reshape(-1)) if scaled else None
    user, item, bias = (t.cpu().numpy().astype(np.float64) for t in (tu, ti, tb))
    if scaled:
        w = tw.cpu().numpy().astype(np.float64)
    ref = _score_ref(kind, user, item, uid, w)
    mu = np.abs(user).max() * (np.abs(w).max() if scaled else 1.0)
    M = D * (mu * np.abs(item).max() if kind == N.ORX_SCORE_DOT else (mu + np.abs(item).max()) ** 2)
    atol = 1e-5 * max(1.0, M)
    for b in (tb, None):
        got = eng.score_all(kind, tu, dev(uid, torch.int32), ti, b, scale=tw)
        want = ref + bias.reshape(1, -1) if b is not None else ref
        close(got, want, atol, 1e-5, what=f"bias={b is not None}")
        bad = (uid < 0) | (uid >= U)
        if b is None:   # a zero user row: DOT scores 0, NEG_SQDIST -||item||^2 (the rows are pinned, not only close)
            zero_row = np.zeros(I) if kind == N.ORX_SCORE_DOT else -(item ** 2).sum(1)
            close(got[torch.from_numpy(bad).cuda()], np.broadcast_to(zero_row, (int(bad.sum()), I)), atol, 1e-5)


# ---- rank_metrics ----------------------------------------------------------------------------------------------------
def _rank_problem(rng, R, I):
    """float32 predictions on a 1/64 grid in [-4, 4] (exp keeps distinct values distinct, exact ties stay ties), with
    overflowing (>= 89: exp = inf) and underflowing (<= -110: exp = 0) values mixed in.  Row 0 .. 6 (when R > 1):
    no positives; no eval items; every item positive; positives that are also excluded; mostly overflow / underflow;
    one whole 1024-item tile positive; a single positive.  Other rows (and R = 1): positives, excluded items and
    excluded positives at random."""
    pred = (rng.integers(-256, 257, (R, I)) / 64).astype(np.float32)
    ext = rng.random((R, I)) < 0.02
    pred[ext] = rng.choice(np.array([89, 100, 1e4, -110, -200, -1e4], np.float32), int(ext.sum()))
    dens = min(0.3, max(30 / I, 0.0))
    pos = rng.random((R, I)) < dens
    excl = rng.random((R, I)) < 0.1
    excl &= ~pos | (rng.random((R, I)) < 0.1)            # about one positive in ten is also excluded
    if R > 1:
        pos[0] = False                                     # no positives
        pos[1] = rng.random(I) < 0.5                       # no eval items
        pos[1, 0] = True
        excl[1] = ~pos[1]
        pos[2], excl[2] = True, False                      # every item positive
        excl[3] = pos[3] | (rng.random(I) < 0.2)           # every positive excluded too
        pos[3, 0] = excl[3, 0] = True
        big = rng.random(I) < 0.6                          # overflow / underflow row
        pred[4, big] = rng.choice(np.array([89, 1e3, -110, -1e3], np.float32), int(big.sum()))
        pos[4, :2] = True
        if I >= 1024:                                      # a tile whose positives fill all TILE slots
            pos[5, :1024] = True
            excl[5, :1024] = False
        pos[6] = False
        pos[6, I // 2] = True                              # a single positive
    return pred, pos, excl


def _nan_ulp(got, want, maxulp, what):
    got = got.detach().cpu().numpy() if torch.is_tensor(got) else got
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    ok = ~np.isnan(want)
    np.testing.assert_array_max_ulp(got[ok], want[ok].astype(np.float32), maxulp=maxulp)


@pytest.mark.parametrize("R", [1, 300])
@pytest.mark.parametrize("I", RANK_I)
def test_rank_metrics(eng, I, R):
    """orx_rank_metrics against O.auc / O.ndcg / O.recall fed the identical float32 predictions: AUC within 1 float32
    ulp (pred_e <= pred_p counted on the raw predictions), recall bit-exact (the integer count of ranks below each
    cut-off over n_pos), NDCG within 1e-6 + 1e-6 |ref|.  exp overflows to inf and ties there; an excluded overflowed
    item scores inf * 0 = NaN and never ranks above anything, exactly as in the reference.  Rows without positives
    give NaN AUC and recall and NDCG 0, rows without eval items NaN AUC.  Cut-offs: none (the AUC metric's call), one,
    and eight including one larger than I; each output requested alone equals the one computed with the others."""
    rng = np.random.default_rng(seed_of(I, R))
    pred, pos, excl = _rank_problem(rng, R, I)
    eight = (1, 2, 3, 5, 10, 50, 100, I + 7)
    with np.errstate(all="ignore"):
        auc_r = O.auc(pos, pred, excl)
        ndcg_r, rec_r = O.ndcg(pos, pred, excl, eight), O.recall(pos, pred, excl, eight)
    dp, dpos, dex = dev(pred), dev(pos, torch.uint8), dev(excl, torch.uint8)
    full = None
    for at, cols in (((), []), ((1,), [0]), (eight, list(range(8)))):
        auc, ndcg, rec = eng.rank_metrics(dp, dpos, dex, at=at)
        what = f"I={I} R={R} at={at}"
        _nan_ulp(auc, auc_r, 1, what)
        assert ndcg.shape == rec.shape == (R, len(at))
        np.testing.assert_array_equal(rec.cpu().numpy(), rec_r[:, cols], err_msg=what)
        np.testing.assert_allclose(ndcg.cpu().numpy(), ndcg_r[:, cols], atol=1e-6, rtol=1e-6, equal_nan=True,
                                   err_msg=what)
        full = (auc, ndcg, rec)
    for k, name in enumerate(("auc", "ndcg", "recall")):
        alone = eng.rank_metrics(dp, dpos, dex, at=eight, want=(name,))
        assert all(x is None for j, x in enumerate(alone) if j != k)
        assert np.array_equal(bits(alone[k]), bits(full[k])), name
    if R > 1:                                              # the special rows hold what the docstring says
        assert np.isnan(auc_r[0]) and np.isnan(rec_r[0]).all() and not ndcg_r[0].any()
        assert np.isnan(auc_r[1]) and np.isnan(auc_r[2]) and (rec_r[2] > 0).all()


# ---- evaluation end to end through openrec.tf2 -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


@pytest.mark.parametrize("model_name", ["bpr", "ucml", "gmf"])
def test_evaluation_end_to_end(tf, model_name):
    """The evaluation of tf2_examples/bpr_citeulike.py at its shape: model.inference on 1000 users, D = 50, I = 16 980,
    then AUC, Recall(at=[50, 100]) and NDCG(at=[50, 100]) from openrec.tf2.metrics with the evaluation generator's
    masks (hits = the user's held-out items, excluded = the user's training items, dataset.py evaluation).  The
    injected weights lie on a dyadic grid (entries k/8, biases k/64, w k/8), so every score is exact in float32 in any
    summation order: scores equal the float64 oracle exactly, and equal scores are exact ties.  Metrics are compared
    with the oracle evaluated on the GPU's own float32 scores."""
    from openrec.tf2.metrics import AUC, NDCG, Recall
    from openrec.tf2.recommenders import BPR, GMF, UCML
    rng = np.random.default_rng(seed_of("e2e", model_name))
    U, I, D, Bu = 1200, 16980, 50, 1000
    cls = {"bpr": BPR, "ucml": UCML, "gmf": GMF}[model_name]
    model = cls(D, D, U, I)
    user, item = rng.integers(-2, 3, (U, D)) / 8, rng.integers(-2, 3, (I, D)) / 8
    bias = rng.integers(-64, 65, (I, 1)) / 64
    model.user_latent_factor.embeddings.assign(user.astype(np.float32))
    model.item_latent_factor.embeddings.assign(item.astype(np.float32))
    model.item_bias.embeddings.assign(bias.astype(np.float32))
    if model_name == "gmf":
        w = rng.integers(-8, 9, (D, 1)) / 8
        model.mlp.layers[0].kernel.assign(w.astype(np.float32))
    users = np.sort(rng.choice(U, Bu, replace=False)).astype(np.int32)
    pos, excl = np.zeros((Bu, I), bool), np.zeros((Bu, I), bool)
    for r in range(Bu):
        items = rng.choice(I, 40, replace=False)
        n_val = 1 + r % 5
        pos[r, items[:n_val]] = True                       # held-out items of the user
        excl[r, items[n_val:]] = True                      # the user's training items
    pred = model.inference(users)
    got = pred.numpy()
    ref = {"bpr": lambda: O.dot_inference(user, item, bias, users),
           "ucml": lambda: np.concatenate([O.ucml_inference(user, item, bias, users[c:c + 25])
                                           for c in range(0, Bu, 25)]),
           "gmf": lambda: O.gmf_inference(user, item, bias, w, users)}[model_name]()
    assert got.shape == (Bu, I) and np.array_equal(got.astype(np.float64), ref)
    auc = AUC(pos_mask=pos, pred=pred, excl_mask=excl).numpy()
    rec = Recall(pos_mask=pos, pred=pred, excl_mask=excl, at=[50, 100]).numpy()
    ndcg = NDCG(pos_mask=pos, pred=pred, excl_mask=excl, at=[50, 100]).numpy()
    _nan_ulp(auc, O.auc(pos, got, excl), 1, "AUC")
    np.testing.assert_array_equal(rec, O.recall(pos, got, excl, (50, 100)))
    np.testing.assert_allclose(ndcg, O.ndcg(pos, got, excl, (50, 100)), atol=1e-6, rtol=1e-6)
    assert 0.3 < auc.mean() < 0.7 and rec[:, 1].max() > 0       # the metrics saw scores, not zeros


# ---- gather / gather_strided -----------------------------------------------------------------------------------------
def _bad_ids(rows, is64):
    return [-1, rows] + ([2 ** 31 + 5, 2 ** 32 + 5] if is64 else [2 ** 31 - 1])


@pytest.mark.parametrize("is64", [False, True], ids=["int32", "int64"])
@pytest.mark.parametrize("D", GATHER_D)
def test_gather(eng, D, is64):
    """orx_gather bit-exact: rows copied, bad ids (-1, rows, and 2^31 + 5, 2^32 + 5 as int64: no wrap to a valid row)
    give zero rows and are all counted in n_bad; nothing outside the n x D output is written.  n = 0 (empty id and
    output tensors pass NULL), 1, 777 and one n past the first grid pass."""
    rng = np.random.default_rng(seed_of(D, is64))
    rows = 1000
    tab = dev(rng.standard_normal((rows, D)))
    tab_h = tab.cpu().numpy()
    for n in _gather_ns():
        ids = rng.integers(0, rows, n)
        bad = _bad_ids(rows, is64)
        at = rng.permutation(n)[:len(bad)]
        ids[at] = bad[:len(at)]
        ok = (ids >= 0) & (ids < rows)
        want = np.where(ok[:, None], tab_h[np.where(ok, ids, 0)], np.float32(0))
        did = dev(ids, torch.int64 if is64 else torch.int32)
        buf, out = sentinel_buffer(n * D)
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        L.check(eng.lib.orx_gather(eng.h, vp(tab), rows, D, vp(did), int(is64), n, out, vp(n_bad), eng.stream()),
               "orx_gather")
        b = bits(buf)
        assert (b[:64] == SENTINEL).all() and (b[64 + n * D:] == SENTINEL).all(), f"n={n}: wrote outside the rows"
        assert np.array_equal(b[64:64 + n * D], want.view(np.int32).reshape(-1)), f"n={n}"
        assert n_bad.item() == int((~ok).sum()), (n, n_bad.item())
        if n == 0:                                         # an empty lookup (NULL ids and out) is an empty result
            assert eng.gather(tab, did).shape == (0, D)


@pytest.mark.parametrize("D,out_ld,c0,F", STRIDED)
def test_gather_strided(eng, D, out_ld, c0, F):
    """orx_gather_strided bit-exact into a column slice [c0, c0 + D) of rows of out_ld floats, ids = ids2d[:, col] with
    stride F: bad ids (-1, rows, 2^31 - 1) give zero rows and are counted in n_bad (called through the C-ABI:
    Engine.gather_strided passes NULL), the rest of each row and the bytes around the view keep the NaN sentinel."""
    rng = np.random.default_rng(seed_of(D, out_ld, F))
    rows, col = 700, F // 2
    tab = dev(rng.standard_normal((rows, D)))
    tab_h = tab.cpu().numpy()
    for n in _gather_ns()[1:]:
        ids2d = rng.integers(0, rows, (n, F)).astype(np.int64)
        at = rng.permutation(n)[:3]
        ids2d[at, col] = _bad_ids(rows, False)[:len(at)]
        ids = ids2d[:, col]
        ok = (ids >= 0) & (ids < rows)
        buf, base = sentinel_buffer(n * out_ld)
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        did = dev(ids2d, torch.int32)
        L.check(eng.lib.orx_gather_strided(eng.h, vp(tab), rows, D, C.c_void_p(did.data_ptr() + 4 * col), F, n,
                                          C.c_void_p(base.value + 4 * c0), out_ld, vp(n_bad), eng.stream()),
               "orx_gather_strided")
        want = np.full(n * out_ld + 128, SENTINEL, dtype=np.int32)
        view = want[64:64 + n * out_ld].reshape(n, out_ld)
        view[:, c0:c0 + D] = np.where(ok[:, None], tab_h[np.where(ok, ids, 0)], np.float32(0)).view(np.int32)
        assert np.array_equal(bits(buf), want), f"n={n}"
        assert n_bad.item() == int((~ok).sum())


# ---- censor ----------------------------------------------------------------------------------------------------------
def _censor_ids(rng, n, rows, touched):
    """n ids over the first `touched` rows with duplicates inside one warp's group of 8, across warps and blocks, and
    the bad ids -1 and rows (ignored)."""
    ids = rng.integers(0, touched, n).astype(np.int64)
    ids[:8] = [7, 7, 9, 7, 11, 11, 7, 9]
    ids[8:16] = 7                                          # the same row again in the next group
    ids[n // 2] = ids[n - 1] = 9                           # and in far-away blocks
    ids[3], ids[20], ids[n - 2] = -1, rows, -1
    return ids


def _run_censor(eng, rng, D, rows, n, touched, min_norm):
    small = rng.random(rows) < 0.5                         # rows below and above min_norm
    tab = rng.standard_normal((rows, D)) * np.where(small, 1e-3, 1.0)[:, None]
    t = dev(tab)
    before = bits(t)
    ref = t.cpu().numpy().astype(np.float64)
    ids = _censor_ids(rng, n, rows, touched)
    eng.censor(t, dev(ids, torch.int32), min_norm)
    valid = ids[(ids >= 0) & (ids < rows)]
    O.censor(ref, valid, min_norm)
    after = bits(t)
    untouched = np.setdiff1d(np.arange(rows), valid)
    assert len(untouched) and np.array_equal(after[untouched], before[untouched])
    close(t, ref, atol=1e-7, rtol=1e-5, what=f"D={D} min_norm={min_norm}")


@pytest.mark.parametrize("D", CENSOR_D)
def test_censor(eng, D):
    """orx_censor against O.censor in float64: each unique row scaled once by 1 / max(||row||, min_norm), with rows
    below and above min_norm, min_norm 0.1 and 1.0; duplicates inside a warp's group of 8 and across warps and blocks;
    bad ids ignored; untouched rows bit-identical.  Bound 1e-7 + 1e-5 |ref| (float32 norm of D terms)."""
    rng = np.random.default_rng(D)
    for min_norm in (0.1, 1.0):
        _run_censor(eng, rng, D, 1000, 2000, 800, min_norm)


@pytest.mark.parametrize("D", CENSOR_BIG_D)
def test_censor_grid_stride(eng, D):
    """300 000 ids over 100 000 rows: more ids than the first grid pass covers, on both paths."""
    _run_censor(eng, np.random.default_rng(seed_of(D, "big")), D, CENSOR_BIG[1], CENSOR_BIG[0], 90000, 0.1)


def _ucml_schedule(rng, order, U, I, D, B):
    """Two UCML SGD steps interleaved with censors, as (kind, payload) events, and the float64 tables they must leave.
    order "step_first": step, three censors of its batch, prefetch of the next batch (bench.py's UCML loop);
    "censor_first": prefetch, three censors of other ids, the step that consumes the prefetch.  Each batch is drawn
    on the tables it will meet, away from the hinge's kink (|h| < 1e-3 flips in float32)."""
    user, item, bias = rng.uniform(-0.4, 0.4, (U, D)), rng.uniform(-0.4, 0.4, (I, D)), rng.uniform(-0.4, 0.4, (I, 1))
    init = [a.astype(np.float32) for a in (user, item, bias)]
    ref = [a.astype(np.float64) for a in init]

    def draw():
        for _ in range(50):
            ids = tuple(rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
            u, p, n = ref[0][ids[0]], ref[1][ids[1]], ref[1][ids[2]]
            h = 0.5 - ((-((u - p) ** 2).sum(1) + ref[2][ids[1], 0]) - (-((u - n) ** 2).sum(1) + ref[2][ids[2], 0]))
            if not (np.abs(h) < 1e-3).any():
                return ids
        raise AssertionError("could not avoid hinge ties")

    def step(ids, k):
        O.pairwise_train_step("ucml", *ref, *ids, O.OPT_SGD, {}, k, 0.05, margin=0.5)

    events = []
    if order == "step_first":
        nxt = draw()
        events.append(("prefetch", nxt))
        for k in (1, 2):
            ids = nxt
            events.append(("step", ids))
            step(ids, k)
            events.append(("censor", ids))
            O.ucml_censor_vec(ref[0], ref[1], *ids)
            if k == 1:
                nxt = draw()
                events.append(("prefetch", nxt))
    else:
        for k in (1, 2):
            cids = tuple(rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
            O.ucml_censor_vec(ref[0], ref[1], *cids)
            ids = draw()
            events += [("prefetch", ids), ("censor", cids), ("step", ids)]
            step(ids, k)
    return init, ref, events


@pytest.mark.parametrize("order", ["step_first", "censor_first"])
def test_censor_with_prefetched_step(eng, order):
    """Censor shares the context's batch hash (index set 0) and its epoch counter with the pairwise step.  Mixed with
    a pipelined step in either order, the step still consumes the prefetched index (set 1 or 2 in its dispatch record)
    and the tables equal O.pairwise_train_step and O.censor in the same order, within 1e-5."""
    rng = np.random.default_rng(seed_of("censor-pf", order))
    U, I, D, B = 300, 500, 64, 600
    init, ref, events = _ucml_schedule(rng, order, U, I, D, B)
    tabs = [dev(a) for a in init]
    tt = [N.table(t) for t in tabs]
    dids = {id(ids): [dev(x, torch.int32) for x in ids] for kind, ids in events}
    torch.cuda.synchronize()                               # the id tensors are complete: ids_ready=True is honest
    eng.debug_dispatch_log()
    out4, k = torch.zeros(4, device="cuda"), 0
    for kind, ids in events:
        d = dids[id(ids)]
        if kind == "prefetch":
            eng.pairwise_prefetch(tt[0], tt[1], *d, L.ORX_OPT_SGD, ids_ready=True)
        elif kind == "censor":
            eng.censor(tabs[0], d[0]), eng.censor(tabs[1], d[1]), eng.censor(tabs[1], d[2])
        else:
            k += 1
            eng.pairwise_step(N.ORX_PAIR_UCML, *tt, *d, N.opt(L.ORX_OPT_SGD, 0.05, step=k), out4, margin=0.5)
            rec = eng.debug_dispatch_log()
            assert len(rec) == 1 and rec[0].op == L.ORX_OP_PAIRWISE_STEP and rec[0].s in (1, 2), rec
    for t, r, name in zip(tabs, ref, ("user", "item", "bias")):
        close(t, r, atol=1e-5, rtol=1e-5, what=name)


# ---- dense_apply / fill_uniform --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DENSE_N)
@pytest.mark.parametrize("kind,step", [(L.ORX_OPT_SGD, 1), (L.ORX_OPT_ADAGRAD, 1), (L.ORX_OPT_ADAM_LAZY, 1),
                                       (L.ORX_OPT_ADAM_LAZY, 7), (L.ORX_OPT_ADAM_DENSE, 1), (L.ORX_OPT_ADAM_DENSE, 7)])
def test_dense_apply(eng, kind, step, n):
    """orx_dense_apply against O.apply_dense in float64 (var and every slot within 1e-5 + 1e-5 |ref|); n = 1, 257 and
    one n past the first grid pass; Adam at steps 1 and 7.  ADAM_DENSE and ADAM_LAZY give identical bits on a dense
    variable."""
    rng = np.random.default_rng(seed_of(n, kind, step))
    lr = {L.ORX_OPT_SGD: 0.05, L.ORX_OPT_ADAGRAD: 0.05}.get(kind, 0.01)
    host = [rng.standard_normal(n), rng.standard_normal(n), np.abs(rng.standard_normal(n)) * 0.1 + 0.1,
            np.abs(rng.standard_normal(n)) * 0.1 + 0.01]
    tv, tg, t0, t1 = (dev(a) for a in host)
    var, grad, s0, s1 = (t.cpu().numpy().astype(np.float64) for t in (tv, tg, t0, t1))
    copies = [t.clone() for t in (tv, t0, t1)]
    eng.dense_apply(tv, t0 if kind else None, t1 if kind >= 2 else None, tg, N.opt(kind, lr, step=step))
    O.apply_dense(kind, var, s0, s1, grad, step, lr)
    close(tv, var, 1e-5, 1e-5, "var")
    if kind:
        close(t0, s0, 1e-5, 1e-5, "s0")
    if kind >= 2:
        close(t1, s1, 1e-5, 1e-5, "s1")
        other = L.ORX_OPT_ADAM_LAZY if kind == L.ORX_OPT_ADAM_DENSE else L.ORX_OPT_ADAM_DENSE
        eng.dense_apply(copies[0], copies[1], copies[2], tg, N.opt(other, lr, step=step))
        for a, b in zip(copies, (tv, t0, t1)):
            assert torch.equal(a, b)


def test_fill_uniform_stream(eng):
    """orx_fill_uniform restated: u_i = (splitmix64(seed * 0xD1342543DE82EF95 + i) >> 40) * 2^-24.  On [0, 1) the output
    is u bit for bit (3 000 001 values: past the first grid pass, odd tail; seeds 0 and 2^63 + 5).  Other ranges:
    within one float32 ulp of max(|lo|, |hi|) of the float64 lo + (hi - lo) u, and below hi."""
    t = torch.empty(FILL_N, device="cuda")
    for seed in (0, 2 ** 63 + 5):
        eng.fill_uniform(t, 0.0, 1.0, seed)
        u = S.fill_uniform_u(seed, 0, FILL_N)
        assert np.array_equal(t.cpu().numpy().view(np.int32), u.view(np.int32)), seed
    seed = 11
    u = S.fill_uniform_u(seed, 0, FILL_N).astype(np.float64)
    for lo, hi in ((-0.05, 0.05), (-3.0, 7.0), (-2.5, -0.5), (0.25, 1000.0), (1.0, 2.0)):
        eng.fill_uniform(t, lo, hi, seed)
        got = t.cpu().numpy()
        lo32, hi32 = np.float32(lo), np.float32(hi)
        want = np.float64(lo32) + (np.float64(hi32) - np.float64(lo32)) * u
        ulp = float(np.spacing(np.float32(max(abs(lo), abs(hi)))))
        assert np.abs(got - want).max() <= ulp, (lo, hi)
        assert got.min() >= lo32 and got.max() < hi32, (lo, hi)


def test_fill_uniform_half_open_bound(eng):
    """[1, 2): lo + (hi - lo) u rounds to hi for u = 1 - 2^-24 (fused or not).  Seed 0 draws that u at index
    3 747 935 (the restatement proves the case is exercised); the kernel must clamp it to the largest float below 2,
    and no value of 2^26 may reach hi."""
    seed, idx, n = 0, 3747935, 1 << 26
    assert S.fill_uniform_u(seed, idx, idx + 1)[0] == np.float32(1 - 2.0 ** -24)
    t = torch.empty(n, device="cuda")
    eng.fill_uniform(t, 1.0, 2.0, seed)
    assert t[idx].item() == float(np.nextafter(np.float32(2), np.float32(1)))
    assert t.max().item() < 2.0 and t.min().item() >= 1.0


# ---- device samplers -------------------------------------------------------------------------------------------------
class Store:
    """orx_sampler_t built by hand from numpy arrays (explicit permutations, no torch.randperm); .sd is the same data
    for the restatement."""

    def __init__(self, U, I, pairs, perm_cur, perm_next):
        users, items = pairs[:, 0].astype(np.int32), pairs[:, 1].astype(np.int32)
        order = np.lexsort((items, users))
        off = np.zeros(U + 1, dtype=np.int64)
        np.cumsum(np.bincount(users, minlength=U), out=off[1:])
        self.sd = dict(rec_user=users, rec_item=items, perm_cur=perm_cur.astype(np.int64),
                       perm_next=perm_next.astype(np.int64), cursor=0, csr_off=off, csr_items=items[order],
                       total_users=U, total_items=I)
        self.d = {k: dev(v, torch.int64 if v.dtype == np.int64 else torch.int32)
                  for k, v in self.sd.items() if isinstance(v, np.ndarray)}
        self.n = len(users)

    def struct(self, cursor):
        self.sd["cursor"] = cursor
        d = self.d
        return L.OrxSampler(d["rec_user"].data_ptr(), d["rec_item"].data_ptr(), d["perm_cur"].data_ptr(),
                            d["perm_next"].data_ptr(), cursor, self.n, d["csr_off"].data_ptr(),
                            d["csr_items"].data_ptr(), self.sd["total_users"], self.sd["total_items"])


def _store(rng, U, I, n, extra=()):
    pairs = np.stack([rng.integers(0, U, n), rng.integers(0, I, n)], 1)
    pairs = np.unique(np.concatenate([pairs] + [np.asarray(e).reshape(-1, 2) for e in extra]), axis=0)
    rng.shuffle(pairs)
    return Store(U, I, pairs, rng.permutation(len(pairs)), rng.permutation(len(pairs)))


def _pairwise_store():
    """60 users x 90 items; user 0 has every item but one, user 1 every item (its negatives give up)."""
    rng = np.random.default_rng(31)
    U, I = 60, 90
    almost = [(0, i) for i in range(I) if i != 41]
    every = [(1, i) for i in range(I)]
    return _store(rng, U, I, 1100, [almost, every])


PAIR_CASES = [("start", 1), ("start", 1000), ("last", 1000), ("end", 1), ("end", "n"), ("start", "n"), ("last", "n")]


@pytest.mark.parametrize("where,B", PAIR_CASES)
def test_sample_pairwise_bit_exact(eng, where, B):
    """k_sample_pairwise against the restatement, uid / pid / nid bit for bit: cursor 0, n - 1 (the batch crosses the
    epoch boundary) and n (the batch starts in the next permutation); B = 1, 1000 and n."""
    st = _pairwise_store()
    cursor = {"start": 0, "last": st.n - 1, "end": st.n}[where]
    B = st.n if B == "n" else B
    seed, pos0 = 2 ** 63 + 12345, 10 ** 12 + 17
    sd = st.struct(cursor)
    out = [torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(3)]
    L.check(eng.lib.orx_sample_pairwise(eng.h, C.byref(sd), seed, pos0, B, *map(vp, out), eng.stream()),
           "orx_sample_pairwise")
    want = S.sample_pairwise(st.sd, seed, pos0, B)
    for name, g, w in zip(("uid", "pid", "nid"), out, want):
        assert np.array_equal(g.cpu().numpy(), w), name
    if B == st.n:                                          # the give-up path and the one-free-item user both ran
        assert {0, 1} <= set(want[0].tolist())


STRAT_B = (1, 31, 1024, 1025, 5000)


@pytest.mark.parametrize("ratio", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("B", STRAT_B)
def test_sample_stratified_bit_exact(eng, B, ratio):
    """k_sample_stratified against the restatement: uid / iid / label and n_pos_out exact.  B > 1024 runs the chunk
    carry of the coin scan; the cursor sits 700 records before the end of the epoch, so large batches cross it."""
    st = _store(np.random.default_rng(32), 300, 500, 6200)
    _run_stratified(eng, st, st.n - 700, B, ratio, seed=987654321, pos0=3 * 10 ** 9 + 1)


def test_sample_stratified_fully_observed(eng):
    """Every (user, item) pair observed: each negative's rejection loop runs to its bound and keeps the last draw."""
    pairs = np.array([(u, i) for u in range(3) for i in range(4)])
    rng = np.random.default_rng(33)
    st = Store(3, 4, pairs, rng.permutation(12), rng.permutation(12))
    _run_stratified(eng, st, 5, 12, 0.3, seed=5, pos0=0)


def _run_stratified(eng, st, cursor, B, ratio, seed, pos0):
    sd = st.struct(cursor)
    uid, iid = (torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(2))
    lab = torch.full((B,), -1.0, device="cuda")
    npos = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    L.check(eng.lib.orx_sample_stratified(eng.h, C.byref(sd), seed, pos0, B, ratio, vp(uid), vp(iid), vp(lab),
                                         vp(npos), eng.stream()), "orx_sample_stratified")
    wu, wi, wl, wn = S.sample_stratified(st.sd, seed, pos0, B, ratio)
    assert np.array_equal(uid.cpu().numpy(), wu) and np.array_equal(iid.cpu().numpy(), wi)
    assert np.array_equal(lab.cpu().numpy(), wl) and npos.item() == wn
    if ratio in (0.0, 1.0):
        assert wn == (B if ratio == 1.0 else 0)


# (I, quota, group offset of stream_pos, B, cursor): quota 0 / 1 / 4 / 64 (= ORX_MAX_QUOTA) / I - 1; stream_pos at a
# group start and inside a group; B smaller than one group; a batch crossing the end of the epoch
PER_POS_CASES = [(65, 0, 0, 500, "start"), (65, 1, 0, 301, "start"), (65, 1, 1, 300, "mid"), (65, 4, 0, 777, "start"),
                 (65, 4, 3, 512, "mid"), (65, 64, 10, 10, "mid"), (65, 64, 0, 1000, "start"), (30, 29, 7, 400, "mid"),
                 (65, 4, 2, 100, "last")]


@pytest.mark.parametrize("I,quota,off,B,where", PER_POS_CASES)
def test_sample_per_positive_bit_exact(eng, I, quota, off, B, where):
    """k_sample_per_positive against the restatement: uid / iid / label bit for bit (the negatives of a group: distinct
    draws in order, the positive removed, the first `quota` kept)."""
    st = _store(np.random.default_rng(seed_of(34, I)), 100, I, 1500)
    g = quota + 1
    cursor = {"start": 17, "mid": 400, "last": st.n - 1}[where]
    pos0 = 123457 * g + off                                # the cursor is the record of stream_pos's group
    seed = 77 + quota
    sd = st.struct(cursor)
    uid, iid = (torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(2))
    lab = torch.full((B,), -1.0, device="cuda")
    L.check(eng.lib.orx_sample_per_positive(eng.h, C.byref(sd), seed, pos0, B, quota, vp(uid), vp(iid), vp(lab),
                                           eng.stream()), "orx_sample_per_positive")
    wu, wi, wl = S.sample_per_positive(st.sd, seed, pos0, B, quota)
    assert np.array_equal(uid.cpu().numpy(), wu) and np.array_equal(iid.cpu().numpy(), wi)
    assert np.array_equal(lab.cpu().numpy(), wl)
