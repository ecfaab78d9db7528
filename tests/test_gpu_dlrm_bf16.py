"""GPU: bf16 embedding tables for DLRM.

- orx_gather_strided_bf16 / orx_bag_gather_bf16 are bit-equal to the fp32 entry points on the fp32 upcast of the tables.
- orx_sparse_apply_strided_bf16 / orx_bag_sparse_apply_bf16 are judged element by element through the rounding's bits:
  each stored element must lie in bf16_np.sr_interval of the fp32 entry point's result on the upcast table (the fp32
  applies are held to float64 by the step, row-wise and momentum suites), at the table's seed and step, table 0.
- DLRM(embedding_dtype="bfloat16") against an fp32 DLRM holding the upcast tables: forward, slices and Dense updates
  bit-equal, rows touched once equal orx_debug_round_bf16 of the fp32 model's row."""
import os
import sys

import numpy as np
import pytest
import torch

import bf16_np as BF
from openrec_b200 import native as N
from openrec_b200.tf2.recommenders.dlrm import table_rounding_seed

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U23 = 2.0 ** -23


@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def bf16_table(rng, rows, D, aligned=True, scale=0.5):
    """A bf16 [rows, D] CUDA table; aligned=False places it 2 bytes past an 8-byte boundary."""
    a = torch.from_numpy((rng.standard_normal((rows, D)) * scale).astype(np.float32)).to(torch.bfloat16)
    buf = torch.empty(rows * D + 4, dtype=torch.bfloat16, device="cuda")
    off = 0 if aligned else 1
    t = buf[off:off + rows * D].view(rows, D)
    t.copy_(a.cuda())
    assert (t.data_ptr() % 8 == 0) == aligned
    return t


def i32bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def u16(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def make_bags(rng, B, sizes, vocab, pad=0.2, bad=0.05):
    col_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    sp = np.empty((B, int(col_off[-1])), np.int32)
    for k, (Lk, V) in enumerate(zip(sizes, vocab)):
        ids = rng.integers(0, V, (B, Lk))
        u = rng.random((B, Lk))
        ids[u < pad] = -1
        m = (u >= pad) & (u < pad + bad)
        ids[m] = V + rng.integers(0, 3, int(m.sum()))
        if Lk > 1:
            d = rng.random(B) < 0.1
            ids[d, 1] = ids[d, 0]
        ids[rng.random(B) < 0.05] = -1                 # empty bags
        sp[:, col_off[k]:col_off[k + 1]] = ids
    return sp, [int(c) for c in col_off]


# ---- gathers ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aligned", (True, False))
@pytest.mark.parametrize("D", (4, 32, 128, 256, 50, 1))
def test_gather_strided_bit_equal_to_fp32_on_upcast(D, aligned):
    rng = np.random.default_rng(D * 2 + aligned)
    rows, B, F = 300, 517, 3
    tab = bf16_table(rng, rows, D, aligned)
    ids = torch.from_numpy(rng.integers(-2, rows + 3, (B, F)).astype(np.int32)).cuda()
    eng = N.engine()
    outs, bads = [], []
    for t in (tab, tab.float()):
        Z = torch.full((B, F, D), float("nan"), device="cuda")
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        for k in range(F):
            eng.gather_strided(t, ids, k, Z[:, k, :], n_bad)
        outs.append(Z)
        bads.append(int(n_bad.item()))
    assert np.array_equal(i32bits(outs[0]), i32bits(outs[1]))
    assert bads[0] == bads[1] > 0


@pytest.mark.parametrize("aligned", (True, False))
@pytest.mark.parametrize("mean", (0, 1))
@pytest.mark.parametrize("D", (4, 32, 128, 256, 50, 1))
def test_bag_gather_bit_equal_to_fp32_on_upcast(D, mean, aligned):
    rng = np.random.default_rng(100 + D * 4 + mean * 2 + aligned)
    B, sizes, vocab = 333, [3, 1, 7, 2], [50, 80, 30, 200]
    tabs = [bf16_table(rng, V, D, aligned) for V in vocab]
    sp, col_off = make_bags(rng, B, sizes, vocab)
    sp_t = torch.from_numpy(sp).cuda()
    eng = N.engine()
    outs, bads = [], []
    for ts in (tabs, [t.float() for t in tabs]):
        Z = torch.full((B, len(vocab) * D), float("nan"), device="cuda")
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        eng.bag_gather(ts, sp_t, col_off, mean, Z, n_bad)
        outs.append(Z)
        bads.append(int(n_bad.item()))
    assert np.array_equal(i32bits(outs[0]), i32bits(outs[1]))
    assert bads[0] == bads[1] > 0
    assert not torch.isnan(outs[0]).any()


def test_bag_gather_refuses_mixed_dtypes():
    rng = np.random.default_rng(3)
    a = bf16_table(rng, 10, 8)
    b = a.float()
    sp = torch.zeros((4, 2), dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="float32 or all bfloat16"):
        N.engine().bag_gather([a, b], sp, [0, 1, 2], 0, torch.empty(4, 16, device="cuda"))


# ---- applies ------------------------------------------------------------------------------------------------------
OPTS = {"sgd": (N.ORX_OPT_SGD, 0.05), "adagrad": (N.ORX_OPT_ADAGRAD, 0.05), "lazy": (N.ORX_OPT_ADAM_LAZY, 0.01),
        "adam": (N.ORX_OPT_ADAM_DENSE, 0.01), "rowwise": (N.ORX_OPT_ROWWISE_ADAGRAD, 0.05),
        "momentum": (N.ORX_OPT_MOMENTUM, 0.05), "nesterov": (N.ORX_OPT_NESTEROV, 0.05)}


def _slots(rng, kind, rows, D):
    if kind == N.ORX_OPT_SGD:
        return None, None
    if kind == N.ORX_OPT_ADAGRAD:
        return torch.from_numpy((0.1 + rng.random((rows, D))).astype(np.float32)).cuda(), None
    if kind == N.ORX_OPT_ROWWISE_ADAGRAD:
        return torch.from_numpy((0.1 + rng.random(rows)).astype(np.float32)).cuda(), None
    if kind == N.ORX_OPT_MOMENTUM or kind == N.ORX_OPT_NESTEROV:
        return torch.from_numpy((rng.standard_normal((rows, D)) * 0.01).astype(np.float32)).cuda(), None
    m = torch.from_numpy((rng.standard_normal((rows, D)) * 0.01).astype(np.float32)).cuda()
    v = torch.from_numpy((rng.random((rows, D)) * 1e-3 + 1e-5).astype(np.float32)).cuda()
    return m, v


def _ids(rng, ids_mode, rows, n):
    if ids_mode == "unique":
        return rng.permutation(rows)[:n]
    if ids_mode == "single":                 # every lookup one row: all staged
        return np.full(n, rows // 3)
    return (rng.zipf(1.3, n) - 1) % rows     # Zipf: a few hot rows staged, the tail seen once


@pytest.fixture(scope="module")
def apply_eng():
    """A liborx handle of the apply cases' own, closed when they end.  A handle's staging rows are sized for the most
    lookups times the widest row it has seen: on the process-wide handle, which earlier suites size for millions of
    lookups, these D = 256 cases would double that allocation for the rest of the session."""
    eng = N.Engine(torch.cuda.current_device())
    yield eng
    torch.cuda.synchronize()
    eng.close()


def _run_apply(eng, which, tab, s0, s1, kind, ids2d, vals, sparse, col_off, o, seed):
    make = N.table_bf16 if tab.dtype == torch.bfloat16 else N.table
    t = make(tab, s0, s1, kind=kind)
    kw = {"sr_seed": seed} if tab.dtype == torch.bfloat16 else {}
    if which == "strided":
        eng.sparse_apply_strided(t, ids2d, 1, vals, o, **kw)
    else:
        eng.bag_sparse_apply(t, sparse, col_off[1], col_off[2] - col_off[1], vals[:, 1, :],
                             0 if which == "bag_sum" else 1, o, **kw)


def _counts(which, ids2d, sparse, col_off, rows):
    if which == "strided":
        ids = ids2d[:, 1]
    else:
        ids = sparse[:, col_off[1]:col_off[2]].reshape(-1)
    ids = ids[(ids >= 0) & (ids < rows)]
    return np.bincount(ids, minlength=rows)


def _contrib_magnitudes(which, ids2d, sparse, col_off, vals, rows):
    """[rows, D] float64: per table element, the sum of the magnitudes of the gradient contributions the apply adds."""
    v = np.abs(vals[:, 1, :].cpu().numpy().astype(np.float64))
    S = np.zeros((rows, v.shape[1]))
    if which == "strided":
        ids = ids2d[:, 1]
        ok = (ids >= 0) & (ids < rows)
        np.add.at(S, ids[ok], v[ok])
        return S
    bag = sparse[:, col_off[1]:col_off[2]]
    ok = (bag >= 0) & (bag < rows)
    scale = 1.0 / np.maximum(ok.sum(1), 1) if which == "bag_mean" else np.ones(len(bag))
    for l in range(bag.shape[1]):
        m = ok[:, l]
        np.add.at(S, bag[m, l], v[m] * scale[m, None])
    return S


@pytest.mark.parametrize("D", (4, 32, 128, 256, 50))
@pytest.mark.parametrize("opt_name", list(OPTS))
def test_apply_bits_through_rounding(apply_eng, opt_name, D):
    """Every updated element lies in the stochastic-rounding interval of the fp32 apply's result on the upcast table
    (tolerance: a few fp32 ulps on rows applied once, the summation order of staged rows on the others); untouched
    rows keep their bits (not under the dense sweep); slots meet the fp32 apply's.  With table k+1's seed, or at
    step + 1, the same check fails."""
    kind, lr = OPTS[opt_name]
    step = 3
    o = N.opt(kind, lr, 1e-7, 0.9, 0.999, step)
    for case, (which, ids_mode) in enumerate([(w, m) for w in ("strided", "bag_sum", "bag_mean")
                                              for m in ("unique", "zipf", "single")]):
        rng = np.random.default_rng(list(OPTS).index(opt_name) * 10000 + D * 10 + case)
        rows, B = 600, 256
        tab = bf16_table(rng, rows, D, scale=0.3)
        s0, s1 = _slots(rng, kind, rows, D)
        ids2d = np.stack([rng.integers(0, rows, B), _ids(rng, ids_mode, rows, B)], 1).astype(np.int32)
        ids2d[rng.random(B) < 0.05, 1] = -1
        sparse = np.stack([rng.integers(0, rows, B), _ids(rng, ids_mode, rows, B), _ids(rng, ids_mode, rows, B),
                           rng.integers(0, rows, B)], 1).astype(np.int32)
        sparse[rng.random(B) < 0.1, 1] = -1
        sparse[rng.random(B) < 0.05, 2] = rows + 1
        col_off = [0, 1, 3, 4]
        vals = torch.from_numpy((rng.standard_normal((B, 2, D)) * 0.1).astype(np.float32)).cuda()
        seed = table_rounding_seed(11, 5)
        ref, rs0, rs1 = tab.float(), *(None if s is None else s.clone() for s in (s0, s1))
        old = u16(tab)
        ids_t, sp_t = torch.from_numpy(ids2d).cuda(), torch.from_numpy(sparse).cuda()
        _run_apply(apply_eng, which, ref, rs0, rs1, kind, ids_t, vals, sp_t, col_off, o, seed)
        bs0, bs1 = (None if s is None else s.clone() for s in (s0, s1))
        _run_apply(apply_eng, which, tab, bs0, bs1, kind, ids_t, vals, sp_t, col_off, o, seed)
        torch.cuda.synchronize()
        cnt = _counts(which, ids2d, sparse, col_off, rows)
        x = ref.cpu().numpy().astype(np.float64)
        got = BF.up(u16(tab))
        r_ix, c_ix = np.meshgrid(np.arange(rows), np.arange(D), indexing="ij")
        upd = np.ones(rows, bool) if kind == N.ORX_OPT_ADAM_DENSE else cnt > 0
        # A staged row's gradient is summed by float atomics in no fixed order: its float32 sum may differ between the
        # two runs by up to n 2^-24 times the sum of its n contributions' magnitudes (E).  Every optimizer here moves a
        # table element by at most 40 lr per unit of gradient (Adam: lr (1 - beta1) / sqrt(v), v >= 1e-5) and a slot
        # element by at most max(1, 2 |G|).
        S = _contrib_magnitudes(which, ids2d, sparse, col_off, vals, rows)
        E = np.where((cnt > 1)[:, None], cnt[:, None] * 2.0 ** -24 * S, 0.0)
        mag = np.maximum(np.abs(x), BF.up(old))
        tol = np.where((cnt > 1)[:, None], 2.0 ** -14 * mag + 1e-7 + 40 * lr * E, 4 * U23 * mag)

        def inside(sd, st):
            lo, hi = BF.sr_interval(x, tol, sd, st, 0, r_ix, c_ix)
            return (got >= lo) & (got <= hi)
        ok = inside(seed, step)
        where = f"{which}/{ids_mode}"
        assert ok[upd].all(), (where, np.argwhere(~ok & upd[:, None])[:5])
        assert np.array_equal(u16(tab)[~upd], old[~upd]), where
        lo, hi = BF.sr_interval(x, tol, seed, step, 0, r_ix, c_ix)
        changed = upd[:, None] & (BF.up(old) != got) & (lo == hi)   # updated elements whose bits the bar pins
        if changed.sum() > 64:   # negative control: another table's seed, or the next step, selects other bits
            assert not inside(table_rounding_seed(11, 6), step)[changed].all(), where
            assert not inside(seed, step + 1)[changed].all(), where
        for a, b in ((rs0, bs0), (rs1, bs1)):
            if a is None:
                continue
            a, b = a.cpu().numpy(), b.cpu().numpy()
            slot_e = 4 * E * np.maximum(1.0, 2 * S)
            bar = 1e-5 * np.abs(a) + 1e-7 + (slot_e if a.ndim == 2 else slot_e.mean(1))
            assert (np.abs(b.astype(np.float64) - a) <= bar).all(), (where, np.argwhere(np.abs(b - a) > bar)[:5])
            if a.ndim == 2:
                assert np.array_equal(a[cnt == 0], b[cnt == 0]) or kind == N.ORX_OPT_ADAM_DENSE, where


def test_apply_needs_a_seed():
    rng = np.random.default_rng(0)
    tab = bf16_table(rng, 10, 8)
    ids = torch.zeros((2, 2), dtype=torch.int32, device="cuda")
    vals = torch.zeros((2, 2, 8), device="cuda")
    with pytest.raises(ValueError, match="sr_seed"):
        N.engine().sparse_apply_strided(N.table_bf16(tab), ids, 1, vals, N.opt(N.ORX_OPT_SGD, 0.1))


# ---- the model ----------------------------------------------------------------------------------------------------
VOCAB = [40, 25, 60]
SIZES = [2, 1, 3]


def _models(variant, seed=3):
    from openrec_b200.tf2.recommenders import DLRM
    kw = dict(m_spa=8, ln_emb=VOCAB, ln_bot=[16, 8], ln_top=[32, 16, 1], interaction_mode="dlrm")
    if variant == "multihot":
        kw.update(bag_sizes=SIZES, pooling="sum")
    elif variant == "mean":
        kw.update(bag_sizes=SIZES, pooling="mean")
    elif variant == "cross":
        kw.update(arch_interaction_op="cross", cross_layers=2, cross_projection_dim=4)
    elif variant == "reference":
        kw.update(interaction_mode="reference")
    bf = DLRM(embedding_dtype="bfloat16", rounding_seed=seed, **kw)
    fp = DLRM(**kw)
    bf._graph(13)
    fp._graph(13)
    for a, b in zip(fp.trainable_variables, bf.trainable_variables):
        a.t.copy_(b.t.float())
    return bf, fp


def _data(variant, B=256, seed=5):
    rng = np.random.default_rng(seed)
    dense = np.log1p(rng.integers(0, 50, (B, 13))).astype(np.float32)
    if variant in ("multihot", "mean"):
        sp, _ = make_bags(rng, B, SIZES, VOCAB)
    else:
        sp = np.stack([rng.integers(0, V, B) for V in VOCAB], 1).astype(np.int32)
    label = (rng.random(B) < 0.4).astype(np.float32)
    return dense, sp, label


def _touch_counts(variant, sp, k):
    if variant in ("multihot", "mean"):
        c = np.concatenate([[0], np.cumsum(SIZES)])
        ids = sp[:, c[k]:c[k + 1]].reshape(-1)
    else:
        ids = sp[:, k]
    ids = ids[(ids >= 0) & (ids < VOCAB[k])]
    return np.bincount(ids, minlength=VOCAB[k])


@pytest.mark.parametrize("variant", ("onehot", "multihot", "mean", "reference", "cross"))
def test_model_forward_and_slices_equal_fp32_on_upcast(tf, variant):
    bf, fp = _models(variant)
    dense, sp, label = _data(variant)
    assert np.array_equal(i32bits(bf.inference(dense, sp).t), i32bits(fp.inference(dense, sp).t))
    with tf.GradientTape() as t1:
        l1 = bf(dense, sp, label)
    with tf.GradientTape() as t2:
        l2 = fp(dense, sp, label)
    assert np.float32(float(l1)).view(np.int32) == np.float32(float(l2)).view(np.int32)
    g1 = t1.gradient(l1, bf.trainable_variables)
    g2 = t2.gradient(l2, fp.trainable_variables)
    for k in range(len(VOCAB)):
        assert np.array_equal(np.asarray(g1[k].indices.numpy()), np.asarray(g2[k].indices.numpy()))
        v1, v2 = np.asarray(g1[k].values.numpy()), np.asarray(g2[k].values.numpy())
        assert v1.dtype == np.float32 and np.array_equal(v1.view(np.int32), v2.view(np.int32))


@pytest.mark.parametrize("opt_name", ("adagrad", "adam"))
@pytest.mark.parametrize("variant", ("onehot", "multihot", "reference", "cross"))
def test_model_step_rounds_the_fp32_step(tf, variant, opt_name):
    bf, fp = _models(variant, seed=17)
    dense, sp, label = _data(variant, seed=9)
    mk = (lambda: tf.keras.optimizers.Adagrad(learning_rate=0.05)) if opt_name == "adagrad" else \
        (lambda: tf.keras.optimizers.Adam())
    o1, o2 = mk(), mk()
    before = [u16(v.t) for v in bf.trainable_variables[:len(VOCAB)]]
    for m, o in ((bf, o1), (fp, o2)):
        with tf.GradientTape() as tape:
            loss = m(dense, sp, label)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
    T = len(VOCAB)
    for a, b in zip(bf.trainable_variables[T:], fp.trainable_variables[T:]):
        assert np.array_equal(i32bits(a.t), i32bits(b.t)), a.name
    eng = N.engine()
    step = o1.iterations
    for k in range(T):
        got, ref = bf.trainable_variables[k].t, fp.trainable_variables[k].t
        D = ref.shape[1]
        seed = table_rounding_seed(17, k)
        exp = u16(eng.debug_round_bf16(ref.contiguous(), 0, D, 0, seed, step))
        g = u16(got)
        cnt = _touch_counts(variant, sp, k)
        once = cnt == 1 if opt_name == "adagrad" else cnt <= 1       # Adam's sweep rewrites the untouched rows too
        assert np.array_equal(g[once], exp[once]), (k, np.argwhere(g[once] != exp[once])[:5])
        many = cnt > 1
        x = ref.cpu().numpy().astype(np.float64)
        r_ix, c_ix = np.meshgrid(np.arange(ref.shape[0]), np.arange(D), indexing="ij")
        lo, hi = BF.sr_interval(x, 8 * U23 * np.abs(x) + 1e-12, seed, step, 0, r_ix, c_ix)
        gv = BF.up(g)
        assert ((gv >= lo) & (gv <= hi))[many].all(), k
        if opt_name == "adagrad":
            assert np.array_equal(g[cnt == 0], before[k][cnt == 0]), k
        assert bf.trainable_variables[k].t.dtype == torch.bfloat16


def test_model_two_runs_bit_identical(tf):
    runs = []
    for _ in range(2):
        bf, _ = _models("multihot", seed=21)
        if runs:
            for a, b in zip(bf.trainable_variables, runs[0][0]):
                a.t.copy_(b)
        else:
            runs.append(([v.t.clone() for v in bf.trainable_variables], None))
        opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
        for s in range(3):
            dense, sp, label = _data("multihot", seed=30 + s)
            with tf.GradientTape() as tape:
                loss = bf(dense, sp, label)
            opt.apply_gradients(zip(tape.gradient(loss, bf.trainable_variables), bf.trainable_variables))
        runs.append([v.t.clone() for v in bf.trainable_variables])
    for a, b in zip(runs[1], runs[2]):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a,
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b)


def test_checkpoint_round_trip_and_dtype_refusal(tf, tmp_path):
    from openrec_b200.tf2 import checkpoint
    from openrec_b200.tf2.recommenders import DLRM
    kw = dict(m_spa=8, ln_emb=VOCAB, ln_bot=[16, 8], ln_top=[32, 16, 1])
    model = DLRM(embedding_dtype="bfloat16", rounding_seed=2, **kw)
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    dense, sp, label = _data("onehot")
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, model.trainable_variables), model.trainable_variables))
    path = str(tmp_path / "ck.npz")
    checkpoint.save(path, model, opt)
    other = DLRM(embedding_dtype="bfloat16", **kw)
    other._graph(13)
    opt2 = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    checkpoint.load(path, other, opt2)
    for a, b in zip(model.variables, other.variables):
        assert a.t.dtype == b.t.dtype
        assert torch.equal(a.t.view(torch.int16) if a.t.dtype == torch.bfloat16 else a.t,
                           b.t.view(torch.int16) if b.t.dtype == torch.bfloat16 else b.t)
    for v, w in zip(model.variables, other.variables):
        for s, t in zip(opt.slots_if_any(v), opt2.slots_if_any(w)):
            assert (s is None and t is None) or torch.equal(s, t)
    fp = DLRM(**kw)
    fp._graph(13)
    with pytest.raises(ValueError):
        checkpoint.load(path, fp)


def test_reference_example_flow_on_bf16_tables(tf):
    """tf2_examples/dlrm_criteo.py's control flow (m_spa = 4, bottom [8, 4], top [128, 64, 1], Keras Adam(), the AUC
    metric) on bf16 tables and seeded synthetic Criteo-shaped arrays."""
    from openrec_b200.tf2.recommenders import DLRM
    rng = np.random.default_rng(42)
    counts = [int(c) for c in rng.integers(3, 5000, 26)]
    B = 1024
    model = DLRM(m_spa=4, ln_emb=counts, ln_bot=[8, 4], ln_top=[128, 64, 1], embedding_dtype="bfloat16")
    optimizer = tf.keras.optimizers.Adam()
    auc = tf.keras.metrics.AUC()

    def batch():
        dense = np.log1p(rng.integers(0, 1000, (B, 13))).astype(np.float32)
        sparse = np.stack([rng.integers(0, c, B) for c in counts], 1).astype(np.int64)
        label = (rng.random(B) < 0.25).astype(np.float32)
        return dense, sparse, label
    for _ in range(5):
        d, s, y = batch()
        with tf.GradientTape() as tape:
            loss_value = model(d, s, y)
        gradients = tape.gradient(loss_value, model.trainable_variables)
        optimizer.apply_gradients(zip(gradients, model.trainable_variables))
        assert np.isfinite(float(loss_value))
    for _ in range(2):
        d, s, y = batch()
        auc.update_state(y_true=y, y_pred=model.inference(d, s))
    a = float(auc.result().numpy())
    assert np.isfinite(a) and 0.0 <= a <= 1.0
    assert model.trainable_variables[0].t.dtype == torch.bfloat16
