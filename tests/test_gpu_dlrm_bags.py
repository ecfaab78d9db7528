"""GPU: multi-hot DLRM features -- orx_bag_gather, orx_bag_sparse_apply and DLRM(bag_sizes=...) against the numpy
restatement in tests/dlrm_bags_np.py (float32 pooling in the kernel's order for exact checks, the float64 oracle for
training)."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest
import torch

import dlrm_bags_np as NB
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def close(t, ref, atol=1e-5, rtol=1e-5):
    got = t.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(t) else np.asarray(t, dtype=np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def make_bags(rng, B, sizes, vocab, pad=0.2, bad=0.05, dup=0.1):
    """[B, sum(sizes)] int32 bags with padding (-1) at the start, the end and in between, all-padding bags, ids past
    the vocabulary and repeated ids inside a bag."""
    col_off = NB.col_offsets(sizes)
    sp = np.empty((B, col_off[-1]), np.int32)
    for k, (Lk, V) in enumerate(zip(sizes, vocab)):
        ids = rng.integers(0, V, (B, Lk))
        u = rng.random((B, Lk))
        ids[u < pad] = -1
        ids[(u >= pad) & (u < pad + bad)] = V + rng.integers(0, 3, int(((u >= pad) & (u < pad + bad)).sum()))
        if Lk > 1:
            d = rng.random(B) < dup
            ids[d, 1] = ids[d, 0]
        ids[rng.random(B) < 0.05] = -1              # whole bags of padding
        sp[:, col_off[k]:col_off[k + 1]] = ids
    return sp, col_off


def tables(rng, vocab, D, neg_zero=False):
    out = [rng.standard_normal((V, D)).astype(np.float32) for V in vocab]
    if neg_zero:
        for t in out:
            t[::3, ::2] = -0.0
    return out


def gather(tabs_t, sp_t, col_off, mode, out_ld=None, offset=0, n_bad=None):
    B, T, D = sp_t.shape[0], len(tabs_t), tabs_t[0].shape[1]
    ld = out_ld or T * D
    buf = torch.full((B * ld + offset + 4,), float("nan"), device="cuda")
    out = buf[offset:offset + B * ld].view(B, ld)
    N.engine().bag_gather(tabs_t, sp_t, col_off, mode, out, n_bad)
    return out, buf


# ---- orx_bag_gather ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 3, 4, 16, 50, 64, 128, 256, 512])
@pytest.mark.parametrize("mean", [0, 1])
def test_bag_gather_grid(D, mean):
    """Every bag size of the grid in one launch (L = 1, 2, 7, 32, 33, 100), B with a tail; bit-exact vs the float32
    restatement, n_bad exact."""
    rng = np.random.default_rng(D * 2 + mean)
    sizes, vocab = [1, 2, 7, 32, 33, 100], [50, 301, 17, 1000, 64, 5000]
    B = 37
    sp, col_off = make_bags(rng, B, sizes, vocab)
    tabs = tables(rng, vocab, D, neg_zero=True)
    nb = torch.zeros(1, dtype=torch.int32, device="cuda")
    out, _ = gather([dev(t) for t in tabs], dev(sp, torch.int32), col_off, mean, n_bad=nb)
    Z, _, bad = NB.pool_f32(tabs, sp, col_off, mean)
    np.testing.assert_array_equal(bits(out.cpu().numpy()), bits(Z.reshape(B, -1)))
    assert int(nb) == bad and bad > 0


@pytest.mark.parametrize("D,out_extra,offset", [(128, 8, 0), (128, 0, 1), (16, 3, 0), (5, 2, 1)])
@pytest.mark.parametrize("B", [1, 129])
def test_bag_gather_layout(D, out_extra, offset, B):
    """out_ld > T*D (the padding columns are not written) and a misaligned out (the scalar path)."""
    rng = np.random.default_rng(D + B)
    sizes, vocab = [3, 1, 40], [100, 7, 900]
    sp, col_off = make_bags(rng, B, sizes, vocab)
    tabs = tables(rng, vocab, D)
    T = len(sizes)
    for mean in (0, 1):
        out, buf = gather([dev(t) for t in tabs], dev(sp, torch.int32), col_off, mean, T * D + out_extra, offset)
        Z, _, _ = NB.pool_f32(tabs, sp, col_off, mean)
        o = out.cpu().numpy()
        np.testing.assert_array_equal(bits(o[:, :T * D]), bits(Z.reshape(B, -1)))
        assert np.isnan(o[:, T * D:]).all() and torch.isnan(buf[:offset]).all()


def test_bag_gather_empty_batch():
    t = torch.ones(4, 8, device="cuda")
    out = torch.full((0, 8), 7.0, device="cuda")
    N.engine().bag_gather([t], torch.empty(0, 2, dtype=torch.int32, device="cuda"), [0, 2], 0, out)
    torch.cuda.synchronize()


@pytest.mark.parametrize("D", [4, 7, 128])
def test_bag_gather_one_hot_equals_gather_strided(D):
    """L = 1 everywhere: bit-equal to T orx_gather_strided calls, -0.0 rows and out-of-range ids included."""
    rng = np.random.default_rng(D)
    vocab, B = [30, 1, 200, 5], 300
    T = len(vocab)
    tabs = tables(rng, vocab, D, neg_zero=True)
    sp = np.stack([rng.integers(0, V + 3, B) for V in vocab], 1).astype(np.int32)
    tt, spt = [dev(t) for t in tabs], dev(sp, torch.int32)
    eng = N.engine()
    ref = torch.empty(B, T, D, device="cuda")
    for k in range(T):
        eng.gather_strided(tt[k], spt, k, ref[:, k, :])
    for mean in (0, 1):
        out, _ = gather(tt, spt, list(range(T + 1)), mean)
        np.testing.assert_array_equal(bits(out.cpu().numpy()), bits(ref.reshape(B, -1).cpu().numpy()))


def test_bag_gather_refusals():
    eng = N.engine()
    lib = eng.lib
    t = torch.zeros(10, 4, device="cuda")
    sp = torch.zeros(3, 64, dtype=torch.int32, device="cuda")
    out = torch.zeros(3, 64 * 4, device="cuda")

    def call(T=1, col=(0, 5), ld=5, out_ld=4, mode=0, tab=True, sparse=True, o=True, rows=10, dim=4, B=3):
        ptrs = (C.c_void_p * max(T, 1))(*([t.data_ptr() if tab else None] * max(T, 1)))
        rws = (C.c_int64 * max(T, 1))(*([rows] * max(T, 1)))
        off = (C.c_int32 * len(col))(*col)
        return lib.orx_bag_gather(eng.h, ptrs, rws, T, dim, C.c_void_p(sp.data_ptr()) if sparse else None, ld, off, B,
                                  mode, C.c_void_p(out.data_ptr()) if o else None, out_ld, None, eng.stream())

    assert call() == 0
    bad = [dict(T=0, col=(0,)), dict(T=64, col=tuple(range(65)), ld=64), dict(T=2, col=(0, 3, 2)),
           dict(col=(0, 6)), dict(col=(-1, 2)), dict(T=2, col=(0, 2, 4), out_ld=7), dict(mode=2), dict(tab=False),
           dict(sparse=False), dict(o=False), dict(rows=0), dict(dim=0), dict(B=-1), dict(ld=0, col=(0, 0))]
    for kw in bad:
        assert call(**kw) == -1, kw
    assert call(T=63, col=tuple(range(64)), ld=64, out_ld=63 * 4) == 0
    torch.cuda.synchronize()


# ---- orx_bag_sparse_apply ---------------------------------------------------------------------------------------
OPTS = [("sgd", L.ORX_OPT_SGD, 1), ("adagrad", L.ORX_OPT_ADAGRAD, 1), ("lazy", L.ORX_OPT_ADAM_LAZY, 1),
        ("adam1", L.ORX_OPT_ADAM_DENSE, 1), ("adam7", L.ORX_OPT_ADAM_DENSE, 7)]


def _case_bags(rng, case, B, Lk, V):
    if case == "hot":          # one id in every bag: every row staged, the hot one many times
        sp = rng.integers(0, V, (B, Lk))
        sp[:, rng.integers(0, Lk)] = 3
        sp[rng.random((B, Lk)) < 0.15] = -1
        sp[rng.random((B, Lk)) < 0.05] = V + 1
    elif case == "once":       # every row seen once (rows >> lookups), padding and bad ids around them
        sp = rng.permutation(V)[:B * Lk].reshape(B, Lk)
        sp[rng.random((B, Lk)) < 0.2] = -1
        sp[rng.random((B, Lk)) < 0.05] = V + 2
    else:                      # every row staged: each id appears twice
        half = rng.permutation(V)[:(B * Lk + 1) // 2]
        sp = np.concatenate([half, half])[:B * Lk]
        sp = rng.permutation(sp).reshape(B, Lk)
        sp[-1, -1] = sp[0, 0]
    return sp.astype(np.int32)


@pytest.mark.parametrize("name,kind,step", OPTS)
@pytest.mark.parametrize("mean", [0, 1])
@pytest.mark.parametrize("case", ["hot", "once", "staged"])
def test_bag_sparse_apply(name, kind, step, mean, case):
    rng = np.random.default_rng(zlib.crc32(f"{name}{mean}{case}".encode()))
    B, Lk, V, D, lo, extra = 97, 7, 300 if case == "hot" else 4000, 36, 2, 3
    bags = _case_bags(rng, case, B, Lk, V)
    sp = rng.integers(-1, V, (B, lo + Lk + extra)).astype(np.int32)      # other tables' columns around the bag
    sp[:, lo:lo + Lk] = bags
    T, k = 3, 1
    dZ = rng.standard_normal((B, T, D)).astype(np.float32)
    var = rng.standard_normal((V, D)).astype(np.float32)
    s0 = (np.full_like(var, 0.1) if kind == L.ORX_OPT_ADAGRAD else rng.random((V, D)).astype(np.float32) * 0.01)
    s1 = rng.random((V, D)).astype(np.float32) * 0.01
    tv, ts0, ts1 = dev(var), dev(s0), dev(s1)
    tab = N.table(tv, None if kind == L.ORX_OPT_SGD else ts0, ts1 if kind in (L.ORX_OPT_ADAM_LAZY,
                                                                               L.ORX_OPT_ADAM_DENSE) else None)
    lr = 0.05
    tdz = dev(dZ)
    N.engine().bag_sparse_apply(tab, dev(sp, torch.int32), lo, Lk, tdz[:, k, :], mean, N.opt(kind, lr, step=step))
    ids, vals = NB.bag_slices(sp, [0, lo, lo + Lk], 1, V, dZ[:, k, :].astype(np.float64), mean)
    r, r0, r1 = var.astype(np.float64), s0.astype(np.float64), s1.astype(np.float64)
    O.apply_sparse(kind, r, r0, r1, ids, vals, step, lr)
    close(tv, r, atol=2e-5)
    if kind != L.ORX_OPT_SGD:
        close(ts0, r0, atol=2e-5)
    if kind in (L.ORX_OPT_ADAM_LAZY, L.ORX_OPT_ADAM_DENSE):
        close(ts1, r1, atol=2e-5)
    if kind != L.ORX_OPT_ADAM_DENSE:      # rows not named (padding / bad ids name none) keep every bit
        untouched = np.setdiff1d(np.arange(V), ids)
        assert len(untouched) > 0
        u = torch.from_numpy(untouched).cuda()
        for t, ref in ((tv, var), (ts0, s0), (ts1, s1)):
            np.testing.assert_array_equal(bits(t[u].cpu().numpy()), bits(ref[untouched]))


@pytest.mark.parametrize("kind", [L.ORX_OPT_SGD, L.ORX_OPT_ADAGRAD, L.ORX_OPT_ADAM_LAZY, L.ORX_OPT_ADAM_DENSE])
@pytest.mark.parametrize("D", [64, 13])
def test_bag_sparse_apply_one_hot_equals_strided(kind, D):
    """L = 1, sum: orx_sparse_apply_strided on the same column -- bit-equal on rows seen once, fp32 RED order on
    staged rows."""
    rng = np.random.default_rng(kind * 10 + D)
    B, T, V, k = 2000, 4, 5000, 2
    sp = rng.integers(-1, V + 2, (B, T)).astype(np.int32)
    dZ = dev(rng.standard_normal((B, T, D)).astype(np.float32))
    init = [rng.standard_normal((V, D)).astype(np.float32)] + [rng.random((V, D)).astype(np.float32) * 0.1] * 2
    spt = dev(sp, torch.int32)
    res = []
    for bag in (True, False):
        tv, ts0, ts1 = (dev(a) for a in init)
        tab = N.table(tv, None if kind == L.ORX_OPT_SGD else ts0,
                      ts1 if kind in (L.ORX_OPT_ADAM_LAZY, L.ORX_OPT_ADAM_DENSE) else None)
        o = N.opt(kind, 0.05, step=3)
        if bag:
            N.engine().bag_sparse_apply(tab, spt, k, 1, dZ[:, k, :], 0, o)
        else:
            N.engine().sparse_apply_strided(tab, spt, k, dZ, o)
        res.append([t.cpu().numpy() for t in (tv, ts0, ts1)])
    col = sp[:, k]
    ids, cnt = np.unique(col[(col >= 0) & (col < V)], return_counts=True)
    once, staged = ids[cnt == 1], ids[cnt > 1]
    for a, b in zip(*res):
        np.testing.assert_array_equal(bits(a[once]), bits(b[once]))
        np.testing.assert_allclose(a[staged], b[staged], atol=1e-5, rtol=1e-5)
        if kind != L.ORX_OPT_ADAM_DENSE:
            np.testing.assert_array_equal(bits(a), bits(np.where(np.isin(np.arange(V), staged)[:, None], a, b)))


def test_bag_sparse_apply_refusals():
    eng = N.engine()
    lib = eng.lib
    var, s0 = torch.zeros(10, 4, device="cuda"), torch.zeros(10, 4, device="cuda")
    sp = torch.zeros(3, 5, dtype=torch.int32, device="cuda")
    dz = torch.zeros(3, 8, device="cuda")

    def call(tab=None, col_lo=0, Lk=2, ld=5, B=3, dz_ld=8, mode=0, kind=L.ORX_OPT_ADAGRAD, sparse=True, d=True):
        tab = tab or N.table(var, s0)
        return lib.orx_bag_sparse_apply(eng.h, C.byref(tab), C.c_void_p(sp.data_ptr()) if sparse else None, ld,
                                        col_lo, Lk, B, C.c_void_p(dz.data_ptr()) if d else None, dz_ld, mode,
                                        C.byref(N.opt(kind, 0.1)), eng.stream())

    assert call() == 0
    for kw in [dict(Lk=0), dict(col_lo=-1), dict(col_lo=4), dict(dz_ld=3), dict(mode=2), dict(B=-1), dict(kind=7),
               dict(tab=N.table(var)), dict(sparse=False), dict(d=False), dict(Lk=1 << 20, B=1 << 12, ld=1 << 21)]:
        assert call(**kw) == -1, kw
    assert lib.orx_bag_sparse_apply(eng.h, None, None, 5, 0, 1, 0, None, 8, 0, C.byref(N.opt(0, 0.1)),
                                    eng.stream()) == -1
    torch.cuda.synchronize()


# ---- the model ----------------------------------------------------------------------------------------------------
SIZES, VOCAB = [3, 1, 7, 2], [50, 31, 77, 20]


def _model_data(rng, B):
    sp, col_off = make_bags(rng, B, SIZES, VOCAB)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    label = (rng.random(B) < 0.3).astype(np.float32)
    return dense, sp.astype(np.int64), label, col_off


def _model(mode, pooling, m_spa=16, **kw):
    from openrec.tf2.recommenders import DLRM
    return DLRM(m_spa=m_spa, ln_emb=VOCAB, ln_bot=[32, m_spa], ln_top=[64, 32, 1], interaction_mode=mode,
                bag_sizes=SIZES, pooling=pooling, **kw)


def _opt(tf, name):
    from openrec_b200.tfshim.keras.optimizers import LazyAdam
    return {"adam": (tf.keras.optimizers.Adam(), O.OPT_ADAM_DENSE),
            "lazy": (LazyAdam(), O.OPT_ADAM_LAZY),
            "sgd": (tf.keras.optimizers.SGD(learning_rate=0.1), O.OPT_SGD),
            "adagrad": (tf.keras.optimizers.Adagrad(learning_rate=0.05), O.OPT_ADAGRAD)}[name]


@pytest.mark.parametrize("optname", ["sgd", "adagrad", "lazy", "adam"])
@pytest.mark.parametrize("mode", ["reference", "dlrm"])
@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_dlrm_bags_training_step(tf, optname, mode, pooling):
    rng = np.random.default_rng(len(optname) * 7 + len(mode) + len(pooling))
    B = 256
    model = _model(mode, pooling)
    dense, sp, label, col_off = _model_data(rng, B)
    model._graph(13)
    tv = model.trainable_variables
    T = len(VOCAB)
    var = [v.numpy().astype(np.float64) for v in tv]
    opt, kind = _opt(tf, optname)
    st = [(np.full_like(v, 0.1), None) if kind == O.OPT_ADAGRAD else (np.zeros_like(v), np.zeros_like(v))
          for v in var]
    for step in (1, 2):
        with tf.GradientTape() as tape:
            loss = model(dense, sp, label)
        opt.apply_gradients(zip(tape.gradient(loss, tv), tv))
        rl = NB.train_step(kind, var[:T], var[T:], st, step, opt.learning_rate, dense.astype(np.float64), sp, label,
                           col_off, pooling == "mean", mode, 2)
        close(float(loss), rl, atol=2e-6)
        for j, (v, ref) in enumerate(zip(tv, var)):
            close(v.numpy(), ref, atol=2e-5)
            s0, s1 = opt.slots(v)
            if kind != O.OPT_SGD:
                close(s0, st[j][0], atol=2e-5)
            if kind in (O.OPT_ADAM_LAZY, O.OPT_ADAM_DENSE):
                close(s1, st[j][1], atol=2e-5)


@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_dlrm_bags_inference_and_gradients(tf, pooling):
    """inference = the oracle forward; explicit tape.gradient IndexedSlices = the oracle's (valid ids in (b, l) order,
    rows scaled for a mean)."""
    rng = np.random.default_rng(5)
    B, T = 200, len(VOCAB)
    model = _model("dlrm", pooling)
    dense, sp, label, col_off = _model_data(rng, B)
    model._graph(13)
    tv = model.trainable_variables
    var = [v.numpy().astype(np.float64) for v in tv]
    mean = pooling == "mean"
    rest = var[T:]
    cache, pooled, ar = NB.forward(var[:T], rest[0:4:2], rest[1:4:2], rest[4::2], rest[5::2],
                                   dense.astype(np.float64), sp, col_off, mean, "dlrm")
    close(model.inference(dense, sp).numpy(), cache["pred"], atol=2e-6)
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    grads = tape.gradient(loss, tv)
    rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = O.dlrm_backward(cache, pooled, rest[0:4:2], rest[4::2], dense.astype(np.float64), ar, dpred,
                         interaction_mode="dlrm")
    close(float(loss), rl, atol=2e-6)
    for k in range(T):
        ids, vals = NB.bag_slices(sp, col_off, k, VOCAB[k], gr["emb"][k], mean)
        np.testing.assert_array_equal(grads[k].indices.numpy(), ids)
        close(grads[k].values.numpy(), vals, atol=2e-6)


def test_dlrm_bags_checkpoint_round_trip(tf, tmp_path):
    from openrec_b200.tf2 import checkpoint
    rng = np.random.default_rng(8)
    dense, sp, label, _ = _model_data(rng, 64)
    a, opt = _model("dlrm", "mean"), tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = a(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, a.trainable_variables), a.trainable_variables))
    checkpoint.save(str(tmp_path / "bags.npz"), a, opt)
    b, opt2 = _model("dlrm", "mean"), tf.keras.optimizers.Adagrad(learning_rate=0.05)
    b._graph(13)                                     # the Dense layers exist after the first call
    checkpoint.load(str(tmp_path / "bags.npz"), b, opt2)
    for x, y in zip(a.variables, b.variables):
        assert torch.equal(x.t, y.t)
    for m, o in ((a, opt), (b, opt2)):
        with tf.GradientTape() as tape:
            loss = m(dense, sp, label)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
    for x, y in zip(a.variables, b.variables):
        assert torch.equal(x.t, y.t)
    assert torch.equal(a.inference(dense, sp).t, b.inference(dense, sp).t)


@pytest.mark.parametrize("optname", ["adagrad", "adam"])
def test_dlrm_one_id_bags_train_like_one_hot(tf, optname):
    """bag_sizes = [1] * T from the same weights: the same losses and tables as the one-hot DLRM."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(9)
    B = 300
    kw = dict(m_spa=8, ln_emb=VOCAB, ln_bot=[16, 8], ln_top=[32, 1], interaction_mode="dlrm")
    one, bag = DLRM(**kw), DLRM(bag_sizes=[1] * len(VOCAB), **kw)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sp = np.stack([rng.integers(0, V, B) for V in VOCAB], 1)
    label = (rng.random(B) < 0.3).astype(np.float32)
    one._graph(13), bag._graph(13)
    for x, y in zip(one.trainable_variables, bag.trainable_variables):
        y.assign(x.numpy())
    opts = [_opt(tf, optname)[0] for _ in range(2)]
    for _ in range(3):
        losses = []
        for m, o in zip((one, bag), opts):
            with tf.GradientTape() as tape:
                loss = m(dense, sp, label)
            o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
            losses.append(float(loss))
        close(losses[1], losses[0], atol=1e-6, rtol=1e-6)   # staged rows: fp32 RED order may differ after step 1
        for x, y in zip(one.trainable_variables, bag.trainable_variables):
            close(y.numpy(), x.numpy(), atol=1e-6, rtol=1e-6)


def test_dlrm_bags_value_errors(tf):
    from openrec.tf2.recommenders import DLRM
    kw = dict(m_spa=8, ln_emb=[10, 20], ln_bot=[8], ln_top=[4, 1])
    for bad in (dict(bag_sizes=[1]), dict(bag_sizes=[2, 0]), dict(bag_sizes=[1, 1], pooling="max"),
                dict(pooling="sqrtn")):
        with pytest.raises(ValueError):
            DLRM(**kw, **bad)
    m = DLRM(bag_sizes=[2, 3], **kw)
    dense = np.zeros((4, 13), np.float32)
    for width in (4, 6, 2):
        with pytest.raises(ValueError):
            m(dense, np.zeros((4, width), np.int64), np.zeros(4, np.float32))
        with pytest.raises(ValueError):
            m.inference(dense, np.zeros((4, width), np.int64))
    m(dense, np.zeros((4, 5), np.int64), np.zeros(4, np.float32))


# ---- full shape ---------------------------------------------------------------------------------------------------
MLPERF_BAGS = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]


def test_dlrm_bags_full_shape_training_step(tf):
    """bench.py's DLRM shape (26 x 1M x 128, B = 32768, Adagrad) with the MLPerf DLRM-DCNv2 multi-hot sizes (214 ids
    per sample): one step against the float64 oracle on the touched rows."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(34)
    B, m_spa, T = 32768, 128, 26
    ln_emb, ln_bot, ln_top = [1_000_000] * T, [512, 256, 128], [1024, 1024, 512, 256, 1]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=ln_bot, ln_top=ln_top, interaction_mode="dlrm",
                 bag_sizes=MLPERF_BAGS, pooling="sum")
    col_off = NB.col_offsets(MLPERF_BAGS)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sp = rng.integers(0, 1_000_000, (B, int(col_off[-1]))).astype(np.int64)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    rows, csp, tabs = [], np.zeros_like(sp), []
    for k in range(T):                              # compact oracle problem: the touched rows of every table
        cols = sp[:, col_off[k]:col_off[k + 1]]
        r = np.unique(cols)
        rows.append(r)
        csp[:, col_off[k]:col_off[k + 1]] = np.searchsorted(r, cols)
        tabs.append(tv[k].t[torch.from_numpy(r).cuda()].cpu().numpy().astype(np.float64))
    untouched = [int(np.setdiff1d(np.arange(2000), rows[k])[0]) for k in (0, 20)]
    before = [tv[k].t[u].clone() for k, u in zip((0, 20), untouched)]
    dvars = [v.numpy().astype(np.float64) for v in tv[T:]]
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, tv), tv))
    checked = (0, 9, 20, T - 1)
    st = [(np.full_like(v, 0.1) if k in checked or k >= T else None, None) for k, v in enumerate(tabs + dvars)]
    rl = NB.train_step(O.OPT_ADAGRAD, tabs, dvars, st, 1, 0.05, dense.astype(np.float64), csp, label, col_off, False,
                       "dlrm", len(ln_bot), apply_tables=checked)
    close(float(loss), rl, atol=2e-6)
    for j, ref in enumerate(dvars):
        close(tv[T + j].numpy(), ref, atol=2e-5)
    for k in checked:
        close(tv[k].t[torch.from_numpy(rows[k]).cuda()], tabs[k], atol=2e-5)
    for k, u, b in zip((0, 20), untouched, before):
        assert torch.equal(tv[k].t[u], b)
