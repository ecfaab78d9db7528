"""GPU: the DCN-v2 cross network -- orx_cross_fwd / orx_cross_bwd on both paths against float64, DLRM(arch_interaction_op=
"cross") steps against the restatement in tests/dcn_np.py, the other model paths, ShardedDLRM's loopback ranks against
the single-GPU model, and one step at bench.py's DLRM shape."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import dcn_np as X
import dlrm_bags_np as NB
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VEC, SCALAR = L.ORX_VARIANT_CROSS_VEC, L.ORX_VARIANT_CROSS_SCALAR
TOP, MID, FINAL = L.ORX_CROSS_TOP, L.ORX_CROSS_MID, L.ORX_CROSS_FINAL


@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def close(t, ref, atol=1e-5, rtol=1e-5):
    got = t.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(t) else np.asarray(t, dtype=np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol)


def f64(t):
    return t.detach().cpu().numpy().astype(np.float64)


# ---- kernels ------------------------------------------------------------------------------------------------------
def operand(rng, B, W, pad, off, fill=None):
    """A [B, W] view with row stride W + pad starting `off` floats into a NaN-filled buffer (off 1: 4 bytes past a
    16-byte boundary).  fill=None: random values."""
    ld = W + pad
    buf = torch.full((off + B * ld + 4,), float("nan"), device="cuda")
    v = buf[off:off + B * ld].view(B, ld)[:, :W]
    if fill is None:
        v.copy_(torch.from_numpy(rng.standard_normal((B, W)).astype(np.float32)))
    else:
        v.fill_(fill)
    return v, buf


def one_ulp_bar(ref):
    """float32 rounding of one operation on a float64 reference (round-to-nearest: half an ulp, with margin)."""
    return np.abs(ref) * 2.0 ** -23 + 1e-38


def assert_rounded(t, ref):
    got = f64(t)
    assert np.all(np.abs(got - ref) <= one_ulp_bar(ref)), float(np.max(np.abs(got - ref) / one_ulp_bar(ref)))


def untouched(buf, views):
    """Every buffer element outside the views is still NaN."""
    mask = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
    for v in views:
        base = (v.data_ptr() - buf.data_ptr()) // 4
        idx = base + torch.arange(v.shape[0], device="cuda")[:, None] * v.stride(0) + torch.arange(v.shape[1],
                                                                                                   device="cuda")
        mask[idx.reshape(-1)] = False
    return bool(torch.isnan(buf[mask]).all())


LAYOUTS = [  # W, row padding, base offset (floats) -> the path orx_cross_* must take
    (64, 0, 0, VEC), (128, 4, 0, VEC), (3456, 0, 0, VEC), (12, 8, 4, VEC),
    (64, 1, 0, SCALAR), (64, 0, 1, SCALAR), (5, 3, 0, SCALAR), (1, 0, 0, SCALAR), (130, 2, 1, SCALAR)]


@pytest.mark.parametrize("W,pad,off,variant", LAYOUTS)
@pytest.mark.parametrize("B", [1, 37])
def test_cross_fwd(W, pad, off, variant, B):
    eng = N.engine()
    rng = np.random.default_rng(W * 7 + pad + off + B)
    (x0, b0), (xl, b1), (y, b2), (out, b3) = (operand(rng, B, W, pad, off, None if k < 3 else float("nan"))
                                              for k in range(4))
    eng.debug_dispatch_log()
    eng.cross_fwd(x0, xl, y, out)
    assert eng.debug_dispatch_log() == [N.Dispatch(L.ORX_OP_CROSS, variant, 0, 0, B, W, 0, 1)]
    assert_rounded(out, f64(x0) * f64(y) + f64(xl))                     # one fused multiply-add per element
    assert untouched(b3, [out])
    again = torch.empty_like(out)
    eng.cross_fwd(x0, xl, y, again)
    assert torch.equal(again, out)


@pytest.mark.parametrize("W,pad,off,variant", LAYOUTS)
@pytest.mark.parametrize("mode", [TOP, MID])
def test_cross_bwd_layer(W, pad, off, variant, mode):
    """TOP: dy = G x0, A = G y (G untouched); MID: g = G + P, dy = g x0, A += g y, G <- g."""
    eng = N.engine()
    B = 29
    rng = np.random.default_rng(W + pad * 3 + off + mode)
    (G, bG), (P, _), (x0, _), (y, _), (A, bA), (dy, bdy) = (operand(rng, B, W, pad, off) for _ in range(6))
    G0, P0, x00, y0, A0 = (f64(t) for t in (G, P, x0, y, A))
    eng.debug_dispatch_log()
    eng.cross_bwd(mode, G, A, P=P, x0=x0, y=y, dy=dy)
    assert eng.debug_dispatch_log() == [N.Dispatch(L.ORX_OP_CROSS, variant, 1, mode, B, W, 0, 1)]
    if mode == TOP:
        assert np.array_equal(f64(G), G0)
        assert_rounded(dy, G0 * x00)
        assert_rounded(A, G0 * y0)
    else:
        g = f64(G)
        assert_rounded(G, G0 + P0)
        assert_rounded(dy, g * x00)                                      # from the rounded g
        assert_rounded(A, g * y0 + A0)
    for buf, v in ((bG, G), (bA, A), (bdy, dy)):
        assert untouched(buf, [v])


@pytest.mark.parametrize("W,D,pad,off,variant", [
    (3456, 128, 0, 0, VEC), (64, 16, 4, 0, VEC), (64, 0, 0, 0, VEC), (64, 64, 0, 0, VEC),
    (64, 18, 0, 0, SCALAR), (64, 16, 0, 1, SCALAR), (15, 5, 1, 0, SCALAR), (1, 1, 0, 0, SCALAR), (3, 0, 2, 1, SCALAR)])
def test_cross_bwd_final(W, D, pad, off, variant):
    """dL/dx0 = G + P + A: columns < D to the bottom gradient (its own stride), the rest to a contiguous dZ."""
    eng = N.engine()
    B = 33
    rng = np.random.default_rng(W + D + pad + off)
    (G, _), (P, _), (A, _) = (operand(rng, B, W, pad, off) for _ in range(3))
    lo, blo = operand(rng, B, D, 4, off, float("nan")) if D else (None, None)
    hi_buf = torch.full((off + B * (W - D) + 4,), float("nan"), device="cuda")
    hi = hi_buf[off:off + B * (W - D)].view(B, W - D) if W > D else None
    eng.debug_dispatch_log()
    eng.cross_bwd(FINAL, G, A, P=P, dx_lo=lo, dx_hi=hi)
    assert eng.debug_dispatch_log() == [N.Dispatch(L.ORX_OP_CROSS, variant, 1, FINAL, B, W, D, 1)]
    ref = (f64(G) + f64(P)) + f64(A)
    got = np.concatenate([f64(lo) if D else np.zeros((B, 0)), f64(hi) if W > D else np.zeros((B, 0))], 1)
    s = np.abs(f64(G) + f64(P)) + np.abs(f64(A))                         # two roundings
    assert np.all(np.abs(got - ref) <= s * 2.0 ** -22 + 1e-38)
    assert (W == D or untouched(hi_buf, [hi])) and (D == 0 or untouched(blo, [lo]))


def test_cross_empty_batch_and_refusals():
    """B = 0 launches nothing and records nothing; every refusal returns ORX_ERR_INVALID before any device work (the
    outputs keep their sentinel, no dispatch record)."""
    eng, lib = N.engine(), L.lib()
    st = eng.stream()
    B, W = 4, 8
    a = [torch.ones(B, W, device="cuda") for _ in range(3)]
    out = torch.full((B, W), 7.0, device="cuda")
    p = [C.c_void_p(t.data_ptr()) for t in a]
    po = C.c_void_p(out.data_ptr())
    eng.debug_dispatch_log()
    assert lib.orx_cross_fwd(eng.h, p[0], W, p[1], W, p[2], W, 0, W, po, W, st) == 0
    for mode in (TOP, MID, FINAL):
        assert lib.orx_cross_bwd(eng.h, mode, 0, W, p[0], W, p[1], W, p[2], W, p[2], W, p[1], W, po, W, 2, po, W,
                                 po, W, st) == 0
    torch.cuda.synchronize()
    assert eng.debug_dispatch_log() == [] and bool((out == 7.0).all())
    fwd = [  # h, x0, ld, xl, ld, y, ld, B, W, out, ld
        (None, p[0], W, p[1], W, p[2], W, B, W, po, W), (eng.h, None, W, p[1], W, p[2], W, B, W, po, W),
        (eng.h, p[0], W, p[1], W, p[2], W, B, W, None, W), (eng.h, p[0], W, p[1], W, p[2], W, -1, W, po, W),
        (eng.h, p[0], W, p[1], W, p[2], W, B, 0, po, W), (eng.h, p[0], W - 1, p[1], W, p[2], W, B, W, po, W),
        (eng.h, p[0], W, p[1], W, p[2], W, B, W, po, W - 1)]
    for args in fwd:
        assert lib.orx_cross_fwd(*args, st) == -1
    G, A, dy = p[0], p[1], p[2]
    good = dict(mode=TOP, B=B, W=W, G=G, lG=W, P=None, lP=0, x0=p[2], l0=W, y=p[2], ly=W, A=A, lA=W, dy=po, ldy=W,
                split=0, lo=None, llo=0, hi=None, lhi=0)
    bad = [dict(mode=3), dict(mode=-1), dict(G=None), dict(A=None), dict(x0=None), dict(y=None), dict(dy=None),
           dict(B=-1), dict(W=0), dict(lG=W - 1), dict(lA=W - 1), dict(ldy=W - 1), dict(mode=MID),      # MID: P null
           dict(mode=MID, P=p[2], lP=W - 1), dict(mode=FINAL, P=p[2], lP=W, split=W + 1, hi=po, lhi=W),
           dict(mode=FINAL, P=p[2], lP=W, split=2, lo=None, llo=2, hi=po, lhi=6),
           dict(mode=FINAL, P=p[2], lP=W, split=2, lo=po, llo=1, hi=po, lhi=6),
           dict(mode=FINAL, P=p[2], lP=W, split=2, lo=po, llo=2, hi=None, lhi=6),
           dict(mode=FINAL, P=p[2], lP=W, split=-1, hi=po, lhi=W)]
    for b in bad:
        k = {**good, **b}
        rc = lib.orx_cross_bwd(eng.h, k["mode"], k["B"], k["W"], k["G"], k["lG"], k["P"], k["lP"], k["x0"], k["l0"],
                               k["y"], k["ly"], k["A"], k["lA"], k["dy"], k["ldy"], k["split"], k["lo"], k["llo"],
                               k["hi"], k["lhi"], st)
        assert rc == -1, b
    assert lib.orx_cross_bwd(None, TOP, B, W, G, W, None, 0, p[2], W, p[2], W, A, W, po, W, 0, None, 0, None, 0, st) == -1
    torch.cuda.synchronize()
    assert eng.debug_dispatch_log() == []
    assert bool((out == 7.0).all()) and all(bool((t == 1.0).all()) for t in a)


# ---- DLRM(arch_interaction_op="cross") ------------------------------------------------------------------------------
VOCAB, SIZES, M_SPA, N_DENSE = [50, 301, 17], [3, 1, 7], 16, 13
LN_BOT, LN_TOP = [32, M_SPA], [64, 32, 1]


def _data(rng, B, bags):
    dense = np.log1p(rng.integers(0, 100, (B, N_DENSE))).astype(np.float32)
    label = (rng.random(B) < 0.3).astype(np.float32)
    if bags:
        sp = np.concatenate([np.where(rng.random((B, s)) < 0.2, -1, rng.integers(0, v, (B, s)))
                             for v, s in zip(VOCAB, SIZES)], 1)
        return dense, sp.astype(np.int64), label, NB.col_offsets(SIZES)
    return dense, np.stack([rng.integers(0, v, B) for v in VOCAB], 1).astype(np.int64), label, None


def _model(r, pooling=None, layers=2, **kw):
    """A small cross model whose initial weights come from a fixed seed, not from whatever tests ran before."""
    from openrec.tf2.recommenders import DLRM
    from openrec_b200.tfshim.keras import layers as KL
    KL.set_seed(20260923)
    bags = dict(bag_sizes=SIZES, pooling=pooling) if pooling else {}
    return DLRM(m_spa=M_SPA, ln_emb=VOCAB, ln_bot=LN_BOT, ln_top=LN_TOP, arch_interaction_op="cross",
                cross_layers=layers, cross_projection_dim=r, **bags, **kw)


OPTS = ["sgd", "momentum", "adagrad", "rowwise", "adam", "lazy"]


def _opt(tf, name):
    """-> (optimizer, kind of the restatement, momentum)."""
    from openrec_b200.tfshim.keras.optimizers import LazyAdam, RowwiseAdagrad
    return {"sgd": (tf.keras.optimizers.SGD(learning_rate=0.1), O.OPT_SGD, 0.0),
            # the velocity carries step 1's gradient into step 2 with weight 1 + m: lr 0.05 keeps the second step's
            # reach, and so the reach of the gradients' 3xTF32 error, about that of SGD's lr 0.1 under the same bar
            "momentum": (tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9), X.OPT_MOMENTUM, 0.9),
            "adagrad": (tf.keras.optimizers.Adagrad(learning_rate=0.05), O.OPT_ADAGRAD, 0.0),
            "rowwise": (RowwiseAdagrad(learning_rate=0.05), X.OPT_ROWWISE_ADAGRAD, 0.0),
            "adam": (tf.keras.optimizers.Adam(), O.OPT_ADAM_DENSE, 0.0),
            "lazy": (LazyAdam(), O.OPT_ADAM_LAZY, 0.0)}[name]


def _slots0(kind, var, T):
    """The restatement's initial slots, tables first (row-wise Adagrad: one accumulator per table row)."""
    out = []
    for j, v in enumerate(var):
        if kind in (O.OPT_ADAGRAD, X.OPT_ROWWISE_ADAGRAD):
            out.append((np.full(v.shape[0] if kind == X.OPT_ROWWISE_ADAGRAD and j < T else v.shape, 0.1), None))
        elif kind in (X.OPT_MOMENTUM,):
            out.append((np.zeros_like(v), None))
        elif kind == O.OPT_SGD:
            out.append((None, None))
        else:
            out.append((np.zeros_like(v), np.zeros_like(v)))
    return out


@pytest.mark.parametrize("optname", OPTS)
@pytest.mark.parametrize("r", [None, 8])
@pytest.mark.parametrize("inputs", ["one-hot", "sum", "mean"])
def test_dlrm_cross_training_step(tf, optname, r, inputs):
    """Two steps: the loss, every table (touched rows move, the rest stay), every Dense and cross variable and their
    slots against the float64 restatement, at the bars of the existing DLRM tests (loss 2e-6, variables / slots 2e-5)."""
    rng = np.random.default_rng(OPTS.index(optname) * 31 + (r or 0) + len(inputs))
    B, T = 256, len(VOCAB)
    pooling = None if inputs == "one-hot" else inputs
    model = _model(r, pooling)
    dense, sp, label, col_off = _data(rng, B, pooling is not None)
    model._graph(N_DENSE)
    tv = model.trainable_variables
    assert len(tv) == T + 2 * (len(LN_BOT) + len(LN_TOP)) + 2 * (2 if r is None else 3)
    var = [v.numpy().astype(np.float64) for v in tv]
    opt, kind, mom = _opt(tf, optname)
    st = _slots0(kind, var, T)
    for step in (1, 2):
        with tf.GradientTape() as tape:
            loss = model(dense, sp, label)
        opt.apply_gradients(zip(tape.gradient(loss, tv), tv))
        rl = X.train_step(kind, var[:T], var[T:], st, step, opt.learning_rate, dense.astype(np.float64), sp, label,
                          len(LN_BOT), len(LN_TOP), r, col_off, pooling == "mean", mom)
        close(float(loss), rl, atol=2e-6)
        for j, (v, ref) in enumerate(zip(tv, var)):
            close(v.numpy(), ref, atol=2e-5)
            s0, s1 = opt.slots(v)
            if st[j][0] is not None:
                close(s0, st[j][0], atol=2e-5)
            if st[j][1] is not None:
                close(s1, st[j][1], atol=2e-5)


def test_dlrm_cross_launches_and_dispatch(tf):
    """One step launches the cross kernels a low-rank network needs: per layer one forward and one backward pass on the
    VEC path (W = 64), one final pass; _launches_per_step counts them."""
    rng = np.random.default_rng(1)
    model = _model(8, layers=3)
    dense, sp, label, _ = _data(rng, 128, False)
    model._graph(N_DENSE)
    eng = N.engine()
    eng.debug_dispatch_log()
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, model.trainable_variables), model.trainable_variables))
    torch.cuda.synchronize()
    rec = [d for d in eng.debug_dispatch_log() if d.op == L.ORX_OP_CROSS]
    W = (len(VOCAB) + 1) * M_SPA
    assert rec == ([N.Dispatch(L.ORX_OP_CROSS, VEC, 0, 0, 128, W, 0, 1)] * 3
                   + [N.Dispatch(L.ORX_OP_CROSS, VEC, 1, m, 128, W, 0, 1) for m in (TOP, MID, MID)]
                   + [N.Dispatch(L.ORX_OP_CROSS, VEC, 1, FINAL, 128, W, M_SPA, 1)])
    full = _model(None)
    from openrec.tf2.recommenders import DLRM
    plain = DLRM(m_spa=M_SPA, ln_emb=VOCAB, ln_bot=LN_BOT, ln_top=LN_TOP)
    n = plain._launches_per_step() - 2                 # without the two interaction kernels
    assert model._launches_per_step() == n + 3 * (2 + (1 + 2 + 1) + (1 + 3 + 2)) + 1
    assert full._launches_per_step() == n + 2 * (2 + 1 + 3 + 2) + 1


@pytest.mark.parametrize("r", [None, 8])
@pytest.mark.parametrize("pooling", [None, "mean"])
def test_dlrm_cross_inference_and_gradients(tf, r, pooling):
    """inference = the restatement's forward; tape.gradient of every cross variable (and the Dense ones) = its
    backward.  The network's direct CrossNetwork call gives the same x_L as the fused graph."""
    rng = np.random.default_rng(5 + (r or 0))
    B, T = 200, len(VOCAB)
    model = _model(r, pooling)
    dense, sp, label, col_off = _data(rng, B, pooling is not None)
    model._graph(N_DENSE)
    tv = model.trainable_variables
    var = [v.numpy().astype(np.float64) for v in tv]
    bw, bb, tw, tb, layers = X.split_dense(var[T:], len(LN_BOT), len(LN_TOP), r)
    embs = X.embeddings(var[:T], sp, col_off, pooling == "mean")
    cache = X.forward(embs, bw, bb, tw, tb, layers, dense.astype(np.float64))
    close(model.inference(dense, sp).numpy(), cache["pred"], atol=2e-6)
    c = model._graph(N_DENSE).forward(torch.from_numpy(dense).cuda(), torch.from_numpy(sp).cuda().to(torch.int32))
    xL = model._cross(c["x0"]).numpy()
    assert np.array_equal(xL, c["xs"][-1].cpu().numpy())
    close(xL, cache["xs"][-1], atol=2e-5)
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    grads = tape.gradient(loss, tv)
    rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = X.backward(cache, bw, tw, layers, dense.astype(np.float64), dpred)
    close(float(loss), rl, atol=2e-6)
    want = [g for l in range(len(LN_BOT)) for g in (gr["bot_w"][l], gr["bot_b"][l])]
    want += [g for l in range(len(LN_TOP)) for g in (gr["top_w"][l], gr["top_b"][l])]
    want += [g for layer in gr["cross"] for pair in layer for g in pair if g is not None]
    for g, w in zip(grads[T:], want):
        assert g.indices is None
        close(g.values.numpy(), w, atol=2e-6)
    for k in range(T):
        if col_off is None:
            np.testing.assert_array_equal(grads[k].indices.numpy(), sp[:, k])
            close(grads[k].values.numpy(), gr["emb"][k], atol=2e-6)
        else:
            ids, vals = NB.bag_slices(sp, col_off, k, VOCAB[k], gr["emb"][k], True)
            np.testing.assert_array_equal(grads[k].indices.numpy(), ids)
            close(grads[k].values.numpy(), vals, atol=2e-6)


def test_dlrm_cross_checkpoint_round_trip(tf, tmp_path):
    """checkpoint.save / load carry the cross variables and their slots by name: the restored model continues bit for
    bit (one-hot ids and each row once per batch, so no staged-row sum whose atomic order could vary)."""
    from openrec_b200.tf2 import checkpoint
    rng = np.random.default_rng(8)
    B = 16
    dense = np.log1p(rng.integers(0, 100, (B, N_DENSE))).astype(np.float32)
    sp = np.stack([rng.permutation(v)[:B] for v in VOCAB], 1).astype(np.int64)     # each row once per table
    label = (rng.random(B) < 0.3).astype(np.float32)
    a, opt = _model(8), tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = a(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, a.trainable_variables), a.trainable_variables))
    checkpoint.save(str(tmp_path / "dcn.npz"), a, opt)
    names = [v.name for v in a.variables]
    assert names[-3:] == ["crossnetwork/cross_layer_1/v", "crossnetwork/cross_layer_1/u",
                          "crossnetwork/cross_layer_1/bias"]
    b, opt2 = _model(8), tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with pytest.raises(ValueError):
        checkpoint.save(str(tmp_path / "unbuilt.npz"), b)            # the cross network has no variables yet
    checkpoint.load(str(tmp_path / "dcn.npz"), b, opt2, build=lambda: b._graph(N_DENSE))
    for x, y in zip(a.variables, b.variables):
        assert torch.equal(x.t, y.t)
        for s, t in zip(opt.slots(x), opt2.slots(y)):
            assert (s is None and t is None) or torch.equal(s, t)
    for m, o in ((a, opt), (b, opt2)):
        with tf.GradientTape() as tape:
            loss = m(dense, sp, label)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
    for x, y in zip(a.variables, b.variables):
        assert torch.equal(x.t, y.t)
    assert torch.equal(a.inference(dense, sp).t, b.inference(dense, sp).t)
    full = _model(None)
    full._graph(N_DENSE)
    with pytest.raises(ValueError):                                   # full-rank names / shapes differ
        checkpoint.load(str(tmp_path / "dcn.npz"), full)


# The 'dot' model's variables, names and seed draws, recorded at the parent commit of the cross network: names, shapes
# and the (seed, bound) of every orx_fill_uniform draw under set_seed(1234).
DOT_EXPECT = [("latentfactor/embeddings", (50, 16), 1234, 0.05), ("latentfactor/embeddings", (301, 16), 1235, 0.05),
              ("latentfactor/embeddings", (17, 16), 1236, 0.05), ("dense/kernel", (13, 32), 1237, 0.365148372),
              ("dense/bias", (32,), None, 0.0), ("dense/kernel", (32, 16), 1238, 0.353553391),
              ("dense/bias", (16,), None, 0.0), ("dense/kernel", (22, 64), 1239, 0.264135272),
              ("dense/bias", (64,), None, 0.0), ("dense/kernel", (64, 32), 1240, 0.25),
              ("dense/bias", (32,), None, 0.0), ("dense/kernel", (32, 1), 1241, 0.426401433),
              ("dense/bias", (1,), None, 0.0)]


def test_dot_model_keeps_its_variables_and_draws():
    """A DLRM without 'cross' builds the same variables, names and initial bits as before the cross network existed."""
    from openrec.tf2.recommenders import DLRM
    from openrec_b200.tfshim.keras import layers as KL
    KL.set_seed(1234)
    m = DLRM(m_spa=16, ln_emb=[50, 301, 17], ln_bot=[32, 16], ln_top=[64, 32, 1], interaction_mode="dlrm")
    m._graph(13)
    assert [(v.name, tuple(v.shape)) for v in m.variables] == [(n, s) for n, s, _, _ in DOT_EXPECT]
    eng = N.engine()
    for v, (_, shape, seed, lim) in zip(m.variables, DOT_EXPECT):
        if seed is None:
            assert not bool(v.t.any())
            continue
        want = torch.empty(shape, device="cuda")
        eng.fill_uniform(want, -np.float32(lim), np.float32(lim), seed)
        assert torch.equal(v.t, want), v.name


# ---- ShardedDLRM ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,pooling,r,optname", [(1, None, 8, "adagrad"), (2, "sum", None, "sgd"),
                                                 (3, None, 4, "lazy"), (4, "mean", 8, "adam")])
def test_sharded_cross_equals_single_gpu(R, pooling, r, optname):
    """ShardedDLRM's cross network on R loopback ranks: three steps of the global batch against the single-GPU model,
    at the bars of the existing sharded DLRM tests; every rank's replicas stay identical."""
    import tensorflow as tf
    from openrec_b200.sharded import DLRMShard, LoopbackExchange, dlrm_step_sharded, dlrm_inference_sharded
    from openrec_b200.tf2.mlp_ops import ACT
    from openrec_b200.tf2.recommenders.dlrm import cross_projections
    tol = {"sgd": 1e-5, "adagrad": 1e-5, "adam": 1e-4, "lazy": 1e-5}[optname]
    lr = {"sgd": 0.1, "adagrad": 0.05, "adam": 0.01, "lazy": 0.01}[optname]
    ref = _model(r, pooling)
    ref._graph(N_DENSE)
    opt = {"sgd": tf.keras.optimizers.SGD, "adagrad": tf.keras.optimizers.Adagrad, "adam": tf.keras.optimizers.Adam,
           "lazy": tf.keras.optimizers.LazyAdam}[optname](learning_rate=lr)
    T = len(VOCAB)
    table = torch.cat([lf.embeddings.t for lf in ref._latent_factors])
    dense_vars = ref.trainable_variables[T:]
    acts = [l.activation for l in ref._mlp_bot.layers + ref._mlp_top.layers]
    nb = 2 * (len(LN_BOT) + len(LN_TOP))
    parts, engines = [], []
    for k in range(R):
        engines.append(N.Engine(0))
        rows = (table.shape[0] - k + R - 1) // R
        t = torch.zeros(max(rows, 1), M_SPA, device="cuda")
        t[:rows] = table[k::R]
        slots = [torch.full_like(t, 0.1 if optname == "adagrad" else 0.0) if s is not None else None
                 for s in opt.slots(ref._latent_factors[0].embeddings)]
        reps = [v.t.clone() for v in dense_vars]
        dslots = [tuple(x.clone() if x is not None else None for x in opt.slots(v)) for v in dense_vars]
        trip = [(reps[2 * l], reps[2 * l + 1], ACT[acts[l]]) for l in range(len(acts))]
        cross, i = [], nb
        for p in cross_projections(ref._cross):
            cross.append([])
            for w, b in p:
                cross[-1].append((reps[i], reps[i + 1] if b is not None else None))
                i += 2 if b is not None else 1
        parts.append(DLRMShard(engines[-1], k, R, VOCAB, M_SPA, trip[:len(LN_BOT)], trip[len(LN_BOT):], t, slots,
                               dslots, mode="reference", col_off=ref._col_off, pooling=ref._pooling, cross=cross))
    xchg = LoopbackExchange()
    rng = np.random.default_rng(R * 5 + (r or 0))
    B = 24
    try:
        for step in range(1, 4):
            dense, sp, label, _ = _data(rng, R * B, pooling is not None)
            dense, sp, label = (torch.from_numpy(x).cuda() for x in (dense, sp.astype(np.int32), label))
            batches = [tuple(x[k * B:(k + 1) * B].contiguous() for x in (dense, sp, label)) for k in range(R)]
            if step == 1:
                preds = dlrm_inference_sharded(parts, xchg, [b[:2] for b in batches])
                torch.testing.assert_close(torch.cat(preds), ref.inference(dense, sp).t, atol=1e-6, rtol=1e-5)
            with tf.GradientTape() as tape:
                lv = ref(dense, sp, label)
            opt.apply_gradients(zip(tape.gradient(lv, ref.trainable_variables), ref.trainable_variables))
            want_loss = float(lv.numpy())
            o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, step)
            for out in dlrm_step_sharded(parts, xchg, batches, o):
                assert abs(float(out[0]) - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (step, want_loss)
        glob = torch.zeros_like(table)
        for p in parts:
            glob[p.rank::R] = p.table[:p.rows]
        torch.testing.assert_close(glob, torch.cat([lf.embeddings.t for lf in ref._latent_factors]), atol=tol, rtol=tol)
        for p in parts:
            assert len(p.dense_vars()) == len(dense_vars)
            for k, (var, v) in enumerate(zip(p.dense_vars(), dense_vars)):
                assert torch.equal(var, parts[0].dense_vars()[k]), "replicas differ"
                torch.testing.assert_close(var, v.t, atol=tol, rtol=tol)
                for j, s in enumerate(opt.slots(v)):
                    if s is not None:
                        torch.testing.assert_close(p.dense_slots[k][j], s, atol=tol, rtol=tol)
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


_CLASS = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(0)
dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
import tensorflow as tf
from openrec.tf2.recommenders import DLRM, ShardedDLRM
vocab, D = [50, 301, 17], 16
kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[32, D], ln_top=[64, 32, 1], arch_interaction_op="cross", cross_layers=2,
          cross_projection_dim=8)
sh, one = ShardedDLRM(**kw), DLRM(**kw)
sh._build(13); one._graph(13)
assert [v.name for v in sh.trainable_variables[-6:]] == [v.name for v in one.trainable_variables[-6:]]
assert sh.trainable_variables[-1].name == "crossnetwork/cross_layer_1/bias"
for lf, k in zip(one._latent_factors, np.cumsum([0] + vocab[:-1])):
    lf.embeddings.t.copy_(sh.embedding_shard.t[k:k + lf.embeddings.t.shape[0]])
for a, b in zip(sh._dense_vars(), one.trainable_variables[len(vocab):]):
    b.t.copy_(a.t)
rng = np.random.default_rng(4)
opts = [tf.keras.optimizers.Adagrad(learning_rate=0.05) for _ in range(2)]
for step in range(2):
    dense = np.log1p(rng.integers(0, 100, (64, 13))).astype(np.float32)
    sp = np.stack([rng.integers(0, v, 64) for v in vocab], 1)
    label = (rng.random(64) < 0.3).astype(np.float32)
    losses = []
    for m, o in ((sh, opts[0]), (one, opts[1])):
        with tf.GradientTape() as tape:
            loss = m(dense, sp, label)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
        losses.append(float(loss))
    assert abs(losses[0] - losses[1]) <= 1e-6, losses
for a, b in zip(sh._dense_vars(), one.trainable_variables[len(vocab):]):
    torch.testing.assert_close(a.t, b.t, atol=1e-5, rtol=1e-5)
torch.testing.assert_close(sh.inference(dense, sp).t, one.inference(dense, sp).t, atol=1e-6, rtol=1e-5)
dist.destroy_process_group()
print("sharded cross class ok")
"""


def test_sharded_dlrm_cross_class_one_rank():
    """The ShardedDLRM class surface with the cross network on a one-rank NCCL group: the cross variables and their
    names, and two steps and inference equal to the single-GPU model from the same weights."""
    from _ranks import run_ranks
    [(rc, out)] = run_ranks(1, _CLASS.format(root=ROOT), "gpu_dcn sharded class", timeout=600)
    assert rc == 0 and "sharded cross class ok" in out, out


# ---- full shape ----------------------------------------------------------------------------------------------------
MLPERF_BAGS = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]
# x_L against float64, normalised per output by the same computation in absolute values (|x0| |y_l| + |x_l|, |y_l| =
# |U|^T |V|^T |x_l| + |b|): each of the 3 x 2 projections is a k_gemm_tma output within 2^-18 of its own scale
# (test_gpu_dlrm.py) and each element-wise pass rounds once, so x_L is held to 8 x 2^-18.
E_XL = 8 * 2.0 ** -18


def test_dlrm_cross_full_shape_step(tf):
    """bench.py's DLRM shape (26 x 1M x 128, B = 32768, bottom 512-256-128, top 1024-1024-512-256-1, Adagrad), the MLPerf
    bag sizes and 3 cross layers of rank 512 (W = 3456): x_L of 2048 sampled rows at the normalised bar above, then one
    step against a float64 restatement (run on the device in float64) -- the loss, sampled rows and columns of every
    Dense and cross variable, and the touched rows of four tables, at the bars of the existing full-shape tests."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(35)
    B, m_spa, T = 32768, 128, 26
    ln_emb, ln_bot, ln_top = [1_000_000] * T, [512, 256, 128], [1024, 1024, 512, 256, 1]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=ln_bot, ln_top=ln_top, arch_interaction_op="cross",
                 cross_layers=3, cross_projection_dim=512, bag_sizes=MLPERF_BAGS, pooling="sum")
    col_off = NB.col_offsets(MLPERF_BAGS)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sp = rng.integers(0, 1_000_000, (B, int(col_off[-1]))).astype(np.int64)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    W = (T + 1) * m_spa
    d64 = lambda t: t.detach().to(torch.float64)
    dense_t, sp_t = torch.from_numpy(dense).cuda(), torch.from_numpy(sp).cuda()

    # x_L on sampled rows, each stage restated from the kernel's own float32 input
    c = model._graph(13).forward(dense_t, sp_t.to(torch.int32))
    rows = torch.from_numpy(np.sort(rng.choice(B, 2048, replace=False))).cuda()
    x0 = d64(c["x0"][rows])
    x, s = x0, x0.abs()
    for l, p in enumerate(model._cross.projections()):
        h, hs = d64(c["xs"][l][rows]), d64(c["xs"][l][rows]).abs()
        for w, b in p:
            h, hs = h @ d64(w.t), hs @ d64(w.t).abs()
            if b is not None:
                h, hs = h + d64(b.t), hs + d64(b.t).abs()
        x, s = x0 * h + d64(c["xs"][l][rows]), x0.abs() * hs + d64(c["xs"][l][rows]).abs()
        e = float(((d64(c["xs"][l + 1][rows]) - x).abs() / s.clamp_min(1e-30)).max())
        print(f"cross layer {l}: normalised error {e:.3e} (bar {E_XL:.3e})")
        assert e <= E_XL
    del c

    # compact float64 problem: the touched rows of every table, on the device
    ids, csp, tabs = [], np.zeros_like(sp), []
    for k in range(T):
        cols = sp[:, col_off[k]:col_off[k + 1]]
        u = np.unique(cols)
        ids.append(u)
        csp[:, col_off[k]:col_off[k + 1]] = np.searchsorted(u, cols)
        tabs.append(d64(tv[k].t[torch.from_numpy(u).cuda()]))
    dvars = [d64(v.t) for v in tv[T:]]
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = model(dense, sp, label)
    opt.apply_gradients(zip(tape.gradient(loss, tv), tv))

    csp_t = torch.from_numpy(csp).cuda()
    embs = [tabs[k][csp_t[:, col_off[k]:col_off[k + 1]]].sum(1) for k in range(T)]
    bw, bb, tw, tb, layers = X.split_dense(dvars, len(ln_bot), len(ln_top), 512)
    rl, dx0, grads = X.loss_and_grads_t(embs, bw, bb, tw, tb, layers, d64(dense_t),
                                        torch.from_numpy(label).cuda().to(torch.float64))
    close(float(loss), rl, atol=2e-6)
    for j, (v, ref, g) in enumerate(zip(tv[T:], dvars, grads)):
        new = ref - 0.05 * g / (torch.sqrt(0.1 + g * g) + 1e-7)
        r_idx = torch.from_numpy(rng.choice(v.t.shape[0], min(v.t.shape[0], 256), replace=False)).cuda()
        if v.t.dim() == 2:
            c_idx = torch.from_numpy(rng.choice(v.t.shape[1], min(v.t.shape[1], 256), replace=False)).cuda()
            close(v.t[r_idx][:, c_idx], new[r_idx][:, c_idx].cpu().numpy(), atol=2e-5)
        else:
            close(v.t[r_idx], new[r_idx].cpu().numpy(), atol=2e-5)
    for k in (0, 9, 20, T - 1):
        gk = torch.zeros_like(tabs[k])
        cols = csp_t[:, col_off[k]:col_off[k + 1]]
        gk.index_add_(0, cols.reshape(-1), dx0[:, m_spa * (k + 1):m_spa * (k + 2)].repeat_interleave(cols.shape[1], 0))
        touched = torch.zeros(tabs[k].shape[0], dtype=torch.bool, device="cuda")
        touched[cols.reshape(-1)] = True
        acc = 0.1 + gk * gk
        new = tabs[k] - 0.05 * gk / (torch.sqrt(acc) + 1e-7)
        got = tv[k].t[torch.from_numpy(ids[k]).cuda()]
        close(got[touched], new[touched].cpu().numpy(), atol=2e-5)
