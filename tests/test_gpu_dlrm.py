"""GPU: DLRM kernels and model vs the oracle / the golden vectors recorded from the reference's dlrm.py."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import openrec_oracle as O

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


@pytest.mark.parametrize("B,inn,out,act", [(37, 13, 8, 1), (300, 479, 96, 2), (1000, 64, 1, 0), (129, 5, 130, 1),
                                            (512, 256, 128, 1), (1111, 479, 1024, 1), (4096, 512, 256, 0),
                                            (200, 13, 512, 1), (777, 1024, 64, 2),
                                            (8192, 13, 512, 1), (8192, 256, 1, 2), (6000, 300, 200, 1)])   # split-K / split col-sum
def test_mlp_layer_fwd_bwd(B, inn, out, act):
    from openrec_b200 import native as N
    eng = N.engine()
    rng = np.random.default_rng(B)
    x, w, b = rng.standard_normal((B, inn)), rng.standard_normal((inn, out)) * 0.3, rng.standard_normal(out) * 0.1
    dy = rng.standard_normal((B, out))
    tx, tw, tb, tdy = dev(x), dev(w), dev(b), dev(dy)
    x, w, b, dy = (t.cpu().numpy().astype(np.float64) for t in (tx, tw, tb, tdy))
    name = {0: None, 1: "relu", 2: "sigmoid"}[act]
    y_ref = O.mlp_forward(x, [w], [b], "relu", name)[0]
    ty = torch.empty(B, out, device="cuda")
    eng.mlp_fwd(tx, tw, tb, act, ty)
    close(ty, y_ref, atol=2e-5)
    dx_ref, dw_ref, db_ref = O.mlp_backward(x, [w], [y_ref], dy, "relu", name)
    tdx, tdw, tdb = torch.empty(B, inn, device="cuda"), torch.empty_like(tw), torch.empty_like(tb)
    # backward from the oracle's y: a relu mask taken from the kernel's own y flips on |y| ~ 1e-7 ties (seen at B = 8192)
    eng.mlp_bwd(tx, dev(y_ref), tw, act, tdy, tdx, tdw, tdb)
    close(tdx, dx_ref, atol=5e-5), close(tdw, dw_ref[0], atol=2e-4, rtol=1e-4), close(tdb, db_ref[0], atol=1e-4)


@pytest.mark.parametrize("self_int", [False, True])
@pytest.mark.parametrize("mode", ["reference", "dlrm"])
def test_interaction_fwd_bwd(golden_dir, self_int, mode):
    from openrec_b200 import native as N
    from openrec_b200.tf2.mlp_ops import interaction_width
    eng = N.engine()
    rng = np.random.default_rng(3)
    B, F, D = 50, 27, 16
    feats = [rng.standard_normal((B, D)).astype(np.float32).astype(np.float64) for _ in range(F)]
    ref = O.second_order_interaction(feats, self_int, mode)
    P = interaction_width(F, self_int)
    emb = dev(np.stack(feats[:-1], 1))
    dense = dev(feats[-1])
    out = torch.empty(B, P, device="cuda")
    eng.interact_fwd(emb, dense, self_int, 0 if mode == "reference" else 1, out)
    close(out, ref, atol=2e-5)
    dout = rng.standard_normal((B, P)).astype(np.float32).astype(np.float64)
    dZ = O.second_order_interaction_bwd(feats, dout, self_int, mode)
    demb, ddense = torch.empty_like(emb), torch.full_like(dense, 0.5)     # ddense is accumulated into
    eng.interact_bwd(emb, dense, dev(dout), self_int, 0 if mode == "reference" else 1, demb, ddense)
    close(demb, dZ[:, :F - 1, :], atol=5e-5), close(ddense, dZ[:, F - 1, :] + 0.5, atol=5e-5)
    if mode == "reference":   # the golden recorded from the reference's own layer (F=5, D=7)
        g = dict(np.load(os.path.join(golden_dir, "interaction.npz")))
        f = [g[f"in{k}"] for k in range(5)]
        o = torch.empty(6, interaction_width(5, self_int), device="cuda")
        eng.interact_fwd(dev(np.stack(f[:-1], 1)), dev(f[-1]), self_int, 0, o)
        close(o, g[f"out_self{int(self_int)}"], atol=2e-5)


def _load_golden_into(model, g):
    """Copy the golden's variables (creation order) into the model."""
    dense = g["dense"]
    model._graph(dense.shape[1])
    tv = model.trainable_variables
    assert len(tv) == int(g["n_vars"])
    for k, v in enumerate(tv):
        assert tuple(v.shape) == g[f"var{k}"].shape, (k, v.shape, g[f"var{k}"].shape)
        v.assign(g[f"var{k}"].astype(np.float32))
    return tv


@pytest.mark.parametrize("tag,kw", [("mse", {}), ("bce_self", dict(loss_func="bce", arch_interaction_itself=True)),
                                    ("clip", dict(loss_threshold=0.45)), ("bce", dict(loss_func="bce"))])
def test_dlrm_model_matches_reference_golden(tf, golden_dir, tag, kw):
    from openrec.tf2.recommenders import DLRM
    g = dict(np.load(os.path.join(golden_dir, f"dlrm_{tag}.npz")))
    model = DLRM(m_spa=4, ln_emb=[11, 7, 13], ln_bot=[8, 4], ln_top=[16, 8, 1], **kw)
    tv = _load_golden_into(model, g)
    close(model.inference(g["dense"].astype(np.float32), g["sparse"]).numpy(), g["pred"], atol=2e-6)
    with tf.GradientTape() as tape:
        loss = model(g["dense"].astype(np.float32), g["sparse"], g["label"])
    # 'bce_self': the self-interaction saturates the top sigmoid, and log(1 - p + 1e-7) at p -> 1 is only good to
    # ~1e-3 in float32 (the reference computes in float32 too; the golden is float64)
    saturated = tag == "bce_self"
    close(float(loss), g["loss"], atol=2e-6, rtol=2e-3 if saturated else 1e-5)
    grads = tape.gradient(loss, tv)
    for k, (gr, v) in enumerate(zip(grads, tv)):
        ref = g[f"grad{k}"]
        if gr.indices is not None:
            got = torch.zeros(v.shape, device="cuda").index_add_(0, gr.indices.t.long(), gr.values.t).cpu().numpy()
        else:
            got = gr.values.numpy()
        if saturated:   # 1 - p is not representable near p = 1 in float32 (the reference computes in float32 too):
            continue    # the gradient is ill-conditioned there; dlrm_bce.npz is the BCE parity case
        close(got, ref, atol=2e-6)


@pytest.mark.parametrize("optname,mode", [("adam", "reference"), ("sgd", "dlrm"), ("adagrad", "dlrm")])
def test_dlrm_training_step(tf, optname, mode):
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(21)
    B, m_spa, ln_emb = 256, 16, [50, 31, 77, 20]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=[32, m_spa], ln_top=[64, 32, 1], interaction_mode=mode)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sparse = np.stack([rng.integers(0, n, B) for n in ln_emb], 1).astype(np.int64)     # un-cast ids (dataloader.py:75)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    var = [v.numpy().astype(np.float64) for v in tv]
    T = len(ln_emb)
    tabs, rest = var[:T], var[T:]
    bot_w, bot_b, top_w, top_b = [rest[0], rest[2]], [rest[1], rest[3]], rest[4::2], rest[5::2]
    opt = {"adam": tf.keras.optimizers.Adam(), "sgd": tf.keras.optimizers.SGD(learning_rate=0.1),
           "adagrad": tf.keras.optimizers.Adagrad(learning_rate=0.05)}[optname]
    kind = {"adam": O.OPT_ADAM_DENSE, "sgd": O.OPT_SGD, "adagrad": O.OPT_ADAGRAD}[optname]
    if kind == O.OPT_ADAGRAD:
        st = [(np.full_like(v, 0.1), None) for v in var]
    else:
        st = [(np.zeros_like(v), np.zeros_like(v)) for v in var]
    for step in (1, 2):
        with tf.GradientTape() as tape:
            loss = model(dense, sparse, label)
        grads = tape.gradient(loss, tv)
        opt.apply_gradients(zip(grads, tv))
        cache = O.dlrm_forward(tabs, bot_w, bot_b, list(top_w), list(top_b), dense.astype(np.float64), sparse,
                               interaction_mode=mode)
        rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
        gr = O.dlrm_backward(cache, tabs, bot_w, list(top_w), dense.astype(np.float64), sparse, dpred,
                             interaction_mode=mode)
        close(float(loss), rl, atol=2e-6)
        dense_grads = [gr["bot_w"][0], gr["bot_b"][0], gr["bot_w"][1], gr["bot_b"][1]]
        for l in range(len(top_w)):
            dense_grads += [gr["top_w"][l], gr["top_b"][l]]
        for k in range(T):
            O.apply_sparse(kind, var[k], st[k][0], st[k][1], sparse[:, k], gr["emb"][k], step, opt.learning_rate)
        for j, gd in enumerate(dense_grads):
            O.apply_dense(kind, var[T + j], st[T + j][0], st[T + j][1], gd, step, opt.learning_rate)
        for v, ref in zip(tv, var):
            close(v.numpy(), ref, atol=2e-5)
    if mode == "dlrm":
        assert np.abs(gr["emb"][0]).max() > 0      # the fixed interaction does train the tables


def test_dlrm_full_shape_training_step(tf):
    """BASELINE.json configs[3]: the Criteo shape (26 tables x 1M x 128, B = 32768, MLPs 13-512-256-128 and
    479-1024-1024-512-256-1, Adagrad): one training step through the class surface (TMA-fed wgmma Dense layers, warp
    interaction kernels, strided gathers / sparse applies) against the float64 oracle on the touched rows."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(33)
    B, m_spa, T = 32768, 128, 26
    ln_emb, ln_bot, ln_top = [1_000_000] * T, [512, 256, 128], [1024, 1024, 512, 256, 1]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=ln_bot, ln_top=ln_top, interaction_mode="dlrm")
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sparse = np.stack([rng.integers(0, n, B) for n in ln_emb], 1).astype(np.int64)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    assert len(tv) == T + 2 * (len(ln_bot) + len(ln_top))
    rows, csparse, tabs = [], np.zeros_like(sparse), []
    for k in range(T):                              # compact oracle problem: the touched rows of every table
        r = np.unique(sparse[:, k])
        rows.append(r)
        csparse[:, k] = np.searchsorted(r, sparse[:, k])
        tabs.append(tv[k].t[torch.from_numpy(r).cuda()].cpu().numpy().astype(np.float64))
    untouched = [int(np.setdiff1d(np.arange(2000), rows[k])[0]) for k in (0, T - 1)]
    before = [tv[k].t[u].clone() for k, u in zip((0, T - 1), untouched)]
    rest = [v.numpy().astype(np.float64) for v in tv[T:]]
    nb = len(ln_bot)
    bot_w, bot_b, top_w, top_b = rest[0:2 * nb:2], rest[1:2 * nb:2], rest[2 * nb::2], rest[2 * nb + 1::2]
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = model(dense, sparse, label)
    opt.apply_gradients(zip(tape.gradient(loss, tv), tv))
    cache = O.dlrm_forward(tabs, bot_w, bot_b, list(top_w), list(top_b), dense.astype(np.float64), csparse,
                           interaction_mode="dlrm")
    rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = O.dlrm_backward(cache, tabs, bot_w, list(top_w), dense.astype(np.float64), csparse, dpred, interaction_mode="dlrm")
    close(float(loss), rl, atol=2e-6)
    dense_grads = []
    for l in range(nb):
        dense_grads += [gr["bot_w"][l], gr["bot_b"][l]]
    for l in range(len(top_w)):
        dense_grads += [gr["top_w"][l], gr["top_b"][l]]
    for j, gd in enumerate(dense_grads):
        ref = rest[j]
        O.apply_dense(O.OPT_ADAGRAD, ref, np.full_like(ref, 0.1), None, gd, 1, 0.05)
        close(tv[T + j].numpy(), ref, atol=2e-5)
    assert np.abs(gr["emb"][0]).max() > 0
    for k in (0, 7, T - 1):
        O.apply_sparse(O.OPT_ADAGRAD, tabs[k], np.full_like(tabs[k], 0.1), None, csparse[:, k], gr["emb"][k], 1, 0.05)
        close(tv[k].t[torch.from_numpy(rows[k]).cuda()], tabs[k], atol=2e-5)
    for k, u, b in zip((0, T - 1), untouched, before):
        assert torch.equal(tv[k].t[u], b)          # rows outside the batch are bit-identical
