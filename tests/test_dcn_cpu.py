"""CPU: the float64 restatement of the DCN-v2 cross network and of the DLRM-DCN step (tests/dcn_np.py) against central
finite differences, and the model surface of DLRM(arch_interaction_op="cross") that needs no device: variable names and
shapes, the widths, constructor refusals, and 'cat' / unknown ops failing as before."""
import os
import subprocess
import sys

import numpy as np
import pytest

import dcn_np as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _layers(rng, W, L, r):
    out = []
    for _ in range(L):
        b = rng.standard_normal(W) * 0.3
        if r is None:
            out.append([(rng.standard_normal((W, W)) * 0.4, b)])
        else:
            out.append([(rng.standard_normal((W, r)) * 0.4, None), (rng.standard_normal((r, W)) * 0.4, b)])
    return out


def _fd(f, a, h=1e-6):
    """Central differences of the scalar f() w.r.t. every element of a (perturbed in place)."""
    g = np.zeros_like(a)
    for i in np.ndindex(a.shape):
        old = a[i]
        a[i] = old + h
        up = f()
        a[i] = old - h
        dn = f()
        a[i] = old
        g[i] = (up - dn) / (2 * h)
    return g


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("r", [None, 2])
def test_cross_gradients_match_finite_differences(L, r):
    rng = np.random.default_rng(L * 10 + (r or 0))
    B, W = 3, 5
    x0 = rng.standard_normal((B, W))
    layers = _layers(rng, W, L, r)
    R = rng.standard_normal((B, W))
    loss = lambda: float((R * X.cross_forward(x0, layers)[0][-1]).sum())
    xs, acts = X.cross_forward(x0, layers)
    dx0, grads = X.cross_backward(x0, layers, xs, acts, R.copy())
    np.testing.assert_allclose(dx0, _fd(loss, x0), rtol=1e-6, atol=1e-7)
    for projs, g in zip(layers, grads):
        for (w, b), (dw, db) in zip(projs, g):
            np.testing.assert_allclose(dw, _fd(loss, w), rtol=1e-6, atol=1e-7)
            assert (b is None) == (db is None)
            if b is not None:
                np.testing.assert_allclose(db, _fd(loss, b), rtol=1e-6, atol=1e-7)


def test_cross_forward_by_hand():
    """One full-rank layer on one sample: x1 = x0 * (K^T x0 + b) + x0."""
    x0 = np.array([[1.0, 2.0]])
    K, b = np.array([[1.0, 0.5], [-1.0, 2.0]]), np.array([0.25, -1.0])
    xs, acts = X.cross_forward(x0, [[(K, b)]])
    y = np.array([1.0 - 2.0 + 0.25, 0.5 + 4.0 - 1.0])
    np.testing.assert_array_equal(acts[0][-1][0], y)
    np.testing.assert_array_equal(xs[1][0], x0[0] * y + x0[0])


@pytest.mark.parametrize("r,L,multi", [(None, 1, False), (3, 2, False), (2, 3, True)])
def test_dlrm_dcn_gradients_match_finite_differences(r, L, multi):
    """The whole DLRM-DCN loss (bottom MLP, x0 layout, cross, top MLP, MSE) w.r.t. every Dense / cross variable and the
    embedding rows of the batch."""
    rng = np.random.default_rng(7 + L)
    B, D, T, n_dense = 4, 2, 2, 3
    W = (T + 1) * D
    vocab = [5, 4]
    tabs = [rng.standard_normal((V, D)) * 0.5 for V in vocab]
    dense = rng.standard_normal((B, n_dense))
    label = rng.random(B)
    if multi:
        col_off = np.array([0, 2, 5])
        sparse = np.stack([rng.integers(-1, 5, B), rng.integers(0, 5, B), rng.integers(0, 4, B), rng.integers(0, 4, B),
                           rng.integers(-1, 4, B)], 1)
    else:
        col_off, sparse = None, np.stack([rng.integers(0, V, B) for V in vocab], 1)
    shapes = [(n_dense, 4), (4,), (4, D), (D,), (W, 3), (3,), (3, 1), (1,)] + X.cross_shapes(W, L, r)
    dvars = [rng.standard_normal(s) * 0.4 for s in shapes]

    def loss():
        bw, bb, tw, tb, layers = X.split_dense(dvars, 2, 2, r)
        c = X.forward(X.embeddings(tabs, sparse, col_off, True), bw, bb, tw, tb, layers, dense)
        return float(((c["pred"] - label) ** 2).mean())

    bw, bb, tw, tb, layers = X.split_dense(dvars, 2, 2, r)
    c = X.forward(X.embeddings(tabs, sparse, col_off, True), bw, bb, tw, tb, layers, dense)
    _, dpred = X.O.dlrm_loss(c["pred"], label, "mse")
    gr = X.backward(c, bw, tw, layers, dense, dpred)
    got = [g for l in range(2) for g in (gr["bot_w"][l], gr["bot_b"][l])]
    got += [g for l in range(2) for g in (gr["top_w"][l], gr["top_b"][l])]
    got += [g for layer in gr["cross"] for pair in layer for g in pair if g is not None]
    for v, g in zip(dvars, got):
        np.testing.assert_allclose(g, _fd(loss, v), rtol=1e-5, atol=1e-8)
    for k, tab in enumerate(tabs):
        if multi:
            ids, rows = X.NB.bag_grad_rows(sparse, col_off, k, vocab[k], gr["emb"][k], True)
        else:
            ids, rows = X.O.dedup(sparse[:, k].astype(np.int64), gr["emb"][k])
        want = _fd(loss, tab)
        np.testing.assert_allclose(rows, want[ids], rtol=1e-5, atol=1e-8)
        untouched = np.setdiff1d(np.arange(vocab[k]), ids)
        np.testing.assert_allclose(want[untouched], 0.0, atol=1e-8)


def test_train_step_sgd_is_a_gradient_step():
    """train_step under SGD moves every variable by -lr * its gradient (from the pre-step values)."""
    rng = np.random.default_rng(3)
    B, D, T, W, r = 6, 4, 2, 12, 2
    tabs = [rng.standard_normal((7, D)) for _ in range(T)]
    sparse = np.stack([rng.integers(0, 7, B) for _ in range(T)], 1)
    dense, label = rng.standard_normal((B, 3)), rng.random(B)
    dvars = [rng.standard_normal(s) * 0.3 for s in [(3, D), (D,), (W, 1), (1,)] + X.cross_shapes(W, 1, r)]
    before = [v.copy() for v in dvars]
    bw, bb, tw, tb, layers = X.split_dense(before, 1, 1, r)
    c = X.forward(X.embeddings(tabs, sparse, None, False), bw, bb, tw, tb, layers, dense)
    _, dpred = X.O.dlrm_loss(c["pred"], label, "mse")
    gr = X.backward(c, bw, tw, layers, dense, dpred)
    st = [(None, None)] * (T + len(dvars))
    X.train_step(X.O.OPT_SGD, [t.copy() for t in tabs], dvars, st, 1, 0.1, dense, sparse, label, 1, 1, r)
    grads = [gr["bot_w"][0], gr["bot_b"][0], gr["top_w"][0], gr["top_b"][0], gr["cross"][0][0][0],
             gr["cross"][0][1][0], gr["cross"][0][1][1]]
    for v, b, g in zip(dvars, before, grads):
        np.testing.assert_allclose(v, b - 0.1 * g, rtol=1e-12, atol=1e-14)


SCRIPT = r"""
import sys
sys.path[:0] = [{compat!r}, {root!r}, {tests!r}]
import torch
import fake_engine
fake_engine.install()
import openrec_b200.tfshim.keras.layers as KL
from openrec.tf2.modules import CrossNetwork
from openrec.tf2.recommenders import DLRM

draws = []
real = KL.next_seed
import openrec_b200.tf2.modules.cross_network as CN
def counted():
    s = real()
    draws.append(s)
    return s
CN.next_seed = counted

kw = dict(m_spa=4, ln_emb=[10, 20, 30], ln_bot=[8, 4], ln_top=[6, 1])
W = 4 * 4
for r, names, shapes in (
        (None, ["kernel", "bias"], [(W, W), (W,)]),
        (3, ["v", "u", "bias"], [(W, 3), (3, W), (W,)])):
    m = DLRM(arch_interaction_op="cross", cross_layers=2, cross_projection_dim=r, **kw)
    m._graph(13)
    tv = m.trainable_variables
    cross = tv[3 + 4 + 4:]                                           # tables, bottom, top, cross
    want = [f"crossnetwork/cross_layer_{{l}}/{{n}}" for l in range(2) for n in names]
    assert [v.name for v in cross] == want, [v.name for v in cross]
    assert [tuple(v.shape) for v in cross] == shapes * 2
    assert tuple(m._mlp_top.layers[0].kernel.shape) == (W, 6)          # the top MLP reads x_L
    assert all(float(v.t.abs().sum()) == 0.0 for v in cross if v.name.endswith("bias"))
    lim = (6.0 / (cross[0].shape[0] + cross[0].shape[1])) ** 0.5    # glorot-uniform
    assert 0 < float(cross[0].t.abs().max()) <= lim
    assert m._cross.built and m._cross.width == W

assert len(draws) == 2 * 1 + 2 * 2, draws          # one kernel per full-rank layer, two per low-rank layer

c = CrossNetwork(1)
c.build(8)
c.build(8)
try:
    c.build(9)
    raise SystemExit("width change accepted")
except ValueError:
    pass
for bad in (dict(num_layers=0), dict(num_layers=2.5), dict(num_layers=1, projection_dim=0)):
    try:
        CrossNetwork(**bad)
        raise SystemExit(f"{{bad}} accepted")
    except ValueError:
        pass
for op in ("cat", "concat", "bogus"):
    try:
        DLRM(arch_interaction_op=op, **kw)
        raise SystemExit(f"{{op}} accepted")
    except AttributeError as e:
        assert "_arch_interaction_op" in str(e), e
d = DLRM(**kw)
d._graph(13)
assert d._cross is None and len(d.trainable_variables) == 3 + 4 + 4
print("dcn surface ok")
"""


def test_dlrm_cross_surface():
    """Names, shapes and widths of the cross variables (built with the oracle-backed engine), CrossNetwork's build and
    constructor rules, and 'cat' / unknown ops still ending in the reference's AttributeError (SURVEY Q2)."""
    code = SCRIPT.format(compat=os.path.join(ROOT, "compat"), root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "dcn surface ok" in r.stdout, r.stdout + r.stderr


def test_torch_restatement_matches_numpy():
    """loss_and_grads_t (torch float64, the full-shape checks) = forward / backward of the numpy restatement."""
    import torch
    rng = np.random.default_rng(11)
    B, D, T, r = 5, 4, 2, 3
    W = (T + 1) * D
    embs = [rng.standard_normal((B, D)) for _ in range(T)]
    dense, label = rng.standard_normal((B, 3)), rng.random(B)
    dvars = [rng.standard_normal(s) * 0.4 for s in [(3, 6), (6,), (6, D), (D,), (W, 5), (5,), (5, 1), (1,)]
             + X.cross_shapes(W, 2, r)]
    bw, bb, tw, tb, layers = X.split_dense(dvars, 2, 2, r)
    c = X.forward(embs, bw, bb, tw, tb, layers, dense)
    loss, dpred = X.O.dlrm_loss(c["pred"], label, "mse")
    gr = X.backward(c, bw, tw, layers, dense, dpred)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    tl, dx0, grads = X.loss_and_grads_t([t(e) for e in embs], *X.split_dense([t(v) for v in dvars], 2, 2, r),
                                        t(dense), t(label))
    assert abs(tl - loss) < 1e-12
    want = [g for l in range(2) for g in (gr["bot_w"][l], gr["bot_b"][l])]
    want += [g for l in range(2) for g in (gr["top_w"][l], gr["top_b"][l])]
    want += [g for layer in gr["cross"] for pair in layer for g in pair if g is not None]
    assert len(grads) == len(want) == len(dvars)
    for g, w in zip(grads, want):
        np.testing.assert_allclose(g.numpy(), w, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(dx0[:, D:].numpy(), np.concatenate(gr["emb"], 1), rtol=1e-12, atol=1e-14)
