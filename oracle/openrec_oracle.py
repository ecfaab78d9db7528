"""NumPy restatement of the openrec.tf2 hot path -- TEST INFRASTRUCTURE, NOT PRODUCT.

Every function cites the reference file:line it follows (paths relative to
the reference checkout).  TensorFlow-internal semantics that cannot be read here
(gradient of ``maximum``, IndexedSlices aggregation, optimizer formulas, Keras
loss epsilons) are marked [TF-mem] -- see oracle/__init__.py "PARITY UNPINNED".

All functions take ``dtype`` implicitly from their inputs: feed float32 arrays for
the reference's arithmetic type, float64 arrays to separate kernel error from
fp32 reduction-order noise.
"""
from __future__ import annotations

import numpy as np

# --------------------------------------------------------------------------------------
# elementwise helpers (numerically stable forms TF uses [TF-mem])
# --------------------------------------------------------------------------------------


def log_sigmoid(y):
    """tf.math.log_sigmoid = -softplus(-y); stable: min(y,0) - log1p(exp(-|y|))."""
    return np.minimum(y, 0) - np.log1p(np.exp(-np.abs(y)))


def sigmoid(y):
    """tf.math.sigmoid, stable for both signs."""
    e = np.exp(-np.abs(y))
    return np.where(y >= 0, 1 / (1 + e), e / (1 + e)).astype(y.dtype)


def l2_loss(x):
    """tf.nn.l2_loss(x) = sum(x**2)/2  (openrec/tf2/recommenders/bpr.py:35)."""
    return (x * x).sum(dtype=x.dtype) * x.dtype.type(0.5)


# --------------------------------------------------------------------------------------
# LatentFactor  (openrec/tf2/modules/latent_factor.py:4-23)
# --------------------------------------------------------------------------------------


def lookup(table, ids):
    """LatentFactor.__call__ = keras Embedding.call: out[b,:] = table[ids[b],:]
    (latent_factor.py:4-15).  ids bit-exact integer gather."""
    return table[np.asarray(ids, dtype=np.int64)]


def unique_first_occurrence(ids):
    """tf.unique: unique values in order of first occurrence + inverse index."""
    ids = np.asarray(ids)
    _, first, inv = np.unique(ids, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    return ids[np.sort(first)], rank[inv]


def censor(table, ids, min_norm=0.1):
    """LatentFactor.censor (latent_factor.py:17-23): for the *unique* ids,
    row <- row / max(||row||_2, 0.1).  In place; rows not in ids untouched."""
    uid, _ = unique_first_occurrence(ids)
    rows = table[uid]
    norm = np.sqrt((rows * rows).sum(axis=1, keepdims=True, dtype=table.dtype))
    table[uid] = rows / np.maximum(norm, table.dtype.type(min_norm))
    return table


# --------------------------------------------------------------------------------------
# forward passes
# --------------------------------------------------------------------------------------


def pairwise_log_loss(u, p, n, bp=None, bn=None):
    """PairwiseLogLoss.call (openrec/tf2/modules/pairwise_log_loss.py:15-34).
    Returns (loss scalar, x [B,1])."""
    dt = u.dtype
    x = (u * p).sum(axis=1, keepdims=True, dtype=dt)
    xn = (u * n).sum(axis=1, keepdims=True, dtype=dt)
    if bp is not None:
        x = x + bp
    if bn is not None:
        xn = xn + bn
    x = x - xn
    y = np.maximum(x, dt.type(-30.0))
    loss = -log_sigmoid(y).mean(dtype=dt)
    return loss, x


def bpr_forward(user_tab, item_tab, item_bias, uid, pid, nid):
    """BPR.call (openrec/tf2/recommenders/bpr.py:21-37) -> (loss, l2_loss)."""
    u, p, n = lookup(user_tab, uid), lookup(item_tab, pid), lookup(item_tab, nid)
    bp, bn = lookup(item_bias, pid), lookup(item_bias, nid)
    loss, _ = pairwise_log_loss(u, p, n, bp, bn)
    return loss, l2_loss(u) + l2_loss(p) + l2_loss(n)


def ucml_forward(user_tab, item_tab, item_bias, uid, pid, nid, margin=0.5):
    """UCML.call (openrec/tf2/recommenders/ucml.py:21-42) -> (loss, l2_loss).
    loss is a SUM over the batch of hinge terms (ucml.py:39)."""
    dt = user_tab.dtype
    u, p, n = lookup(user_tab, uid), lookup(item_tab, pid), lookup(item_tab, nid)
    bp, bn = lookup(item_bias, pid), lookup(item_bias, nid)
    dp = ((u - p) ** 2).sum(axis=-1, keepdims=True, dtype=dt)
    dn = ((u - n) ** 2).sum(axis=-1, keepdims=True, dtype=dt)
    diff = ((-dp) + bp) - ((-dn) + bn)
    loss = np.maximum(dt.type(margin) - diff, 0).sum(dtype=dt)
    return loss, l2_loss(u) + l2_loss(p) + l2_loss(n)


def bce_with_logits(label, z):
    """keras BinaryCrossentropy(from_logits=True) elementwise [TF-mem]:
    max(z,0) - z*label + log1p(exp(-|z|))."""
    return np.maximum(z, 0) - z * label + np.log1p(np.exp(-np.abs(z)))


def gmf_forward(user_tab, item_tab, item_bias, w, uid, iid, label):
    """GMF.call (openrec/tf2/recommenders/gmf.py:22-34).  ``w`` is the [D,1] kernel of
    Dense(1, use_bias=False) (gmf.py:19, modules/multi_layer_perceptron.py:14-16).
    loss = mean BCE-with-logits; l2 includes 0.5*sum(w**2) (gmf.py:31-32)."""
    dt = user_tab.dtype
    u, i, b = lookup(user_tab, uid), lookup(item_tab, iid), lookup(item_bias, iid)
    z = ((u * i) @ w.reshape(-1, 1) + b).reshape(-1)
    loss = bce_with_logits(label.astype(dt), z).mean(dtype=dt)
    return loss, l2_loss(u) + l2_loss(i) + l2_loss(w)


def pointwise_mse_loss(u, i, b, label, a=1.0, bb=1.0, use_sigmoid=False):
    """PointwiseMSELoss.call (openrec/tf2/modules/pointwise_mse_loss.py:18-31)."""
    dt = u.dtype
    pred = (u * i).sum(axis=1, dtype=dt) + b.reshape(-1)
    if use_sigmoid:
        pred = sigmoid(pred)
    wgt = dt.type(a - bb) * label + dt.type(bb)
    return (wgt * (label - pred) ** 2).sum(dtype=dt), pred


def wrmf_forward(user_tab, item_tab, item_bias, uid, iid, label, a=1.0, b=1.0, use_sigmoid=False):
    """WRMF.call (openrec/tf2/recommenders/wrmf.py:21-34) -> (loss, l2_loss)."""
    u, i, bi = lookup(user_tab, uid), lookup(item_tab, iid), lookup(item_bias, iid)
    loss, _ = pointwise_mse_loss(u, i, bi, label.astype(u.dtype), a, b, use_sigmoid)
    return loss, l2_loss(u) + l2_loss(i)


# --------------------------------------------------------------------------------------
# closed-form gradients of  c_loss*loss + c_l2*l2_loss  (the examples differentiate the
# tuple (loss, l2_loss) => c_loss=c_l2=1; tf2_examples/bpr_citeulike.py:36-37, SURVEY Q3).
# Returned in TF's IndexedSlices form: per-lookup value rows, NOT deduplicated; the two
# lookups of the item table are concatenated p||n as tape.gradient does [TF-mem].
# --------------------------------------------------------------------------------------


def bpr_grads(user_tab, item_tab, item_bias, uid, pid, nid, c_loss=1.0, c_l2=1.0):
    """d(c_loss*loss + c_l2*l2)/d{gathered rows} for BPR (bpr.py:21-37,
    pairwise_log_loss.py:19-32).  maximum(x,-30) passes gradient when x >= -30
    (TF MaximumGrad tie rule [TF-mem])."""
    dt = user_tab.dtype
    B = len(uid)
    u, p, n = lookup(user_tab, uid), lookup(item_tab, pid), lookup(item_tab, nid)
    bp, bn = lookup(item_bias, pid), lookup(item_bias, nid)
    _, x = pairwise_log_loss(u, p, n, bp, bn)
    y = np.maximum(x, dt.type(-30.0))
    g = -(dt.type(c_loss) / dt.type(B)) * sigmoid(-y) * (x >= dt.type(-30.0))  # [B,1]
    g = g.astype(dt)
    c2 = dt.type(c_l2)
    return {
        "g": g.reshape(-1),
        "user": (np.asarray(uid), g * (p - n) + c2 * u),
        "item": (np.concatenate([pid, nid]), np.concatenate([g * u + c2 * p, -g * u + c2 * n])),
        "bias": (np.concatenate([pid, nid]), np.concatenate([g, -g])),
    }


def ucml_grads(user_tab, item_tab, item_bias, uid, pid, nid, margin=0.5, c_loss=1.0, c_l2=1.0):
    """Gradients for UCML (ucml.py:29-40).  hinge active when margin-diff >= 0
    (tf.maximum(x,0) passes gradient to x when x >= 0 [TF-mem])."""
    dt = user_tab.dtype
    u, p, n = lookup(user_tab, uid), lookup(item_tab, pid), lookup(item_tab, nid)
    bp, bn = lookup(item_bias, pid), lookup(item_bias, nid)
    dp = ((u - p) ** 2).sum(axis=-1, keepdims=True, dtype=dt)
    dn = ((u - n) ** 2).sum(axis=-1, keepdims=True, dtype=dt)
    h = dt.type(margin) - (((-dp) + bp) - ((-dn) + bn))
    a = (dt.type(c_loss) * (h >= 0)).astype(dt)  # [B,1]
    c2 = dt.type(c_l2)
    two = dt.type(2.0)
    return {
        "g": a.reshape(-1),
        "user": (np.asarray(uid), two * a * (n - p) + c2 * u),
        "item": (np.concatenate([pid, nid]),
                 np.concatenate([-two * a * (u - p) + c2 * p, two * a * (u - n) + c2 * n])),
        "bias": (np.concatenate([pid, nid]), np.concatenate([-a, a])),
    }


def gmf_grads(user_tab, item_tab, item_bias, w, uid, iid, label, c_loss=1.0, c_l2=1.0):
    """Gradients for GMF (gmf.py:22-34): dz = (sigmoid(z)-label)/B."""
    dt = user_tab.dtype
    B = len(uid)
    u, i, b = lookup(user_tab, uid), lookup(item_tab, iid), lookup(item_bias, iid)
    wv = w.reshape(1, -1)
    z = ((u * i) @ w.reshape(-1, 1) + b).reshape(-1)
    dz = (dt.type(c_loss) * (sigmoid(z) - label.astype(dt)) / dt.type(B)).reshape(-1, 1).astype(dt)
    c2 = dt.type(c_l2)
    return {
        "g": dz.reshape(-1),
        "user": (np.asarray(uid), dz * (wv * i) + c2 * u),
        "item": (np.asarray(iid), dz * (wv * u) + c2 * i),
        "bias": (np.asarray(iid), dz),
        "w": ((dz * (u * i)).sum(axis=0, dtype=dt) + c2 * w.reshape(-1)).reshape(w.shape),
    }


def wrmf_grads(user_tab, item_tab, item_bias, uid, iid, label, a=1.0, b=1.0, use_sigmoid=False,
               c_loss=1.0, c_l2=1.0):
    """Gradients for WRMF (wrmf.py:21-34, pointwise_mse_loss.py:22-31)."""
    dt = user_tab.dtype
    u, i, bi = lookup(user_tab, uid), lookup(item_tab, iid), lookup(item_bias, iid)
    label = label.astype(dt)
    _, pred = pointwise_mse_loss(u, i, bi, label, a, b, use_sigmoid)
    wgt = dt.type(a - b) * label + dt.type(b)
    dpred = dt.type(c_loss) * dt.type(-2.0) * wgt * (label - pred)
    if use_sigmoid:
        dpred = dpred * pred * (1 - pred)
    dpred = dpred.reshape(-1, 1).astype(dt)
    c2 = dt.type(c_l2)
    return {
        "g": dpred.reshape(-1),
        "user": (np.asarray(uid), dpred * i + c2 * u),
        "item": (np.asarray(iid), dpred * u + c2 * i),
        "bias": (np.asarray(iid), dpred),
    }


# --------------------------------------------------------------------------------------
# optimizers  [TF-mem]  (tf2_examples/bpr_citeulike.py:31,38 use keras Adam())
# --------------------------------------------------------------------------------------


def dedup(indices, values):
    """OptimizerV2._deduplicate_indexed_slices: unique(indices) +
    unsorted_segment_sum(values) [TF-mem].  Sum in batch order."""
    uniq, inv = unique_first_occurrence(indices)
    out = np.zeros((len(uniq),) + values.shape[1:], dtype=values.dtype)
    np.add.at(out, inv, values)
    return uniq, out


def sgd_sparse(var, indices, values, lr=0.01):
    """keras SGD sparse apply: var[idx] -= lr*G after dedup [TF-mem]."""
    idx, g = dedup(indices, values)
    var[idx] -= var.dtype.type(lr) * g


def adagrad_sparse(var, acc, indices, values, lr=0.001, eps=1e-7):
    """keras Adagrad (initial accumulator 0.1) ResourceSparseApplyAdagradV2 on the
    deduplicated rows: acc += G^2; var -= lr*G/(sqrt(acc)+eps) [TF-mem]."""
    idx, g = dedup(indices, values)
    dt = var.dtype
    a = acc[idx] + g * g
    acc[idx] = a
    var[idx] -= dt.type(lr) * g / (np.sqrt(a) + dt.type(eps))


def adam_lr_t(step, lr=0.001, beta1=0.9, beta2=0.999):
    """lr_t = lr*sqrt(1-b2^t)/(1-b1^t), t = 1-based step [TF-mem]."""
    return lr * np.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)


def adam_dense_on_sparse(var, m, v, indices, values, step, lr=0.001, beta1=0.9, beta2=0.999, eps=1e-7):
    """keras-2.0 Adam._resource_apply_sparse (NOT lazy, SURVEY Q5): m,v decay and the
    var update run over the WHOLE table; only the scatter-add is sparse [TF-mem]."""
    dt = var.dtype
    idx, g = dedup(indices, values)
    m *= dt.type(beta1)
    m[idx] += dt.type(1 - beta1) * g
    v *= dt.type(beta2)
    v[idx] += dt.type(1 - beta2) * g * g
    var -= dt.type(adam_lr_t(step, lr, beta1, beta2)) * m / (np.sqrt(v) + dt.type(eps))


def adam_lazy(var, m, v, indices, values, step, lr=0.001, beta1=0.9, beta2=0.999, eps=1e-7):
    """Row-sparse ("lazy") Adam: same formula restricted to the touched rows.
    NOT the reference's semantics; offered as an explicit mode."""
    dt = var.dtype
    idx, g = dedup(indices, values)
    mm = dt.type(beta1) * m[idx] + dt.type(1 - beta1) * g
    vv = dt.type(beta2) * v[idx] + dt.type(1 - beta2) * g * g
    m[idx], v[idx] = mm, vv
    var[idx] -= dt.type(adam_lr_t(step, lr, beta1, beta2)) * mm / (np.sqrt(vv) + dt.type(eps))


def adam_dense(var, m, v, grad, step, lr=0.001, beta1=0.9, beta2=0.999, eps=1e-7):
    """keras Adam dense apply (GMF w, MLP kernels/biases) [TF-mem]."""
    dt = var.dtype
    m *= dt.type(beta1)
    m += dt.type(1 - beta1) * grad
    v *= dt.type(beta2)
    v += dt.type(1 - beta2) * grad * grad
    var -= dt.type(adam_lr_t(step, lr, beta1, beta2)) * m / (np.sqrt(v) + dt.type(eps))


def adagrad_dense(var, acc, grad, lr=0.001, eps=1e-7):
    dt = var.dtype
    acc += grad * grad
    var -= dt.type(lr) * grad / (np.sqrt(acc) + dt.type(eps))


def sgd_dense(var, grad, lr=0.01):
    var -= var.dtype.type(lr) * grad


OPT_SGD, OPT_ADAGRAD, OPT_ADAM_LAZY, OPT_ADAM_DENSE = 0, 1, 2, 3


def apply_sparse(kind, var, s0, s1, indices, values, step, lr, eps=1e-7, beta1=0.9, beta2=0.999):
    if kind == OPT_SGD:
        sgd_sparse(var, indices, values, lr)
    elif kind == OPT_ADAGRAD:
        adagrad_sparse(var, s0, indices, values, lr, eps)
    elif kind == OPT_ADAM_LAZY:
        adam_lazy(var, s0, s1, indices, values, step, lr, beta1, beta2, eps)
    elif kind == OPT_ADAM_DENSE:
        adam_dense_on_sparse(var, s0, s1, indices, values, step, lr, beta1, beta2, eps)
    else:
        raise ValueError(kind)


def apply_dense(kind, var, s0, s1, grad, step, lr, eps=1e-7, beta1=0.9, beta2=0.999):
    if kind == OPT_SGD:
        sgd_dense(var, grad, lr)
    elif kind == OPT_ADAGRAD:
        adagrad_dense(var, s0, grad, lr, eps)
    else:
        adam_dense(var, s0, s1, grad, step, lr, beta1, beta2, eps)


# --------------------------------------------------------------------------------------
# full training steps: model(...) -> tape.gradient((loss,l2), vars) -> apply_gradients
# (tf2_examples/bpr_citeulike.py:33-39).  ``state`` = dict var_name -> (s0, s1).
# --------------------------------------------------------------------------------------


def pairwise_train_step(kind, user_tab, item_tab, item_bias, uid, pid, nid, opt_kind, state, step,
                        lr, margin=0.5, c_loss=1.0, c_l2=1.0, eps=1e-7, beta1=0.9, beta2=0.999):
    """kind 'bpr' | 'ucml'.  Mutates tables/state in place; returns (loss, l2_loss)
    computed on the PRE-step tables (TF gathers before any update)."""
    if kind == "bpr":
        out = bpr_forward(user_tab, item_tab, item_bias, uid, pid, nid)
        gr = bpr_grads(user_tab, item_tab, item_bias, uid, pid, nid, c_loss, c_l2)
    else:
        out = ucml_forward(user_tab, item_tab, item_bias, uid, pid, nid, margin)
        gr = ucml_grads(user_tab, item_tab, item_bias, uid, pid, nid, margin, c_loss, c_l2)
    for name, var in (("user", user_tab), ("item", item_tab), ("bias", item_bias)):
        s0, s1 = state.get(name, (None, None))
        idx, val = gr[name]
        apply_sparse(opt_kind, var, s0, s1, idx, val.reshape(len(idx), -1), step, lr, eps, beta1, beta2)
    return out


def pointwise_train_step(kind, user_tab, item_tab, item_bias, w, uid, iid, label, opt_kind, state, step,
                         lr, a=1.0, b=1.0, use_sigmoid=False, c_loss=1.0, c_l2=1.0,
                         eps=1e-7, beta1=0.9, beta2=0.999):
    """kind 'gmf' | 'wrmf'."""
    if kind == "gmf":
        out = gmf_forward(user_tab, item_tab, item_bias, w, uid, iid, label)
        gr = gmf_grads(user_tab, item_tab, item_bias, w, uid, iid, label, c_loss, c_l2)
    else:
        out = wrmf_forward(user_tab, item_tab, item_bias, uid, iid, label, a, b, use_sigmoid)
        gr = wrmf_grads(user_tab, item_tab, item_bias, uid, iid, label, a, b, use_sigmoid, c_loss, c_l2)
    for name, var in (("user", user_tab), ("item", item_tab), ("bias", item_bias)):
        s0, s1 = state.get(name, (None, None))
        idx, val = gr[name]
        apply_sparse(opt_kind, var, s0, s1, idx, val.reshape(len(idx), -1), step, lr, eps, beta1, beta2)
    if kind == "gmf":
        s0, s1 = state.get("w", (None, None))
        apply_dense(opt_kind, w, s0, s1, gr["w"], step, lr, eps, beta1, beta2)
    return out


def ucml_censor_vec(user_tab, item_tab, uid, pid, nid):
    """UCML.censor_vec (ucml.py:44-48): three sequential censors, in this order."""
    censor(user_tab, uid)
    censor(item_tab, pid)
    censor(item_tab, nid)


# --------------------------------------------------------------------------------------
# inference (full-catalogue scoring)
# --------------------------------------------------------------------------------------


def dot_inference(user_tab, item_tab, item_bias, uid):
    """BPR.inference / WRMF.inference (bpr.py:39-43, wrmf.py:36-40)."""
    return lookup(user_tab, uid) @ item_tab.T + item_bias.reshape(-1)


def ucml_inference(user_tab, item_tab, item_bias, uid):
    """UCML.inference (ucml.py:50-53): -||u-i||^2 + bias."""
    u = lookup(user_tab, uid)
    d = ((u[:, None, :] - item_tab[None, :, :]) ** 2).sum(axis=-1, dtype=user_tab.dtype)
    return -d + item_bias.reshape(-1)


def gmf_inference(user_tab, item_tab, item_bias, w, uid):
    """GMF.inference (gmf.py:36-41)."""
    u = lookup(user_tab, uid)
    return (u * w.reshape(1, -1)) @ item_tab.T + item_bias.reshape(-1)


# --------------------------------------------------------------------------------------
# DLRM  (openrec/tf2/recommenders/dlrm.py, modules/second_order_feature_interaction.py,
#        modules/multi_layer_perceptron.py)
# --------------------------------------------------------------------------------------


def second_order_interaction(inputs, self_interaction=False, mode="reference"):
    """SecondOrderFeatureInteraction.call (second_order_feature_interaction.py:12-34).

    mode='reference': bug-compatible (SURVEY Q1).  P = lower_tri(Z Z^T) (line 21);
    mask = upper_tri(ones) [- diag] (lines 24-27); boolean_mask picks, row-major, the
    strict-upper entries of a lower-triangular matrix => all zeros (only the F squared
    norms survive when self_interaction=True).
    mode='dlrm': what Naumov et al. intend -- the strictly-lower (or lower incl. diag)
    triangle of Z Z^T, row-major.  Both return [B, F(F-+1)/2]."""
    Z = np.stack(inputs, axis=1)  # [B,F,D]
    B, F, _ = Z.shape
    P = Z @ Z.transpose(0, 2, 1)
    if mode == "reference":
        P = np.tril(P)
        mask = np.triu(np.ones((F, F), dtype=bool), 0 if self_interaction else 1)
    elif mode == "dlrm":
        mask = np.tril(np.ones((F, F), dtype=bool), 0 if self_interaction else -1)
    else:
        raise ValueError(mode)
    return P[:, mask].reshape(B, -1)


def second_order_interaction_bwd(inputs, dout, self_interaction=False, mode="reference"):
    """Backward of the above wrt the stacked features Z [B,F,D]."""
    Z = np.stack(inputs, axis=1)
    B, F, _ = Z.shape
    dP = np.zeros((B, F, F), dtype=Z.dtype)
    if mode == "reference":
        mask = np.triu(np.ones((F, F), dtype=bool), 0 if self_interaction else 1)
        dP[:, mask] = dout
        dP = np.tril(dP)  # only the diagonal can survive
    else:
        mask = np.tril(np.ones((F, F), dtype=bool), 0 if self_interaction else -1)
        dP[:, mask] = dout
    # P = Z Z^T  => dZ = (dP + dP^T) Z
    return (dP + dP.transpose(0, 2, 1)) @ Z


def _act(x, name):
    if name == "relu":
        return np.maximum(x, 0)
    if name == "sigmoid":
        return sigmoid(x)
    return x


def _act_bwd(y, dy, name):
    """Gradient through the activation given its OUTPUT y."""
    if name == "relu":
        return dy * (y > 0)
    if name == "sigmoid":
        return dy * y * (1 - y)
    return dy


def mlp_forward(x, weights, biases, activation="relu", out_activation=None):
    """MLP (multi_layer_perceptron.py:5-18): Dense(units, activation) stack; returns the list of
    layer outputs (post-activation), last = result."""
    outs = []
    L = len(weights)
    for l, (W, b) in enumerate(zip(weights, biases)):
        z = x @ W
        if b is not None:
            z = z + b
        x = _act(z, out_activation if l == L - 1 else activation)
        outs.append(x)
    return outs


def mlp_backward(x0, weights, outs, dy, activation="relu", out_activation=None):
    """Returns (dx0, [dW], [db])."""
    L = len(weights)
    dWs, dbs = [None] * L, [None] * L
    for l in range(L - 1, -1, -1):
        dz = _act_bwd(outs[l], dy, out_activation if l == L - 1 else activation)
        xin = x0 if l == 0 else outs[l - 1]
        dWs[l] = xin.T @ dz
        dbs[l] = dz.sum(axis=0, dtype=dz.dtype)
        dy = dz @ weights[l].T
    return dy, dWs, dbs


def dlrm_forward(emb_tables, bot_w, bot_b, top_w, top_b, dense, sparse, *, self_interaction=False,
                 sigmoid_bot=False, sigmoid_top=True, loss_threshold=0.0, interaction_mode="reference"):
    """DLRM.inference (dlrm.py:76-100) with arch_interaction_op='dot'.  Returns a cache dict
    with 'pred' [B]."""
    embs = [lookup(t, sparse[:, k]) for k, t in enumerate(emb_tables)]  # dlrm.py:83-85
    bot = mlp_forward(dense, bot_w, bot_b, "relu", "sigmoid" if sigmoid_bot else "relu")  # :34-35,87
    feats = embs + [bot[-1]]
    inter = second_order_interaction(feats, self_interaction, interaction_mode)  # :91
    top_in = np.concatenate([bot[-1], inter], axis=1)  # :90
    top = mlp_forward(top_in, top_w, top_b, "relu", "sigmoid" if sigmoid_top else "relu")
    pred = top[-1]
    clip = None
    if 0.0 < loss_threshold < 1.0:  # :97-98
        lo, hi = pred.dtype.type(loss_threshold), pred.dtype.type(1.0 - loss_threshold)
        clip = (pred >= lo) & (pred <= hi)
        pred = np.clip(pred, lo, hi)
    return dict(embs=embs, bot=bot, feats=feats, inter=inter, top_in=top_in, top=top,
                pred=pred.reshape(-1), clip=clip)


def dlrm_loss(pred, label, loss_func="mse"):
    """keras MeanSquaredError / BinaryCrossentropy on probabilities (dlrm.py:52-55) [TF-mem:
    BCE clips p to [1e-7, 1-1e-7] and adds 1e-7 inside the logs].  Returns (loss, dloss/dpred)."""
    dt = pred.dtype
    B = dt.type(len(pred))
    label = label.astype(dt)
    if loss_func == "mse":
        return ((label - pred) ** 2).mean(dtype=dt), dt.type(2.0) * (pred - label) / B
    eps = dt.type(1e-7)
    ph = np.clip(pred, eps, 1 - eps)
    loss = -(label * np.log(ph + eps) + (1 - label) * np.log(1 - ph + eps)).mean(dtype=dt)
    inside = (pred >= eps) & (pred <= 1 - eps)
    d = -(label / (ph + eps) - (1 - label) / (1 - ph + eps)) / B
    return loss, d * inside


def dlrm_backward(cache, emb_tables, bot_w, top_w, dense, sparse, dpred, *, self_interaction=False,
                  sigmoid_bot=False, sigmoid_top=True, interaction_mode="reference"):
    """Backprop of dlrm_forward.  Returns dict: 'emb' -> list of per-lookup grad rows [B,D] per table
    (IndexedSlices values, indices = sparse[:,k]), 'bot_w','bot_b','top_w','top_b' lists."""
    dy = dpred.reshape(-1, 1)
    if cache["clip"] is not None:
        dy = dy * cache["clip"]
    dtop_in, dtw, dtb = mlp_backward(cache["top_in"], top_w, cache["top"], dy, "relu",
                                     "sigmoid" if sigmoid_top else "relu")
    mb = cache["bot"][-1].shape[1]
    ddense_vec = dtop_in[:, :mb]
    dinter = dtop_in[:, mb:]
    dZ = second_order_interaction_bwd(cache["feats"], dinter, self_interaction, interaction_mode)
    demb = [dZ[:, k, :] for k in range(len(emb_tables))]
    ddense_vec = ddense_vec + dZ[:, len(emb_tables), :]
    _, dbw, dbb = mlp_backward(dense, bot_w, cache["bot"], ddense_vec, "relu",
                               "sigmoid" if sigmoid_bot else "relu")
    return dict(emb=demb, bot_w=dbw, bot_b=dbb, top_w=dtw, top_b=dtb)


# --------------------------------------------------------------------------------------
# ranking metrics (openrec/tf2/metrics/ranking_metrics.py:8-69), per user
# --------------------------------------------------------------------------------------


def auc(pos_mask, pred, excl_mask):
    """AUC (ranking_metrics.py:8-25): count(eval_pred <= pos_pred)/(n_pos*n_eval)."""
    out = np.zeros(len(pred), dtype=np.float32)
    for r in range(len(pred)):
        ev = ~(pos_mask[r] | excl_mask[r])
        e, p = pred[r][ev], pred[r][pos_mask[r]]
        out[r] = np.float32(np.count_nonzero(e[None, :] <= p[:, None])) / np.float32(p.size * np.count_nonzero(ev))
    return out


def _rank_above(pos_mask, pred, excl_mask, r):
    s = np.exp(pred[r]) * (~excl_mask[r]).astype(pred.dtype)  # :33,56
    p = s[pos_mask[r]]
    return np.count_nonzero(s[None, :] > p[:, None], axis=1).astype(np.float32), p.size


def ndcg(pos_mask, pred, excl_mask, at=(100,)):
    """NDCG (ranking_metrics.py:28-47): DCG@k without ideal normaliser (SURVEY Q10)."""
    out = np.zeros((len(pred), len(at)), dtype=np.float32)
    for r in range(len(pred)):
        ra, _ = _rank_above(pos_mask, pred, excl_mask, r)
        rec = (np.float32(1) / (np.log(ra + 2) / np.log(np.float32(2.0)))).astype(np.float32)
        for j, k in enumerate(at):
            out[r, j] = (rec * (ra < k)).sum(dtype=np.float32)
    return out


def recall(pos_mask, pred, excl_mask, at=(100,)):
    """Recall (ranking_metrics.py:50-69)."""
    out = np.zeros((len(pred), len(at)), dtype=np.float32)
    for r in range(len(pred)):
        ra, npos = _rank_above(pos_mask, pred, excl_mask, r)
        for j, k in enumerate(at):
            out[r, j] = np.float32(np.count_nonzero(ra < k)) / np.float32(npos)
    return out
