"""float64 restatement of the DCN-v2 cross network (CrossNetwork, orx_cross_fwd / orx_cross_bwd) and of one training step
of DLRM(arch_interaction_op="cross"), composed from the oracle's MLP and loss pieces and the optimizer restatements of
tests/rowwise_bar.py and tests/momentum_bar.py.  cross_forward / cross_backward also take float64 torch tensors, and
loss_and_grads_t restates the whole forward and backward in torch float64 on any device (the bench.py-shape checks).

A cross layer is a list of projections (kernel [in, out], bias or None), applied in order without activation:
[(V, None), (U, b)] at low rank, [(K, b)] at full rank.  x_{l+1} = x0 * y_l + x_l with y_l the last projection."""
import numpy as np

import dlrm_bags_np as NB
import momentum_bar as MB
import rowwise_bar as RB
from oracle import openrec_oracle as O

OPT_ROWWISE_ADAGRAD, OPT_MOMENTUM, OPT_NESTEROV = RB.OPT_ROWWISE_ADAGRAD, MB.OPT_MOMENTUM, MB.OPT_NESTEROV


def cross_forward(x0, layers):
    """-> (xs = [x_0 .. x_L], acts = per layer the outputs of its projections, y_l last)."""
    xs, acts = [x0], []
    for projs in layers:
        h, outs = xs[-1], []
        for w, b in projs:
            h = h @ w + (0.0 if b is None else b)
            outs.append(h)
        xs.append(x0 * outs[-1] + xs[-1])
        acts.append(outs)
    return xs, acts


def cross_backward(x0, layers, xs, acts, G):
    """G = dL/dx_L -> (dL/dx0, per layer [(dw, db or None)] in projection order)."""
    A = x0 * 0.0
    grads = [None] * len(layers)
    for l in range(len(layers) - 1, -1, -1):
        dy = G * x0
        A = A + G * acts[l][-1]
        g, d = [None] * len(layers[l]), dy
        for j in range(len(layers[l]) - 1, -1, -1):
            w, b = layers[l][j]
            xin = xs[l] if j == 0 else acts[l][j - 1]
            g[j] = (xin.T @ d, None if b is None else d.sum(0))
            d = d @ w.T
        grads[l] = g
        G = G + d
    return G + A, grads


def cross_shapes(W, num_layers, projection_dim):
    """The cross variables' shapes in model order: per layer v, u, bias (low rank) or kernel, bias (full rank)."""
    per = [(W, W), (W,)] if projection_dim is None else [(W, projection_dim), (projection_dim, W), (W,)]
    return per * num_layers


def cross_layers(cvars, projection_dim):
    """The model-order cross variables -> layers of (kernel, bias or None) projections."""
    if projection_dim is None:
        return [[(cvars[i], cvars[i + 1])] for i in range(0, len(cvars), 2)]
    return [[(cvars[i], None), (cvars[i + 1], cvars[i + 2])] for i in range(0, len(cvars), 3)]


def split_dense(dvars, n_bot, n_top, projection_dim):
    """Model-order Dense variables (bottom kernel, bias, .., top kernel, bias, .., cross) -> (bot_w, bot_b, top_w,
    top_b, layers)."""
    bot, top, cross = dvars[:2 * n_bot], dvars[2 * n_bot:2 * (n_bot + n_top)], dvars[2 * (n_bot + n_top):]
    return bot[0::2], bot[1::2], top[0::2], top[1::2], cross_layers(cross, projection_dim)


def forward(embs, bot_w, bot_b, top_w, top_b, layers, dense):
    """DLRM-DCN inference from the looked-up (or pooled) embeddings embs [T] of [B, D]: x0 = (bottom output | embs)."""
    bot = O.mlp_forward(dense, bot_w, bot_b, "relu", "relu")
    x0 = np.concatenate([bot[-1]] + list(embs), axis=1)
    xs, acts = cross_forward(x0, layers)
    top = O.mlp_forward(xs[-1], top_w, top_b, "relu", "sigmoid")
    return dict(bot=bot, x0=x0, xs=xs, acts=acts, top=top, pred=top[-1].reshape(-1))


def backward(cache, bot_w, top_w, layers, dense, dpred):
    """-> dict emb [T] of [B, D] (dL/d the embedding rows), bot_w, bot_b, top_w, top_b, cross (per layer pairs)."""
    dxL, dtw, dtb = O.mlp_backward(cache["xs"][-1], top_w, cache["top"], dpred.reshape(-1, 1), "relu", "sigmoid")
    dx0, cg = cross_backward(cache["x0"], layers, cache["xs"], cache["acts"], dxL)
    D = cache["bot"][-1].shape[1]
    T = dx0.shape[1] // D - 1
    _, dbw, dbb = O.mlp_backward(dense, bot_w, cache["bot"], dx0[:, :D], "relu", "relu")
    return dict(emb=[dx0[:, D * (k + 1):D * (k + 2)] for k in range(T)], bot_w=dbw, bot_b=dbb, top_w=dtw, top_b=dtb,
                cross=cg)


def embeddings(tabs, sparse, col_off, mean):
    """One-hot (col_off None): tab_k[sparse[:, k]]; multi-hot: the pooled bags."""
    if col_off is None:
        return [t[sparse[:, k]] for k, t in enumerate(tabs)]
    Z, _ = NB.pool64(tabs, sparse, col_off, mean)
    return [Z[:, k] for k in range(len(tabs))]


def apply_sparse(kind, var, s0, s1, ids, rows, step, lr, momentum=0.0):
    if kind == OPT_ROWWISE_ADAGRAD:
        RB.adagrad_rowwise_sparse(var, s0, ids, rows, lr)
    elif kind in (OPT_MOMENTUM, OPT_NESTEROV):
        MB.momentum_sparse(var, s0, ids, rows, lr, momentum, kind == OPT_NESTEROV)
    else:
        O.apply_sparse(kind, var, s0, s1, ids, rows, step, lr)


def apply_dense(kind, var, s0, s1, grad, step, lr, momentum=0.0):
    """Dense variables keep element-wise slots under row-wise Adagrad."""
    if kind == OPT_ROWWISE_ADAGRAD:
        O.adagrad_dense(var, s0, grad, lr)
    elif kind in (OPT_MOMENTUM, OPT_NESTEROV):
        MB.momentum_dense(var, s0, grad, lr, momentum, kind == OPT_NESTEROV)
    else:
        O.apply_dense(kind, var, s0, s1, grad, step, lr)


def train_step(kind, tabs, dvars, st, step, lr, dense, sparse, label, n_bot, n_top, projection_dim, col_off=None,
               mean=False, momentum=0.0, apply_tables=None):
    """One oracle step of DLRM(arch_interaction_op="cross") with MSE, in place on tabs (only those in apply_tables,
    default all) and dvars (model order), st the optimizer slots (tables first).  -> loss."""
    bot_w, bot_b, top_w, top_b, layers = split_dense(dvars, n_bot, n_top, projection_dim)
    cache = forward(embeddings(tabs, sparse, col_off, mean), bot_w, bot_b, top_w, top_b, layers, dense)
    loss, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = backward(cache, bot_w, top_w, layers, dense, dpred)
    T = len(tabs)
    for k in range(T) if apply_tables is None else apply_tables:
        if col_off is None:
            ids, rows = sparse[:, k].astype(np.int64), gr["emb"][k]
        else:
            ids, rows = NB.bag_grad_rows(sparse, col_off, k, tabs[k].shape[0], gr["emb"][k], mean)
        apply_sparse(kind, tabs[k], st[k][0], st[k][1], ids, rows, step, lr, momentum)
    dgr = [g for l in range(n_bot) for g in (gr["bot_w"][l], gr["bot_b"][l])]
    dgr += [g for l in range(n_top) for g in (gr["top_w"][l], gr["top_b"][l])]
    dgr += [g for layer in gr["cross"] for pair in layer for g in pair if g is not None]
    assert len(dgr) == len(dvars)
    for j, g in enumerate(dgr):
        apply_dense(kind, dvars[j], st[T + j][0], st[T + j][1], g, step, lr, momentum)
    return loss


def loss_and_grads_t(embs, bot_w, bot_b, top_w, top_b, layers, dense, label):
    """The DLRM-DCN forward and backward (relu bottom MLP, sigmoid top output, MSE) on float64 torch tensors.  -> (loss,
    dL/dx0 [B, W], the Dense and cross gradients in model order)."""
    import torch
    bot, h = [], dense
    for w, b in zip(bot_w, bot_b):
        h = (h @ w + b).clamp_min(0)
        bot.append(h)
    x0 = torch.cat([bot[-1]] + list(embs), 1)
    xs, acts = cross_forward(x0, layers)
    top, h = [], xs[-1]
    for j, (w, b) in enumerate(zip(top_w, top_b)):
        h = h @ w + b
        h = torch.sigmoid(h) if j == len(top_w) - 1 else h.clamp_min(0)
        top.append(h)
    pred = top[-1].reshape(-1)
    d = (2 * (pred - label) / pred.shape[0]).reshape(-1, 1)
    g_top = [None] * len(top_w)
    for j in range(len(top_w) - 1, -1, -1):
        d = d * top[j] * (1 - top[j]) if j == len(top_w) - 1 else d * (top[j] > 0)
        g_top[j] = ((xs[-1] if j == 0 else top[j - 1]).T @ d, d.sum(0))
        d = d @ top_w[j].T
    dx0, g_cross = cross_backward(x0, layers, xs, acts, d)
    d = dx0[:, :bot[-1].shape[1]]
    g_bot = [None] * len(bot_w)
    for j in range(len(bot_w) - 1, -1, -1):
        d = d * (bot[j] > 0)
        g_bot[j] = ((dense if j == 0 else bot[j - 1]).T @ d, d.sum(0))
        d = d @ bot_w[j].T
    grads = [t for pair in g_bot + g_top for t in pair]
    grads += [t for layer in g_cross for pair in layer for t in pair if t is not None]
    return float(((pred - label) ** 2).mean()), dx0, grads
