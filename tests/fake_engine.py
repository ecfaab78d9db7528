"""TEST INFRASTRUCTURE: an oracle-backed stand-in for openrec_b200.native.Engine on CPU tensors.

It lets the HOST logic (sharded-step orchestration over gloo, the tensorflow step protocol driving the
unmodified reference examples) run in the GPU-less build container.  It is never importable from the
product (lives under tests/), and the arithmetic it provides is the numpy oracle -- the thing the CUDA
kernels are checked against, not a fallback for them."""
from __future__ import annotations

import numpy as np
import torch

from oracle import openrec_oracle as O


class FakeTable:
    def __init__(self, var, s0=None, s1=None):
        self.var, self.s0, self.s1 = var, s0, s1


class FakeOpt:
    def __init__(self, kind, lr, eps=1e-7, beta1=0.9, beta2=0.999, step=1):
        self.kind, self.lr, self.eps, self.beta1, self.beta2, self.step = kind, lr, eps, beta1, beta2, step


def _np(t):
    return None if t is None else t.numpy()


class FakeEngine:
    device = torch.device("cpu")
    make_table = staticmethod(FakeTable)
    make_opt = staticmethod(FakeOpt)

    def fill_uniform(self, dst, lo, hi, seed):
        g = torch.Generator().manual_seed(int(seed) % (2 ** 31))
        dst.copy_(torch.rand(dst.shape, generator=g) * (hi - lo) + lo)

    def gather(self, tab, ids, n_bad=None):
        return tab[ids.long().reshape(-1)].clone()

    def censor(self, tab, ids, min_norm=0.1):
        O.censor(tab.numpy(), ids.numpy().reshape(-1), min_norm)

    def owner_bucket_combined(self, ids, n_user, total_users, world):
        a = ids.numpy()
        owner = a % world
        user_rows = (total_users - owner + world - 1) // world
        local = a // world + np.where(np.arange(len(a)) >= n_user, user_rows, 0)
        order = np.argsort(owner, kind="stable")
        slot = np.empty(len(a), dtype=np.int32)
        slot[order] = np.arange(len(a), dtype=np.int32)
        return (torch.from_numpy(np.bincount(owner, minlength=world).astype(np.int32)),
                torch.from_numpy(local[order].astype(np.int32)), torch.from_numpy(slot))

    def pairwise_grad_rows(self, kind, rows, dim, uslot, pslot, nslot, inv_B, d_rows, out4, margin=0.5, c_loss=1.0,
                           c_l2=1.0):
        r = rows.numpy().astype(np.float64)
        emb, bias = r[:, :dim], r[:, dim:dim + 1]
        us, ps, ns = (t.numpy() for t in (uslot, pslot, nslot))
        B = len(us)
        if kind == 0:
            loss, l2 = O.bpr_forward(emb, emb, bias, us, ps, ns)
            gr = O.bpr_grads(emb, emb, bias, us, ps, ns, c_loss * B * inv_B, c_l2)
            loss = loss * B * inv_B
        else:
            loss, l2 = O.ucml_forward(emb, emb, bias, us, ps, ns, margin)
            gr = O.ucml_grads(emb, emb, bias, us, ps, ns, margin, c_loss, c_l2)
        d = d_rows.numpy()
        d[np.concatenate([us, ps, ns]), dim:] = 0.0
        d[gr["user"][0], :dim] = gr["user"][1]
        d[gr["item"][0], :dim] = gr["item"][1]
        d[gr["bias"][0], dim] = gr["bias"][1].reshape(-1)
        out4[0], out4[1] = float(loss), float(l2)

    def sparse_apply(self, tab, ids, values, o):
        if ids is None or ids.numel() == 0:
            return
        O.apply_sparse(o.kind, _np(tab.var), _np(tab.s0), _np(tab.s1), ids.numpy(),
                       values.numpy().reshape(ids.numel(), -1), o.step, o.lr, o.eps, o.beta1, o.beta2)


# ---------------------------------------------------------------------------------------
# full-engine surface for driving the tensorflow step protocol on CPU (reference examples)
# ---------------------------------------------------------------------------------------
def _state(*tabs):
    return {k: (_np(t.s0), _np(t.s1)) for k, t in zip(("user", "item", "bias", "w"), tabs) if t is not None}


def _pairwise_step(self, kind, user, item, bias, uid, pid, nid, o, out4, margin=0.5, c_loss=1.0, c_l2=1.0):
    loss, l2 = O.pairwise_train_step("bpr" if kind == 0 else "ucml", user.var.numpy(), item.var.numpy(),
                                     bias.var.numpy(), uid.numpy(), pid.numpy(), nid.numpy(), o.kind,
                                     _state(user, item, bias), o.step, o.lr, margin, c_loss, c_l2, o.eps, o.beta1,
                                     o.beta2)
    out4[0], out4[1], out4[2], out4[3] = float(loss), float(l2), 0.0, 0.0


def _pairwise_fwd(self, kind, user, item, bias, uid, pid, nid, out4, margin=0.5):
    f = O.bpr_forward if kind == 0 else (lambda *a: O.ucml_forward(*a, margin=margin))
    loss, l2 = f(user.var.numpy(), item.var.numpy(), bias.var.numpy(), uid.numpy(), pid.numpy(), nid.numpy())
    out4[0], out4[1] = float(loss), float(l2)


def _score_all(self, kind, user_tab, uid, item_tab, item_bias, scale=None):
    u = user_tab.numpy()[uid.numpy().reshape(-1)]
    if scale is not None:
        u = u * scale.numpy().reshape(1, -1)
    if kind == 0:
        s = u @ item_tab.numpy().T + item_bias.numpy().reshape(-1)
    else:
        s = -((u[:, None, :] - item_tab.numpy()[None]) ** 2).sum(-1) + item_bias.numpy().reshape(-1)
    return torch.from_numpy(s.astype(np.float32))


def _rank_metrics(self, pred, pos, excl, at=(), want=("auc", "ndcg", "recall")):
    p, m, x = pred.numpy(), pos.numpy().astype(bool), excl.numpy().astype(bool)
    return (torch.from_numpy(O.auc(m, p, x)) if "auc" in want else None,
            torch.from_numpy(O.ndcg(m, p, x, tuple(at))) if "ndcg" in want else None,
            torch.from_numpy(O.recall(m, p, x, tuple(at))) if "recall" in want else None)


FakeEngine.pairwise_step = _pairwise_step
FakeEngine.pairwise_fwd = _pairwise_fwd
FakeEngine.score_all = _score_all
FakeEngine.rank_metrics = _rank_metrics


def install():
    """Route the product's host code to the oracle-backed engine on CPU tensors (tests only)."""
    import openrec_b200.native as N
    import openrec_b200.tfshim.core as core
    fake = FakeEngine()
    core.device = lambda: torch.device("cpu")
    N.engine = lambda device=None: fake
    N.table = FakeTable
    N.opt = FakeOpt
    N.ids32 = lambda t: t.to(torch.int32).contiguous().reshape(-1)
    import openrec_b200.tfshim.keras.layers as L
    import openrec_b200.tfshim.keras.metrics as M
    L.device = core.device
    M.device = core.device
    import openrec_b200.tf2.metrics.dict_mean as DM
    DM.device = core.device
    return fake


# ---------------------------------------------------------------------------------------
# DLRM pieces (oracle arithmetic on CPU views; in-place into the caller's tensors like liborx)
# ---------------------------------------------------------------------------------------
_ACT = {0: None, 1: "relu", 2: "sigmoid"}


def _gather_strided(self, tab, ids2d, col, out2d):
    out2d.copy_(tab[ids2d[:, col].long()])


def _mlp_fwd(self, x, w, bias, act, y):
    z = x.numpy().astype(np.float64) @ w.numpy().astype(np.float64)
    if bias is not None:
        z = z + bias.numpy()
    y.copy_(torch.from_numpy(O._act(z, _ACT[act]).astype(np.float32)))


def _mlp_bwd(self, x, y, w, act, dy, dx, dw, db):
    dz = O._act_bwd(y.numpy().astype(np.float64), dy.numpy().astype(np.float64), _ACT[act])
    dy.copy_(torch.from_numpy(dz.astype(np.float32)))
    dw.copy_(torch.from_numpy((x.numpy().astype(np.float64).T @ dz).astype(np.float32)))
    if db is not None:
        db.copy_(torch.from_numpy(dz.sum(0).astype(np.float32)))
    if dx is not None:
        dx.copy_(torch.from_numpy((dz @ w.numpy().astype(np.float64).T).astype(np.float32)))


def _feats(emb3d, dense2d):
    return [emb3d[:, k, :].numpy().astype(np.float64) for k in range(emb3d.shape[1])] + [dense2d.numpy().astype(np.float64)]


def _interact_fwd(self, emb3d, dense2d, self_interaction, mode, out2d):
    r = O.second_order_interaction(_feats(emb3d, dense2d), bool(self_interaction), "reference" if mode == 0 else "dlrm")
    out2d.copy_(torch.from_numpy(r.astype(np.float32)))


def _interact_bwd(self, emb3d, dense2d, dout2d, self_interaction, mode, demb3d, ddense2d):
    dZ = O.second_order_interaction_bwd(_feats(emb3d, dense2d), dout2d.numpy().astype(np.float64),
                                        bool(self_interaction), "reference" if mode == 0 else "dlrm")
    T = emb3d.shape[1]
    demb3d.copy_(torch.from_numpy(dZ[:, :T, :].astype(np.float32)))
    ddense2d.add_(torch.from_numpy(dZ[:, T, :].astype(np.float32)))


def _pred_loss(self, pred, label, kind, clip, pred_out, dpred, out4):
    p = pred.numpy().astype(np.float64)
    passed = np.ones_like(p)
    if 0.0 < clip < 1.0:
        passed = ((p >= clip) & (p <= 1 - clip)).astype(np.float64)
        p = np.clip(p, clip, 1 - clip)
    loss, d = O.dlrm_loss(p, label.numpy(), "mse" if kind == 0 else "bce")
    if pred_out is not None:
        pred_out.copy_(torch.from_numpy(p.astype(np.float32)))
    if dpred is not None:
        dpred.copy_(torch.from_numpy((d * passed).astype(np.float32)))
    out4[0] = float(loss)


def _sparse_apply_strided(self, tab, ids2d, col, values3d, o):
    O.apply_sparse(o.kind, _np(tab.var), _np(tab.s0), _np(tab.s1), ids2d[:, col].numpy(),
                   values3d[:, col, :].numpy(), o.step, o.lr, o.eps, o.beta1, o.beta2)


def _dense_apply(self, var, s0, s1, grad, o):
    O.apply_dense(o.kind, var.numpy(), _np(s0), _np(s1), grad.numpy(), o.step, o.lr, o.eps, o.beta1, o.beta2)


for _n, _f in (("gather_strided", _gather_strided), ("mlp_fwd", _mlp_fwd), ("mlp_bwd", _mlp_bwd),
               ("interact_fwd", _interact_fwd), ("interact_bwd", _interact_bwd), ("pred_loss", _pred_loss),
               ("sparse_apply_strided", _sparse_apply_strided), ("dense_apply", _dense_apply)):
    setattr(FakeEngine, _n, _f)
