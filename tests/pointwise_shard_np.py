"""TEST INFRASTRUCTURE: numpy restatements of the row-sharded GMF / WRMF step's kernels (orx_pointwise_shard_lookups,
orx_pointwise_serve, orx_pointwise_grad_rows, orx_rows_scale) and ``PointwiseShardEngine``, the oracle-backed engine of
tests/fake_engine.py with these entry points, the numpy orx_lookup_bucket / orx_rows_segment_sum of tests/dlrm_shard_np.py
and orx_sparse_apply_strided's skipping of negative ids, so the sharded pointwise step runs on CPU over gloo.  The
gradient arithmetic is the oracle's (oracle/openrec_oracle.py gmf_* / wrmf_*)."""
from __future__ import annotations

import numpy as np
import torch

import dlrm_shard_np
import fake_engine
from fake_engine import FakeEngine
from oracle import openrec_oracle as O


def shard_lookups_np(uid, iid, U, I):
    """-> int32 [B, 2]: (uid, iid), or (-1, -1) when either id is out of range."""
    u, i = np.asarray(uid, np.int64), np.asarray(iid, np.int64)
    ok = (u >= 0) & (u < U) & (i >= 0) & (i < I)
    return np.where(ok[:, None], np.stack([u, i], 1), -1).astype(np.int32)


def serve_np(user, item, bias, local_users, local_items, Lu, req, ld):
    """-> (rows [n, ld], user_local [n], item_local [n]) as orx_pointwise_serve defines them."""
    q = np.asarray(req, np.int64)
    D = user.shape[1]
    rows = np.zeros((len(q), ld), np.float32)
    is_u = (q >= 0) & (q < local_users)
    is_i = (q >= Lu) & (q - Lu < local_items)
    rows[is_u, :D] = user[q[is_u]]
    rows[is_i, :D] = item[q[is_i] - Lu]
    rows[is_i, D] = np.asarray(bias).reshape(-1)[q[is_i] - Lu]
    return rows, np.where(is_u, q, -1).astype(np.int32), np.where(is_i, q - Lu, -1).astype(np.int32)


def grad_rows_np(kind, rows, dim, slot, label, w, inv_B, a=1.0, b=1.0, use_sigmoid=False, c_loss=1.0, c_l2=1.0,
                 add_w_terms=False):
    """-> (d_rows [2B, ld], gw [dim] or None, (loss, l2)) in float64, from the oracle's closed-form gradients."""
    r = np.asarray(rows, np.float64)
    sl = np.asarray(slot).reshape(-1, 2)
    lab = np.asarray(label, np.float64)
    B, ld = len(lab), r.shape[1]
    ok = (sl[:, 0] >= 0) & (sl[:, 1] >= 0)
    us, it = sl[ok, 0], sl[ok, 1]
    emb, bias = r[:, :dim], r[:, dim:dim + 1]
    d = np.zeros((2 * B, ld))
    wv = None if w is None else np.asarray(w, np.float64).reshape(-1, 1)
    gw = None if kind != 0 else np.zeros(dim)
    loss = l2 = 0.0
    if ok.any():
        if kind == 0:
            nv = int(ok.sum())
            loss, l2 = O.gmf_forward(emb, emb, bias, wv, us, it, lab[ok])
            loss, l2 = loss * nv * inv_B, l2 - O.l2_loss(wv)
            gr = O.gmf_grads(emb, emb, bias, wv, us, it, lab[ok], c_loss * nv * inv_B, c_l2)
            gw = (gr["g"][:, None] * emb[us] * emb[it]).sum(0)
        else:
            loss, l2 = O.wrmf_forward(emb, emb, bias, us, it, lab[ok], a, b, use_sigmoid)
            gr = O.wrmf_grads(emb, emb, bias, us, it, lab[ok], a, b, use_sigmoid, c_loss, c_l2)
        t = np.flatnonzero(ok)
        d[2 * t, :dim] = gr["user"][1]
        d[2 * t + 1, :dim] = gr["item"][1]
        d[2 * t + 1, dim] = gr["bias"][1].reshape(-1)
    if kind == 0 and add_w_terms:
        gw = gw + c_l2 * wv.reshape(-1)
        l2 = l2 + O.l2_loss(wv)
    return d, gw, (float(loss), float(l2))


class PointwiseShardEngine(FakeEngine):
    """The oracle-backed CPU engine with the entry points of the row-sharded pointwise step (tests only)."""

    lookup_bucket = dlrm_shard_np._lookup_bucket
    rows_segment_sum = dlrm_shard_np._rows_segment_sum

    def pointwise_shard_lookups(self, uid, iid, total_users, total_items):
        return torch.from_numpy(shard_lookups_np(uid.numpy(), iid.numpy(), total_users, total_items))

    def pointwise_serve(self, user, item, bias, local_users, local_items, user_rows_per_rank, req, ld):
        rows, ul, il = serve_np(user.numpy(), item.numpy(), bias.numpy(), local_users, local_items,
                                user_rows_per_rank, req.numpy(), ld)
        return torch.from_numpy(rows), torch.from_numpy(ul), torch.from_numpy(il)

    def pointwise_grad_rows(self, kind, rows, dim, slot, label, w, inv_B, a=1.0, b=1.0, use_sigmoid=False,
                            c_loss=1.0, c_l2=1.0, add_w_terms=False):
        d, gw, out = grad_rows_np(kind, rows.numpy(), dim, slot.numpy(), label.numpy(),
                                  None if w is None else w.numpy(), inv_B, a, b, use_sigmoid, c_loss, c_l2,
                                  add_w_terms)
        f32 = lambda x: torch.from_numpy(np.asarray(x, np.float32))   # noqa: E731
        return f32(d), None if gw is None else f32(gw), f32(out)

    def sparse_apply_rows(self, tab, ids, values, o):
        keep = ids.numpy() >= 0
        vals = values.numpy()
        fake_engine.O.apply_sparse(o.kind, fake_engine._np(tab.var), fake_engine._np(tab.s0),
                                   fake_engine._np(tab.s1), ids.numpy()[keep],
                                   np.ascontiguousarray(vals[keep]).reshape(int(keep.sum()), vals.shape[1]), o.step,
                                   o.lr, o.eps, o.beta1, o.beta2)

    def rows_scale(self, x, scale):
        v = x.view(torch.float32).reshape(-1, scale.numel())
        v.copy_(v * scale.reshape(1, -1))


def install():
    """Route the product's host code to a PointwiseShardEngine on CPU tensors (tests only)."""
    import openrec_b200.native as N
    fake_engine.install()
    eng = PointwiseShardEngine()
    N.engine = lambda device=None: eng
    return eng
