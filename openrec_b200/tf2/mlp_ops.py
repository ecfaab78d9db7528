"""Dense / interaction operators behind keras Dense, MLP and SecondOrderFeatureInteraction, and the
DLRM forward/backward composition -- all arithmetic in liborx (orx_mlp_layer_*, orx_interact_*,
orx_gather_strided / orx_bag_gather, orx_pred_loss); this module only sequences launches and owns activations."""
from __future__ import annotations

import torch

from .. import native as N

GEMM_KERNEL_NAME = "k_gemm_tma (TMA-fed wgmma .tf32, 3xTF32, 128x128 tile, register accumulators)"


def _rows(B, n, device):
    """[B, n] activations whose row stride is a multiple of 4 floats: the TMA descriptors of the Dense-layer GEMMs need
    16-byte row strides (the 479-wide (dense_vec | interactions) block gets ld = 480); kernels take explicit strides."""
    ld = (n + 3) // 4 * 4
    t = torch.empty(B, ld, dtype=torch.float32, device=device)
    return t if ld == n else t[:, :n]


class GemmProfile:
    """bench.py's roofline hook: while active, every Dense-layer GEMM call (forward, and the dgrad + wgrad pair of a
    backward call) is bracketed by CUDA events on the launch stream; totals() -> (ms, flops, calls)."""
    active = None

    def __enter__(self):
        self.ev = []
        GemmProfile.active = self
        return self

    def __exit__(self, *a):
        GemmProfile.active = None

    def time(self, eng, flops, call):
        """Run call() between two events; the call is 'pure' when the engine's dispatch log shows exactly one
        k_gemm_tma launch without split-K."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        eng.debug_dispatch_log()                  # drop the records of earlier calls
        e0.record()
        call()
        e1.record()
        rec = eng.debug_dispatch_log()
        pure = len(rec) == 1 and rec[0].op == N.ORX_OP_GEMM and rec[0].variant == N.ORX_VARIANT_GEMM_TMA \
            and rec[0].s == 1
        self.ev.append((e0, e1, flops, pure))

    def totals(self, pure_only=False):
        """(ms, flops, calls) over all bracketed Dense-layer calls, or only over the calls that are ONE wgmma GEMM
        launch (forward layers on the tensor-core path: bias + activation are fused into the GEMM's epilogue)."""
        torch.cuda.synchronize()
        ev = [e for e in self.ev if e[3]] if pure_only else self.ev
        return (sum(a.elapsed_time(b) for a, b, _, _ in ev), float(sum(f for _, _, f, _ in ev)), len(ev))


def _mlp_fwd(eng, x, w, b, act, y):
    p = GemmProfile.active
    if p is None:
        return eng.mlp_fwd(x, w, b, act, y)
    p.time(eng, 2.0 * x.shape[0] * w.shape[0] * w.shape[1], lambda: eng.mlp_fwd(x, w, b, act, y))


def _mlp_bwd(eng, x, y, w, act, dy, dx, dw, db):
    p = GemmProfile.active
    if p is None:
        return eng.mlp_bwd(x, y, w, act, dy, dx, dw, db)
    p.time(eng, (4.0 if dx is not None else 2.0) * x.shape[0] * w.shape[0] * w.shape[1],
           lambda: eng.mlp_bwd(x, y, w, act, dy, dx, dw, db))

ACT = {None: 0, "linear": 0, "relu": 1, "sigmoid": 2}


def dense_forward(x, kernel, bias, activation):
    x = x.reshape(-1, x.shape[-1]).contiguous()
    y = torch.empty(x.shape[0], kernel.shape[1], dtype=torch.float32, device=x.device)
    N.engine().mlp_fwd(x, kernel, bias, ACT[activation], y)
    return y


def interaction_width(F, self_interaction):
    return F * (F + 1) // 2 if self_interaction else F * (F - 1) // 2


def interaction_forward(feats, self_interaction, mode):
    """feats [B,F,D] (last feature = the dense vector) -> [B, F(F-+1)/2]."""
    B, F, D = feats.shape
    out = torch.empty(B, interaction_width(F, self_interaction), dtype=torch.float32, device=feats.device)
    emb = feats[:, :F - 1, :].contiguous() if F > 1 else feats.new_empty(B, 0, D)
    N.engine().interact_fwd(emb, feats[:, F - 1, :].contiguous(), self_interaction, 0 if mode == "reference" else 1,
                            out)
    return out


class DLRMGraph:
    """Forward / backward of DLRM.inference + loss (recommenders/dlrm.py:63-100) on preallocated views:
    Z [B,T,D] embeddings, top_in [B, D+P] = (dense_vec | interactions) written in place by the last
    bottom layer and the interaction kernel.

    With ``cross`` (the DCN-v2 cross network in place of the dot interaction) the last bottom layer and the gathers
    write x0 [B, W] = (dense_vec | Z_0 | .. | Z_{T-1}) in place, W = (T + 1) D, and the top MLP reads x_L."""

    def __init__(self, tables, bot, top, m_spa, self_interaction, mode, loss_kind, clip, col_off=None, pooling=0,
                 cross=None):
        """col_off: the multi-hot bag layout (table k's bag = sparse columns col_off[k] .. col_off[k+1]), pooled by a
        sum (pooling 0) or a mean (1); None: one id per table, sparse [B, T].  cross: one list of projections per cross
        layer, each a (kernel [in, out], bias or None) pair, applied in order without activation: [(V, None), (U, b)]
        at low rank, [(K, b)] at full rank; None: the dot interaction."""
        self.tables, self.bot, self.top = tables, bot, top          # lists of tensors / (w, b, act) triples
        self.D, self.self_int, self.mode = m_spa, self_interaction, 0 if mode == "reference" else 1
        self.loss_kind, self.clip = loss_kind, clip
        self.col_off, self.pooling = col_off, pooling
        self.cross = cross

    def forward(self, dense, sparse, label=None, want_grad=False, Z=None):
        """Z: the embeddings [B, T, D] when the caller has gathered them already (the row-sharded step: rows fetched
        from their owners); the per-table gathers of ``sparse`` are then skipped."""
        eng = N.engine()
        dev = dense.device
        B, T, D = dense.shape[0], len(self.tables), self.D
        c = {"dense": dense, "sparse": sparse}
        if self.cross is not None:
            top_in = c["x0"] = _rows(B, (T + 1) * D, dev)            # (dense_vec | Z_0 | .. | Z_{T-1})
            if Z is not None:                                        # fetched rows: one strided copy into x0
                top_in[:, D:].copy_(Z.reshape(B, T * D))
            Z, gather = top_in[:, D:].unflatten(1, (T, D)), Z is None
        else:
            gather = Z is None
            if gather:
                Z = torch.empty(B, T, D, dtype=torch.float32, device=dev)
            top_in = c["top_in"] = _rows(B, D + interaction_width(T + 1, self.self_int), dev)
        if gather:
            if self.col_off is not None:                             # dlrm.py:83-85, one pooled bag per table
                eng.bag_gather(self.tables, sparse, self.col_off, self.pooling, top_in[:, D:] if self.cross is not None
                               else Z.view(B, T * D))
            else:
                for k, tab in enumerate(self.tables):                # dlrm.py:83-85
                    eng.gather_strided(tab, sparse, k, Z[:, k, :])
        c["Z"] = Z
        x, acts = dense, []
        for l, (w, b, act) in enumerate(self.bot):                   # dlrm.py:87
            last = l == len(self.bot) - 1
            if last and w.shape[1] != D:
                raise ValueError("the bottom MLP's last width must equal m_spa (tf.stack in the interaction)")
            y = top_in[:, :D] if last else torch.empty(B, w.shape[1], dtype=torch.float32, device=dev)
            _mlp_fwd(eng, x, w, b, act, y)
            acts.append(y)
            x = y
        c["bot_acts"] = acts
        if self.cross is not None:
            c["top_in"] = self._cross_forward(eng, c)
        else:
            eng.interact_fwd(Z, top_in[:, :D], self.self_int, self.mode, top_in[:, D:])      # dlrm.py:89-92
        x, acts = c["top_in"], []
        for w, b, act in self.top:
            y = torch.empty(B, w.shape[1], dtype=torch.float32, device=dev)
            _mlp_fwd(eng, x, w, b, act, y)
            acts.append(y)
            x = y
        c["top_acts"] = acts
        raw = x.reshape(-1)
        pred = c["pred"] = torch.empty(B, dtype=torch.float32, device=dev)
        out4 = c["out4"] = torch.zeros(4, dtype=torch.float32, device=dev)
        lab = label if label is not None else torch.zeros(B, dtype=torch.float32, device=dev)
        c["dpred"] = torch.empty(B, dtype=torch.float32, device=dev) if want_grad else None
        eng.pred_loss(raw, lab, self.loss_kind, self.clip, pred, c["dpred"], out4)       # dlrm.py:72-73,97-98
        return c

    def _cross_forward(self, eng, c):
        """x_{l+1} = x0 * (projections of x_l) + x_l for every cross layer; keeps x_l (c["xs"]) and each layer's
        projection outputs (c["cross_acts"][l], y_l last).  -> x_L."""
        x0 = c["x0"]
        B, W = x0.shape
        xs, cross_acts = [x0], []
        for projs in self.cross:
            h, outs = xs[-1], []
            for w, b in projs:
                y = _rows(B, w.shape[1], x0.device)
                _mlp_fwd(eng, h, w, b, 0, y)
                outs.append(y)
                h = y
            nxt = _rows(B, W, x0.device)
            eng.cross_fwd(x0, xs[-1], outs[-1], nxt)
            xs.append(nxt)
            cross_acts.append(outs)
        c["xs"], c["cross_acts"] = xs, cross_acts
        return xs[-1]

    def _cross_backward(self, eng, c, G):
        """G = dL/dx_L (overwritten).  -> (dL/dx0's dense columns [B, D], dZ [B, T, D], per layer [(dw, db)] in
        projection order)."""
        x0 = c["x0"]
        B, W = x0.shape
        D, dev = self.D, x0.device
        A, P, dy = _rows(B, W, dev), _rows(B, W, dev), _rows(B, W, dev)
        L = len(self.cross)
        cross_g = [None] * L
        for l in range(L - 1, -1, -1):
            projs, outs = self.cross[l], c["cross_acts"][l]
            eng.cross_bwd(N.ORX_CROSS_TOP if l == L - 1 else N.ORX_CROSS_MID, G, A, P=P, x0=x0, y=outs[-1], dy=dy)
            g, d = [None] * len(projs), dy
            for j in range(len(projs) - 1, -1, -1):
                w, b = projs[j]
                dx = P if j == 0 else _rows(B, w.shape[0], dev)
                dw = torch.empty_like(w)
                db = torch.empty_like(b) if b is not None else None
                _mlp_bwd(eng, c["xs"][l] if j == 0 else outs[j - 1], outs[j], w, 0, d, dx, dw, db)
                g[j] = (dw, db)
                d = dx
            cross_g[l] = g
        d_dense = _rows(B, D, dev)
        dZ = torch.empty(B, W // D - 1, D, dtype=torch.float32, device=dev)
        eng.cross_bwd(N.ORX_CROSS_FINAL, G, A, P=P, dx_lo=d_dense, dx_hi=dZ.view(B, W - D))
        return d_dense, dZ, cross_g

    def backward(self, c):
        """-> (dZ [B,T,D], bottom [(dw, db)], top [(dw, db)], cross [[(dw, db)] per projection] per layer, [] without
        the cross network)."""
        eng = N.engine()
        dense, top_in, Z = c["dense"], c["top_in"], c["Z"]
        B, D = dense.shape[0], self.D
        dev = dense.device
        dy = c["dpred"].reshape(B, 1)
        d_top_in = _rows(B, top_in.shape[1], dev)
        top_g = [None] * len(self.top)
        for l in range(len(self.top) - 1, -1, -1):
            w, b, act = self.top[l]
            x = top_in if l == 0 else c["top_acts"][l - 1]
            dx = d_top_in if l == 0 else torch.empty(B, w.shape[0], dtype=torch.float32, device=dev)
            dw = torch.empty_like(w)
            db = torch.empty_like(b) if b is not None else None
            _mlp_bwd(eng, x, c["top_acts"][l], w, act, dy, dx, dw, db)
            top_g[l] = (dw, db)
            dy = dx
        if self.cross is not None:
            dy, dZ, cross_g = self._cross_backward(eng, c, d_top_in)
        else:
            dZ, cross_g = torch.empty_like(Z), []
            eng.interact_bwd(Z, top_in[:, :D], d_top_in[:, D:], self.self_int, self.mode, dZ, d_top_in[:, :D])
            dy = d_top_in[:, :D]
        bot_g = [None] * len(self.bot)
        for l in range(len(self.bot) - 1, -1, -1):
            w, b, act = self.bot[l]
            x = dense if l == 0 else c["bot_acts"][l - 1]
            dx = None if l == 0 else torch.empty(B, w.shape[0], dtype=torch.float32, device=dev)
            dw = torch.empty_like(w)
            db = torch.empty_like(b) if b is not None else None
            _mlp_bwd(eng, x, c["bot_acts"][l], w, act, dy, dx, dw, db)
            bot_g[l] = (dw, db)
            dy = dx
        return dZ, bot_g, top_g, cross_g
