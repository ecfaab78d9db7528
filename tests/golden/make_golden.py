"""Generate tests/golden/*.npz by running the REFERENCE's own Python code.

Needs a checkout of the reference (ylongqi/openrec); the fixtures it writes are committed, so the tests do not:

    OPENREC_REFERENCE=/path/to/openrec python tests/golden/make_golden.py

The reference's openrec/tf2/{modules,recommenders,metrics,data} files are imported verbatim
from that checkout; ``tensorflow`` is replaced by the torch stand-in of tf_standin.py
(TensorFlow itself is not installable here -- "parity unpinned" for TF internals, see
oracle/__init__.py).  Forward values and autograd gradients are recorded in float64; the
fixtures are the pin for oracle/openrec_oracle.py and, through it, for the CUDA kernels.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_standin  # noqa: E402

REF = os.environ.get("OPENREC_REFERENCE", "")


def _fresh_reference():
    for k in [k for k in sys.modules if k == "openrec" or k.startswith("openrec.")]:
        del sys.modules[k]
    if not os.path.isdir(os.path.join(REF, "openrec")):
        raise SystemExit("set OPENREC_REFERENCE to a checkout of ylongqi/openrec")
    tf = tf_standin.install()
    if REF not in sys.path:
        sys.path.insert(0, REF)
    return tf


def _np(x):
    return x.detach().numpy().copy()


def _grads(target, variables):
    gs = torch.autograd.grad(target, [v.t for v in variables], allow_unused=True)
    return [np.zeros(tuple(v.t.shape)) if g is None else _np(g) for g, v in zip(gs, variables)]


def make_pairwise(rng):
    _fresh_reference()
    from openrec.tf2.recommenders import BPR, UCML
    U, I, D, B = 37, 53, 12, 96
    uid = rng.integers(0, U, B).astype(np.int32)
    pid = rng.integers(0, I, B).astype(np.int32)
    nid = rng.integers(0, I, B).astype(np.int32)
    nid[:4] = pid[:4]  # same item as pos and neg in one triplet
    for name, cls, kw in (("bpr", BPR, {}), ("ucml", UCML, {"margin": 0.5})):
        torch.manual_seed(7)
        m = cls(dim_user_embed=D, dim_item_embed=D, total_users=U, total_items=I, **kw)
        if name == "ucml":  # make some hinges inactive: spread the embeddings out
            with torch.no_grad():
                for lf in (m.user_latent_factor, m.item_latent_factor):
                    lf.embeddings.t.mul_(8.0)
        out = dict(uid=uid, pid=pid, nid=nid,
                   user=_np(m.user_latent_factor.embeddings.t), item=_np(m.item_latent_factor.embeddings.t),
                   bias=_np(m.item_bias.embeddings.t))
        loss, l2 = m(torch.tensor(uid), torch.tensor(pid), torch.tensor(nid))
        tv = m.trainable_variables  # creation order: user, item, bias
        g = _grads(loss + l2, tv)
        out.update(loss=_np(loss), l2=_np(l2), g_user=g[0], g_item=g[1], g_bias=g[2])
        out["inference"] = _np(m.inference(torch.tensor(uid[:5])))
        if name == "ucml":
            m.censor_vec(torch.tensor(uid), torch.tensor(pid), torch.tensor(nid))
            out["user_censored"] = _np(m.user_latent_factor.embeddings.t)
            out["item_censored"] = _np(m.item_latent_factor.embeddings.t)
        np.savez(os.path.join(HERE, f"pairwise_{name}.npz"), **out)


def make_pointwise(rng):
    _fresh_reference()
    from openrec.tf2.recommenders import GMF, WRMF
    U, I, D, B = 29, 41, 10, 80
    uid = rng.integers(0, U, B).astype(np.int32)
    iid = rng.integers(0, I, B).astype(np.int32)
    label = (rng.random(B) < 0.4).astype(np.float32)
    for name, cls, kw in (("gmf", GMF, {}), ("wrmf", WRMF, {"a": 3.0, "b": 0.5})):
        torch.manual_seed(11)
        m = cls(dim_user_embed=D, dim_item_embed=D, total_users=U, total_items=I, **kw)
        lab = torch.tensor(label, dtype=torch.float64)
        loss, l2 = m(torch.tensor(uid), torch.tensor(iid), lab)
        tv = m.trainable_variables
        g = _grads(loss + l2, tv)
        out = dict(uid=uid, iid=iid, label=label,
                   user=_np(m.user_latent_factor.embeddings.t), item=_np(m.item_latent_factor.embeddings.t),
                   bias=_np(m.item_bias.embeddings.t), loss=_np(loss), l2=_np(l2),
                   g_user=g[0], g_item=g[1], g_bias=g[2], a=kw.get("a", 1.0), b=kw.get("b", 1.0))
        if name == "gmf":
            out["w"] = _np(m.mlp.layers[0].kernel.t)
            out["g_w"] = g[3]
        out["inference"] = _np(m.inference(torch.tensor(uid[:5])))
        np.savez(os.path.join(HERE, f"pointwise_{name}.npz"), **out)


def make_interaction(rng):
    _fresh_reference()
    from openrec.tf2.modules import SecondOrderFeatureInteraction
    B, F, D = 6, 5, 7
    feats = [torch.tensor(rng.standard_normal((B, D))) for _ in range(F)]
    out = {f"in{k}": _np(f) for k, f in enumerate(feats)}
    for si in (False, True):
        out[f"out_self{int(si)}"] = _np(SecondOrderFeatureInteraction(self_interaction=si)(feats))
    np.savez(os.path.join(HERE, "interaction.npz"), **out)


def make_dlrm(rng):
    _fresh_reference()
    from openrec.tf2.recommenders import DLRM
    B, m_spa = 48, 4
    ln_emb, ln_bot, ln_top = [11, 7, 13], [8, 4], [16, 8, 1]
    dense = np.log1p(rng.integers(0, 100, (B, 5))).astype(np.float64)
    sparse = np.stack([rng.integers(0, n, B) for n in ln_emb], axis=1).astype(np.int32)
    label = (rng.random(B) < 0.3).astype(np.float32)
    for tag, kw in (("mse", {}), ("bce_self", dict(loss_func="bce", arch_interaction_itself=True)),
                    ("clip", dict(loss_threshold=0.45)), ("bce", dict(loss_func="bce"))):
        torch.manual_seed(3)
        m = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=ln_bot, ln_top=ln_top, **kw)
        loss = m(torch.tensor(dense), torch.tensor(sparse), torch.tensor(label, dtype=torch.float64))
        pred = m.inference(torch.tensor(dense), torch.tensor(sparse))
        tv = m.trainable_variables
        g = _grads(loss, tv)
        out = dict(dense=dense, sparse=sparse, label=label, loss=_np(loss), pred=_np(pred), n_vars=len(tv))
        for k, (v, gv) in enumerate(zip(tv, g)):
            out[f"var{k}"] = _np(v.t)
            out[f"grad{k}"] = gv
        np.savez(os.path.join(HERE, f"dlrm_{tag}.npz"), **out)


def make_metrics(rng):
    tf_standin.DTYPE[0] = torch.float32
    try:
        _fresh_reference()
        from openrec.tf2.metrics import AUC, NDCG, Recall
        R, I = 7, 60
        pred = rng.standard_normal((R, I)).astype(np.float32)
        pred[:, 5] = pred[:, 6]  # ties
        pos = rng.random((R, I)) < 0.12
        pos[:, 0] = True
        excl = (rng.random((R, I)) < 0.2) & ~pos
        a = [torch.tensor(pos), torch.tensor(pred), torch.tensor(excl)]
        np.savez(os.path.join(HERE, "metrics.npz"), pos=pos, pred=pred, excl=excl,
                 auc=_np(AUC(*a)), ndcg=_np(NDCG(*a, at=[5, 20])), recall=_np(Recall(*a, at=[5, 20])))
    finally:
        tf_standin.DTYPE[0] = torch.float64


def make_sampler(rng):
    _fresh_reference()
    from openrec.tf2.data import dataset as ref_ds
    from openrec.tf2.data.utils import _DataStore
    U, I, N = 23, 57, 300
    pairs = set()
    while len(pairs) < N:
        pairs.add((int(rng.integers(0, U)), int(rng.integers(0, I))))
    raw = np.array(sorted(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
    raw = raw[rng.permutation(N)]
    out = dict(raw_user=raw["user_id"], raw_item=raw["item_id"], U=U, I=I)

    def take(gen, n):
        rows = []
        for _ in range(n):
            d = next(gen)
            rows.append([float(d[k]) for k in sorted(d)])
        return np.array(rows)

    ds = _DataStore(raw_data=raw, total_users=U, total_items=I, seed=123)
    out["pairwise"] = take(ref_ds._pairwise_generator(ds), 700)  # keys sorted: n_item_id,p_item_id,user_id
    ds = _DataStore(raw_data=raw, total_users=U, total_items=I, seed=5)
    out["stratified"] = take(ref_ds._stratified_pointwise_generator(ds, 0.3), 500)  # item_id,label,user_id
    ds = _DataStore(raw_data=raw, total_users=U, total_items=I, seed=9)
    out["per_pos"] = take(ref_ds._per_pos_stratified_pointwise_generator(ds, 0.2), 500)
    # evaluation generator: val split excluded by a train split
    tr = _DataStore(raw_data=raw[:200], total_users=U, total_items=I, seed=1)
    va = _DataStore(raw_data=raw[200:], total_users=U, total_items=I, seed=1)

    class _D:  # the generator reads excl_d.datastore
        def __init__(self, s):
            self.datastore = s
    ev = list(ref_ds._evaluation_generator(va, [_D(tr)]))
    out["eval_user"] = np.array([e["user_id"] for e in ev], dtype=np.int32)
    out["eval_pos"] = np.stack([e["pos_mask"] for e in ev])
    out["eval_excl"] = np.stack([e["excl_mask"] for e in ev])
    np.savez(os.path.join(HERE, "sampler.npz"), **out)


if __name__ == "__main__":
    rng = np.random.default_rng(20260923)
    random.seed(0)
    make_pairwise(rng)
    make_pointwise(rng)
    make_interaction(rng)
    make_dlrm(rng)
    make_metrics(rng)
    make_sampler(rng)
    print("golden fixtures written to", HERE)
