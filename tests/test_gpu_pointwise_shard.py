"""GPU: the row-sharded GMF / WRMF.  The four new kernels (orx_pointwise_shard_lookups, orx_pointwise_serve,
orx_pointwise_grad_rows, orx_rows_scale) against numpy and their refusals; the sharded step with R virtual ranks on one
device (LoopbackExchange: every rank its own liborx handle, the multi-GPU code and kernels) against the single-GPU
orx_pointwise_step on the global batch; sharded evaluation and retrieval of both models (GMF with its w scale) against
orx_score_rank / orx_score_topk on the gathered tables; ShardedGMF / ShardedWRMF in a one-rank NCCL group against GMF /
WRMF, with a checkpoint round trip and RankingEvaluator / Retriever; and a worker-process job on >= 2 GPUs."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]

from _ranks import run_ranks  # noqa: E402
from pointwise_shard_np import grad_rows_np, serve_np, shard_lookups_np  # noqa: E402

GMF, WRMF = 0, 1


@pytest.fixture(scope="module")
def eng():
    from openrec_b200 import native
    return native.engine()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def records(eng):
    from openrec_b200 import native as N
    return [r for r in eng.debug_dispatch_log() if r.op == N.ORX_OP_POINTWISE_GRAD_ROWS]


# ---- kernels ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_shard_lookups(eng, R):
    rng = np.random.default_rng(R)
    U, I = 13, 9
    Lu = (U + R - 1) // R
    uid = rng.choice(np.array([-1, -5, 2 ** 31 - 1] + list(range(U, R * Lu + 1)) + list(range(U)) * 3), 1000)
    iid = rng.choice(np.array([-1, I, I + 1] + list(range(I)) * 4), 1000)
    got = eng.pointwise_shard_lookups(dev(uid, torch.int32), dev(iid, torch.int32), U, I).cpu().numpy()
    np.testing.assert_array_equal(got, shard_lookups_np(uid, iid, U, I))
    assert (got[(uid >= U) & (uid < R * Lu)] == -1).all()
    assert eng.pointwise_shard_lookups(dev(np.zeros(0), torch.int32), dev(np.zeros(0), torch.int32), U, I).shape == (0, 2)


@pytest.mark.parametrize("D,ld", [(4, 8), (50, 54), (128, 132), (3, 5)])
def test_serve(eng, D, ld):
    rng = np.random.default_rng(D)
    lu, li, Lu = 7, 5, 9                           # local rows 7, 8 are past the user shard: no table
    user, item, bias = rng.random((lu, D)).astype(np.float32), rng.random((li, D)).astype(np.float32), \
        rng.random((li, 1)).astype(np.float32)
    req = rng.integers(-2, Lu + li + 2, 300).astype(np.int32)
    rows, ul, il = eng.pointwise_serve(dev(user), dev(item), dev(bias), lu, li, Lu, dev(req, torch.int32), ld)
    want = serve_np(user, item, bias, lu, li, Lu, req, ld)
    np.testing.assert_array_equal(rows.cpu().numpy(), want[0])
    np.testing.assert_array_equal(ul.cpu().numpy(), want[1])
    np.testing.assert_array_equal(il.cpu().numpy(), want[2])


@pytest.mark.parametrize("D", [4, 50, 64, 128, 256, 32])
@pytest.mark.parametrize("case", ["gmf", "wrmf", "wrmf_sigmoid"])
def test_grad_rows(eng, D, case):
    """Against the oracle's closed forms (float64) on fetched rows with repeats and skipped samples; the dispatch record
    names the path; repeated calls give the same bits (the kernel has no atomics)."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(D * 7 + len(case))
    kind = GMF if case == "gmf" else WRMF
    B, n_rows, ld = 777, 300, D + 4
    rows = np.zeros((n_rows, ld), np.float32)
    rows[:, :D + 1] = rng.uniform(-0.5, 0.5, (n_rows, D + 1))
    slot = rng.integers(0, n_rows, (B, 2)).astype(np.int32)
    slot[rng.random(B) < 0.1] = -1
    label = (rng.random(B) < 0.4).astype(np.float32)
    w = rng.uniform(-1, 1, D).astype(np.float32) if kind == GMF else None
    a, b, sig = (1.0, 1.0, False) if kind == GMF else (2.0, 0.3, case == "wrmf_sigmoid")
    inv_B = 1.0 / (3 * B)
    eng.debug_dispatch_log()
    outs = []
    for add_w in (True, True, False):
        outs.append(eng.pointwise_grad_rows(kind, dev(rows), D, dev(slot, torch.int32), dev(label),
                                            None if w is None else dev(w), inv_B, a, b, sig, 1.3, 0.7, add_w))
    rec = records(eng)
    want_variant = N.ORX_VARIANT_STEP if D in (32, 64, 128, 256) else N.ORX_VARIANT_STEP_GENERIC
    assert [(r.variant, r.ta, r.m, r.n, r.k) for r in rec] == [(want_variant, kind, B, D, ld)] * 3, rec
    for x, y in zip(outs[0], outs[1]):
        if x is not None:
            assert torch.equal(x, y)
    for add_w, (d_rows, gw, out2) in zip((True, False), outs[1:]):
        wd, wgw, (wl, wq) = grad_rows_np(kind, rows, D, slot, label, w, inv_B, a, b, sig, 1.3, 0.7, add_w)
        np.testing.assert_allclose(d_rows.cpu().numpy(), wd, rtol=2e-5, atol=1e-6)
        np.testing.assert_allclose(out2.cpu().numpy(), [wl, wq], rtol=2e-5, atol=1e-6)
        if kind == GMF:
            np.testing.assert_allclose(gw.cpu().numpy(), wgw, rtol=1e-4, atol=1e-6)
        else:
            assert gw is None


def test_rows_scale(eng):
    rng = np.random.default_rng(0)
    for rows, D in ((1, 1), (37, 50), (1000, 128)):
        x = rng.standard_normal((rows, D)).astype(np.float32)
        s = rng.standard_normal(D).astype(np.float32)
        t = dev(x)
        eng.rows_scale(t, dev(s))
        np.testing.assert_array_equal(t.cpu().numpy().view(np.int32), (x * s[None]).view(np.int32))
        xi = dev(x).view(torch.int32)                            # the xrows exchange buffer: float bits in int32
        eng.rows_scale(xi, dev(s))
        np.testing.assert_array_equal(xi.cpu().numpy(), (x * s[None]).view(np.int32))


def test_refusals(eng):
    """Every new entry point refuses bad arguments with ORX_ERR_INVALID, before any device work."""
    lib, h, s = eng.lib, eng.h, eng.stream()
    t = torch.zeros(64, dtype=torch.float32, device="cuda")
    i = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    bad = [
        lib.orx_pointwise_shard_lookups(h, p(i), p(i), -1, 5, 5, p(i), s),
        lib.orx_pointwise_shard_lookups(h, p(i), p(i), 4, 2 ** 31, 5, p(i), s),
        lib.orx_pointwise_shard_lookups(h, None, p(i), 4, 5, 5, p(i), s),
        lib.orx_pointwise_serve(h, p(t), p(t), p(t), 4, 2, 2, 2, p(i), 4, 4, p(t), p(i), p(i), s),      # ld <= dim
        lib.orx_pointwise_serve(h, p(t), p(t), p(t), 4, 3, 2, 2, p(i), 4, 8, p(t), p(i), p(i), s),      # Lu < users
        lib.orx_pointwise_serve(h, p(t), p(t), p(t), 0, 2, 2, 2, p(i), 4, 8, p(t), p(i), p(i), s),
        lib.orx_pointwise_serve(h, p(t), p(t), p(t), 4, 2, 2, 2, None, 4, 8, p(t), p(i), p(i), s),
        lib.orx_pointwise_grad_rows(h, 2, p(t), 8, 4, p(i), p(t), p(t), 4, 1, 1, 0, 1, 1, 0.25, 0, p(t), p(t), p(t), s),
        lib.orx_pointwise_grad_rows(h, 0, p(t), 8, 4, p(i), p(t), p(t), 0, 1, 1, 0, 1, 1, 0.25, 0, p(t), p(t), p(t), s),
        lib.orx_pointwise_grad_rows(h, 0, p(t), 4, 4, p(i), p(t), p(t), 4, 1, 1, 0, 1, 1, 0.25, 0, p(t), p(t), p(t), s),
        lib.orx_pointwise_grad_rows(h, 0, p(t), 2000, 1025, p(i), p(t), p(t), 4, 1, 1, 0, 1, 1, 0.25, 0, p(t), p(t),
                                    p(t), s),
        lib.orx_pointwise_grad_rows(h, 0, p(t), 8, 4, p(i), p(t), None, 4, 1, 1, 0, 1, 1, 0.25, 0, p(t), p(t), p(t), s),
        lib.orx_pointwise_grad_rows(h, 1, p(t), 8, 4, p(i), p(t), None, 4, 1, 1, 0, 1, 1, 1, 0, p(t), None, None, s),
        lib.orx_pointwise_grad_rows(h, 1, p(t), 8, 4, C.c_void_p(i.data_ptr() + 4), p(t), None, 4, 1, 1, 0, 1, 1, 1, 0,
                                    p(t), None, p(t), s),
        lib.orx_rows_scale(h, p(t), -1, 4, p(t), s),
        lib.orx_rows_scale(h, p(t), 4, 0, p(t), s),
        lib.orx_rows_scale(h, None, 4, 4, p(t), s),
    ]
    assert bad == [-1] * len(bad), bad
    assert lib.orx_rows_scale(h, None, 0, 4, None, s) == 0
    assert lib.orx_pointwise_serve(h, None, None, None, 4, 0, 0, 0, None, 0, 8, None, None, None, s) == 0


def test_sparse_apply_skips_negative_ids(eng):
    """The owner apply passes -1 for requests of the other table: orx_sparse_apply_strided must skip them, also in its
    index build (no staged row, no dedup slot), so the result equals the apply of the valid ids alone."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(1)
    for kind in (N.ORX_OPT_ADAGRAD, N.ORX_OPT_ADAM_LAZY, N.ORX_OPT_ADAM_DENSE):
        tab0 = rng.standard_normal((20, 8)).astype(np.float32)
        ids = rng.integers(-1, 20, 200).astype(np.int32)
        ids[rng.random(200) < 0.5] = -1
        vals = rng.standard_normal((200, 12)).astype(np.float32)
        res = []
        for keep in (np.ones(200, bool), ids >= 0):
            var = dev(tab0)
            s0 = torch.full_like(var, 0.1 if kind == N.ORX_OPT_ADAGRAD else 0.0)
            s1 = torch.zeros_like(var)
            eng.sparse_apply_rows(N.table(var, s0, s1), dev(ids[keep], torch.int32), dev(vals[keep])[:, 2:10],
                                  N.opt(kind, 0.05, step=2))
            res.append((var, s0, s1))
        for x, y in zip(*res):
            torch.testing.assert_close(x, y, rtol=1e-6, atol=1e-7)


# ---- loopback step against the single-GPU step ------------------------------------------------------------------------
def _batches(rng, ids, U, I, n):
    if ids == "zipf":
        u, i = np.minimum(rng.zipf(1.3, n) - 1, U - 1), np.minimum(rng.zipf(1.2, n) - 1, I - 1)
    else:
        u, i = rng.integers(0, U, n), rng.integers(0, I, n)
    if ids == "bad":
        m = rng.random(n) < 0.15
        u[m] = rng.choice(np.array([-1, U, U + 1, 2 ** 31 - 1]), m.sum())
        m = rng.random(n) < 0.1
        i[m] = rng.choice(np.array([-3, I, I + 5]), m.sum())
    return u.astype(np.int32), i.astype(np.int32), (rng.random(n) < 0.3).astype(np.float32)


_STEP_CASES = [
    # (R, model, opt, ids, U, I, D, c_loss, c_l2)
    (1, "gmf", "adagrad", "uniform", 500, 700, 64, 1.0, 1.0),
    (2, "gmf", "sgd", "zipf", 500, 700, 128, 1.0, 1.0),
    (3, "gmf", "lazyadam", "bad", 500, 700, 50, 1.0, 1.0),
    (8, "gmf", "adam", "uniform", 500, 700, 128, 2.0, 0.5),
    (8, "gmf", "adagrad", "bad", 5, 3, 32, 0.5, 2.0),            # tables smaller than R: ranks without rows
    (2, "wrmf", "adagrad", "uniform", 500, 700, 128, 1.0, 1.0),
    (3, "wrmf_sigmoid", "adam", "zipf", 500, 700, 64, 1.0, 0.25),
    (8, "wrmf", "lazyadam", "bad", 500, 700, 256, 1.5, 1.0),
    (1, "wrmf_sigmoid", "sgd", "bad", 6, 4, 4, 1.0, 1.0),
    (8, "wrmf", "sgd", "zipf", 3, 7, 64, 1.0, 1.0),
]


@pytest.mark.parametrize("case", _STEP_CASES, ids=lambda c: "-".join(map(str, c[:4])))
def test_loopback_step_equals_single_gpu(case):
    from openrec_b200 import native as N
    from openrec_b200.sharded import LoopbackExchange, PointwiseShard, pointwise_step_sharded
    from openrec_b200.tf2.recommenders._base import w_table
    R, model, opt_name, ids, U, I, D, c_loss, c_l2 = case
    kind = GMF if model == "gmf" else WRMF
    a, b, sig = (1.0, 1.0, False) if kind == GMF else (1.0, 0.1, model == "wrmf_sigmoid")
    okind = {"sgd": N.ORX_OPT_SGD, "adagrad": N.ORX_OPT_ADAGRAD, "lazyadam": N.ORX_OPT_ADAM_LAZY,
             "adam": N.ORX_OPT_ADAM_DENSE}[opt_name]
    # SGD's step grows with a row's lookup count (l2 counts every lookup), so its rate keeps lr * lookups < 1 on the hot
    # rows of Zipf batches; otherwise the rows diverge and any summation-order difference is amplified past 1e-5
    lr = {"sgd": 0.001, "adagrad": 0.05, "lazyadam": 0.01, "adam": 0.01}[opt_name]
    fill = 0.1 if okind == N.ORX_OPT_ADAGRAD else 0.0
    rng = np.random.default_rng(R * 31 + D)
    glob = [rng.uniform(-0.5, 0.5, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1))]
    w0 = rng.uniform(-1, 1, (D, 1)).astype(np.float32)
    # single GPU
    tabs = [dev(t) for t in glob]
    slots = [(torch.full_like(t, fill), torch.full_like(t, fill)) for t in tabs]
    w = dev(w0)
    ws = (torch.full_like(w, fill), torch.full_like(w, fill))
    eng1 = N.engine()
    # virtual ranks
    engs = [N.Engine(0) for _ in range(R)]
    parts = []
    for r in range(R):
        sh = []
        for t in glob:
            rows = t[r::R]
            x = torch.zeros(max(len(rows), 1), t.shape[1], dtype=torch.float32, device="cuda")
            x[:len(rows)] = dev(rows)
            sh.append(x)
        sl = [(torch.full_like(x, fill), torch.full_like(x, fill)) for x in sh]
        wr = dev(w0) if kind == GMF else None
        wsl = (torch.full_like(wr, fill), torch.full_like(wr, fill)) if kind == GMF else (None, None)
        parts.append(PointwiseShard(engs[r], r, R, U, I, D, kind, *sh, sl, w=wr, w_slots=wsl, a=a, b=b,
                                    use_sigmoid=sig))
    B = 512 if min(U, I) >= R else 16      # tables smaller than R: a few dozen lookups per row, as on the large tables
    # Both Adams divide m by sqrt(v): an element whose summed gradient nearly cancels (a hot row's many terms) moves by up
    # to lr whatever its size, so the summation-order noise between the fused step's staging adds and the segment sum
    # reaches 1e-5 there (one element in 128 000 measured at 6.4e-5 with LazyAdam).  SGD and Adagrad stay within 1e-5.
    # Such an element's value then enters the next step's gradient (c_l2 * u), so its m and v follow it: the slots of the
    # Adams are held to 1e-3 (measured: 1.2e-4 on that element's m).
    adam = okind in (N.ORX_OPT_ADAM_DENSE, N.ORX_OPT_ADAM_LAZY)
    atol = 1e-4 if adam else 1e-5
    atol_slots = 1e-3 if adam else 1e-5
    for step in range(1, 4):
        uid, iid, lab = _batches(rng, ids, U, I, R * B)
        o = N.opt(okind, lr, step=step)
        out4 = torch.zeros(4, device="cuda")
        eng1.pointwise_step(kind, *[N.table(t, *s) for t, s in zip(tabs, slots)],
                            w_table(w, *ws) if kind == GMF else None, dev(uid, torch.int32), dev(iid, torch.int32),
                            dev(lab), o, out4, a, b, sig, c_loss, c_l2)
        batches = [(dev(uid[r * B:(r + 1) * B], torch.int32), dev(iid[r * B:(r + 1) * B], torch.int32),
                    dev(lab[r * B:(r + 1) * B])) for r in range(R)]
        outs = pointwise_step_sharded(parts, LoopbackExchange, batches, (okind, lr, 1e-7, 0.9, 0.999, step), c_loss,
                                      c_l2)
        for x in outs:
            assert torch.equal(x, outs[0])
        torch.testing.assert_close(outs[0].cpu(), out4[:2].cpu(), rtol=1e-5, atol=1e-5)
    for k, (t, (s0, s1)) in enumerate(zip(tabs, slots)):
        full = [torch.zeros_like(x) for x in (t, s0, s1)]
        for r, p in enumerate(parts):
            n = len(range(r, t.shape[0], R))
            mine = (p.user, p.item, p.bias)[k]
            msl = (p.user_slots, p.item_slots, p.bias_slots)[k]
            for f, x in zip(full, (mine, *msl)):
                f[r::R] = x[:n]
        for name, f, x in zip(("table", "s0", "s1"), full, (t, s0, s1)):
            what = f"{('user', 'item', 'bias')[k]} {name}"
            tol = atol if name == "table" else atol_slots
            torch.testing.assert_close(f, x, rtol=tol, atol=tol, msg=lambda m, what=what: f"{what}: {m}")
    if kind == GMF:
        for p in parts:
            assert torch.equal(p.w, parts[0].w)
            torch.testing.assert_close(p.w, w, rtol=atol, atol=atol)
            for x, y in zip(p.w_slots, ws):
                torch.testing.assert_close(x, y, rtol=atol_slots, atol=atol_slots)
    for e in engs:
        e.close()


# ---- evaluation and retrieval -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("model", ["gmf", "wrmf"])
def test_loopback_eval_and_topk(eng, R, model):
    from openrec_b200 import native as N
    from openrec_b200.sharded import loopback_sum, score_rank_sharded, score_topk_sharded
    from test_gpu_score_rank import check_equal, make_problem
    rng = np.random.default_rng(R * 5 + len(model))
    pb = make_problem(rng, N.ORX_SCORE_DOT, 300, 2000, 64, scaled=model == "gmf")
    at = (10, 50)
    uid = dev(pb.uid, torch.int32)
    engs = [N.Engine(0) for _ in range(R)]
    parts = []
    for r in range(R):
        g = N.rowshard(R, r, pb.U, pb.I)
        pad = lambda t: t[r::R] if len(t[r::R]) else torch.zeros((1,) + tuple(t.shape[1:]), device="cuda")  # noqa
        parts.append((engs[r], N.ORX_SCORE_DOT, pad(pb.user).contiguous(), pad(pb.item).contiguous(),
                      pad(pb.bias).contiguous(), g))
    scale = [None if pb.scale is None else pb.scale.clone() for _ in range(R)]
    got = score_rank_sharded(parts, loopback_sum, uid, pb.pos_off, pb.pos_items, pb.excl_off, pb.excl_items,
                             pb.max_pos(), at=at, scale=scale)
    want = eng.score_rank(N.ORX_SCORE_DOT, pb.user, uid, pb.item, pb.bias, pb.pos_off, pb.pos_items, pb.excl_off,
                          pb.excl_items, pb.max_pos(), at=at, scale=pb.scale)
    for g_ in got:
        check_equal(g_, want, f"R={R} {model}")
    for k in (1, 37):
        top = score_topk_sharded(parts, loopback_sum, uid, pb.excl_off, pb.excl_items, k, scale=scale)
        wi, ws = eng.score_topk(N.ORX_SCORE_DOT, pb.user, uid, pb.item, pb.bias, pb.excl_off, pb.excl_items, k,
                                scale=pb.scale)
        for it, sc in top:
            assert torch.equal(it, wi)
            np.testing.assert_array_equal(sc.cpu().numpy().view(np.int32) & 0x7fffffff,
                                          ws.cpu().numpy().view(np.int32) & 0x7fffffff)   # -0.0 may read +0.0
    for e in engs:
        e.close()


# ---- class surface ----------------------------------------------------------------------------------------------------
_CLASS = r"""
import os, sys, tempfile
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(0)
dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
import tensorflow as tf
from openrec.tf2.metrics import RankingEvaluator
from openrec.tf2.recommenders import GMF, WRMF, Retriever, ShardedGMF, ShardedWRMF
from openrec_b200.tf2 import checkpoint
from _score_rank_shard_worker import datasets
from test_gpu_score_rank import check_equal
U, I, D = 300, 2000, 64
rng = np.random.default_rng(0)
train, val = datasets(rng, U, I)
for name, mk, ref_cls, opt_cls in (("gmf", lambda s: ShardedGMF(D, D, U, I, seed=s), GMF, tf.keras.optimizers.Adagrad),
                                   ("wrmf", lambda s: ShardedWRMF(D, D, U, I, a=1.0, b=0.1, seed=s),
                                    lambda *a: WRMF(*a, a=1.0, b=0.1), tf.keras.optimizers.Adam)):
    models = [mk(3), ref_cls(D, D, U, I)]
    for a_, b_ in zip(models[1].trainable_variables, models[0].trainable_variables):
        a_.t.copy_(b_.t)
    data = [(rng.integers(0, U, 256).astype(np.int32), rng.integers(0, I, 256).astype(np.int32),
             (rng.random(256) < 0.3).astype(np.float32)) for _ in range(3)]
    losses, opts = [], []
    for model in models:
        optimizer = opt_cls(learning_rate=0.01)

        @tf.function
        def train_step(u, i, l):
            with tf.GradientTape() as tape:
                loss, l2 = model(u, i, l)
            gradients = tape.gradient((loss, l2), model.trainable_variables)
            optimizer.apply_gradients(zip(gradients, model.trainable_variables))
            return loss, l2

        losses.append([[float(x.numpy()) for x in train_step(*b)] for b in data])
        opts.append(optimizer)
    np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5, atol=1e-6)
    tol = 1e-4 if name == "wrmf" else 1e-5
    for a_, b_ in zip(models[0].trainable_variables, models[1].trainable_variables):
        torch.testing.assert_close(a_.t, b_.t, atol=tol, rtol=tol)
        for x, y in zip(opts[0].slots(a_), opts[1].slots(b_)):
            if x is not None:
                torch.testing.assert_close(x, y, atol=tol, rtol=tol)
    # evaluation and retrieval on the sharded model equal those of the single-device model holding its tables
    for a_, b_ in zip(models[0].trainable_variables, models[1].trainable_variables):
        b_.t.copy_(a_.t)
    at = [10, 50]
    res = [RankingEvaluator(val, excl_datasets=[train], at=at, batch_size=100).evaluate(m) for m in models]
    check_equal(*[[torch.from_numpy(r[k].numpy()) for k in ("AUC", "NDCG", "Recall")] for r in res], name)
    users = np.arange(-1, U + 1)
    top = [Retriever(excl_datasets=[train], k=20, batch_size=128).recommend(m, users) for m in models]
    assert torch.equal(top[0][0].t, top[1][0].t)
    assert np.array_equal(top[0][1].numpy().view(np.int32) & 0x7fffffff, top[1][1].numpy().view(np.int32) & 0x7fffffff)
    # checkpoint round trip: shards, slots and the w replica
    path = os.path.join(tempfile.mkdtemp(), "rank0.npz")
    checkpoint.save(path, models[0], opts[0])
    fresh, opt1 = mk(9), opt_cls(learning_rate=0.01)
    checkpoint.load(path, fresh, opt1)
    assert opt1.iterations == 3
    for a_, b_ in zip(models[0].trainable_variables, fresh.trainable_variables):
        assert torch.equal(a_.t, b_.t)
        for x, y in zip(opts[0].slots(a_), opt1.slots(b_)):
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y))
dist.destroy_process_group()
print("class ok")
"""


def test_sharded_pointwise_classes_one_rank():
    [(rc, out)] = run_ranks(1, _CLASS.format(root=ROOT), "gpu_pointwise_shard class", timeout=600)
    assert rc == 0 and "class ok" in out, out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("model,opt", [("gmf", "adagrad"), ("wrmf_sigmoid", "adam")])
def test_sharded_pointwise_multi_gpu(model, opt):
    for rc, out in run_ranks(torch.cuda.device_count(), [os.path.join(ROOT, "tests", "_pointwise_shard_worker.py"),
                                                         "nccl", model, opt], f"gpu_pointwise_shard {model} {opt}",
                             timeout=600):
        assert rc == 0 and "rank ok" in out, out
