"""GPU: the row-sharded DLRM.  orx_lookup_bucket and orx_rows_segment_sum against numpy; the sharded step with R virtual
ranks on one device (LoopbackExchange: every rank its own liborx handle, the multi-GPU code and kernels) against the
single-GPU DLRM on the global batch; sharded inference; ShardedDLRM in a one-rank NCCL group with the reference
example's train_step and Keras Adam(), and a checkpoint round trip; and a worker-process job on >= 2 GPUs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]

from _ranks import run_ranks  # noqa: E402
from dlrm_shard_np import lookup_bucket_np  # noqa: E402


@pytest.fixture(scope="module")
def eng():
    from openrec_b200 import native
    return native.engine()


def _ids(rng, vocab, B, kind):
    cols = []
    for v in vocab:
        if kind == "zipf":
            c = np.minimum(rng.zipf(1.3, B) - 1, v - 1)
        elif kind == "bad":                    # < 0, = vocab, >> vocab among valid ids
            c = rng.choice(np.array([-1, -7, v, v + 1, 2 ** 31 - 1] + list(range(max(v, 1)))), B)
        else:
            c = rng.integers(0, max(v, 1), B)
        cols.append(c)
    return np.stack(cols, 1).astype(np.int32)


@pytest.mark.parametrize("R", [1, 2, 3, 8, 64])
@pytest.mark.parametrize("T", [1, 3, 26])
@pytest.mark.parametrize("kind", ["uniform", "zipf", "bad", "tiny"])
def test_lookup_bucket_exact(eng, R, T, kind):
    rng = np.random.default_rng(R * 100 + T)
    if kind == "tiny":                          # vocabularies of 1-3 rows: G < R for the large R
        vocab = list(rng.integers(1, 4, T))
    else:
        vocab = list(rng.integers(1, 4, T // 3)) + list(rng.integers(50, 5000, T - T // 3))
    off = np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64)
    for B in (0, 1, 777):
        sparse = _ids(rng, vocab, B, "uniform" if kind == "tiny" else kind)
        got = eng.lookup_bucket(torch.from_numpy(sparse).cuda(), off.tolist(), R)
        counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(sparse, off, R)
        n_uniq, n_valid = len(send_local), int(grp_off[-1])
        g = [t.cpu().numpy() for t in got]
        np.testing.assert_array_equal(g[0], counts)
        np.testing.assert_array_equal(g[1][:n_uniq], send_local)
        np.testing.assert_array_equal(g[2], slot)
        np.testing.assert_array_equal(g[3][:n_uniq + 1], grp_off)
        np.testing.assert_array_equal(g[4][:n_valid], grp_idx)


def test_lookup_bucket_refusals(eng):
    s = torch.zeros(4, 2, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        eng.lookup_bucket(s, [0, 2 ** 30, 2 ** 31], 2)          # G > 2^31 - 1
    with pytest.raises(RuntimeError):
        eng.lookup_bucket(s, [0, 3, 2], 2)                      # offsets decrease
    with pytest.raises(RuntimeError):
        eng.lookup_bucket(s, [0, 3, 5], 1025)                   # world > 1024
    with pytest.raises(ValueError):
        eng.lookup_bucket(s, [0, 3], 2)                         # T + 1 offsets


@pytest.mark.parametrize("D", [1, 4, 6, 128, 512])
def test_rows_segment_sum(eng, D):
    rng = np.random.default_rng(D)
    n, ld = 5000, D + 4
    src = torch.from_numpy(rng.standard_normal((n, ld)).astype(np.float32)).cuda()[:, :D]
    sparse = np.concatenate([rng.integers(0, 3, (n // 2, 1)), rng.integers(0, 900, (n - n // 2, 1))]).astype(np.int32)
    counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(sparse, [0, 1000], 1)
    n_uniq = len(send_local)
    go, gi = torch.from_numpy(grp_off).cuda(), torch.from_numpy(grp_idx).cuda()
    out = eng.rows_segment_sum(src, go, gi, n_uniq)
    s = src.cpu().numpy().astype(np.float64)
    want = np.stack([s[grp_idx[grp_off[j]:grp_off[j + 1]]].sum(0) for j in range(n_uniq)])
    scale = np.stack([np.abs(s[grp_idx[grp_off[j]:grp_off[j + 1]]]).sum(0) for j in range(n_uniq)])
    err = np.abs(out.cpu().numpy() - want) / np.maximum(scale, 1e-30)
    assert err.max() <= 2.0 ** -24 * (grp_off[1:] - grp_off[:-1]).max() * 2, err.max()
    for _ in range(3):
        assert torch.equal(eng.rows_segment_sum(src, go, gi, n_uniq), out)
    assert eng.rows_segment_sum(src, go, gi, 0).shape == (0, D)


# ---- loopback: R virtual ranks against the single-GPU DLRM ---------------------------------------------------------
OPTS = {"sgd": 0.1, "adagrad": 0.05, "adam": 0.01, "lazyadam": 0.01}
# Keras Adam() sweeps every row with m / (sqrt(v) + eps): a gradient element that is a near-cancelling sum (|g| ~ 1e-9)
# is normalised to about +-1, so a reordered sum can move its row by up to lr.  1e-4 = lr / 100 bounds that on these
# shapes; SGD, Adagrad and LazyAdam are held to 1e-5.
TOL = {"sgd": 1e-5, "adagrad": 1e-5, "adam": 1e-4, "lazyadam": 1e-5}

CASES = [  # R, optimizer, interaction mode, loss, loss threshold, D, vocabularies, id kind
    (1, "adagrad", "dlrm", "mse", 0.0, 128, [3, 1000, 1, 700], "uniform"),
    (2, "sgd", "reference", "bce", 0.0, 4, [3, 1, 50, 2, 9], "bad"),
    (3, "lazyadam", "dlrm", "bce", 0.02, 4, [3, 1, 50, 2, 9], "zipf"),
    (8, "adagrad", "dlrm", "mse", 0.0, 4, [2, 1, 3], "bad"),          # G = 6 < R
    (8, "adam", "reference", "mse", 0.0, 128, [3, 500, 2, 40], "zipf"),
    (3, "adam", "dlrm", "bce", 0.02, 4, [3, 1, 50, 2, 9], "uniform"),
    (2, "sgd", "dlrm", "mse", 0.0, 128, [1, 2, 3, 400], "bad"),
]


def _ref_and_parts(R, opt_name, mode, loss, thr, D, vocab, n_dense=5):
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM
    from openrec_b200 import native
    from openrec_b200.sharded import DLRMShard
    ref = DLRM(m_spa=D, ln_emb=vocab, ln_bot=[16, D], ln_top=[32, 1], loss_func=loss, loss_threshold=thr,
               interaction_mode=mode)
    ref._graph(n_dense)
    opt = {"sgd": tf.keras.optimizers.SGD, "adagrad": tf.keras.optimizers.Adagrad, "adam": tf.keras.optimizers.Adam,
           "lazyadam": tf.keras.optimizers.LazyAdam}[opt_name](learning_rate=OPTS[opt_name])
    table = torch.cat([lf.embeddings.t for lf in ref._latent_factors])          # the concatenated row space
    dense_vars = ref.trainable_variables[len(vocab):]
    engines = [native.Engine(0) for _ in range(R)]
    parts = []
    for r in range(R):
        rows = (table.shape[0] - r + R - 1) // R
        t = torch.zeros(max(rows, 1), D, device="cuda")
        t[:rows] = table[r::R]
        slots = [torch.zeros_like(t) if s is not None else None for s in opt.slots(ref._latent_factors[0].embeddings)]
        for s in slots:
            if s is not None and opt_name == "adagrad":
                s.fill_(0.1)
        reps = [v.t.clone() for v in dense_vars]
        dslots = [tuple(x.clone() if x is not None else None for x in opt.slots(v)) for v in dense_vars]
        acts = [l.activation for l in ref._mlp_bot.layers + ref._mlp_top.layers]
        from openrec_b200.tf2.mlp_ops import ACT
        trip = [(reps[2 * l], reps[2 * l + 1], ACT[acts[l]]) for l in range(len(acts))]
        parts.append(DLRMShard(engines[r], r, R, vocab, D, trip[:2], trip[2:], t, slots, dslots,
                               self_interaction=False, mode=mode, loss_kind=0 if loss == "mse" else 1,
                               clip=thr))
    return ref, opt, parts, engines, dense_vars


def _global(parts, what):
    R, G = parts[0].world, parts[0].G
    out = torch.zeros(G, parts[0].D, device="cuda")
    for p in parts:
        src = p.table if what is None else p.slots[what]
        out[p.rank::R] = src[:p.rows]
    return out


@pytest.mark.parametrize("case", CASES, ids=[f"R{c[0]}-{c[1]}-{c[2]}-{c[3]}-D{c[5]}-{c[7]}" for c in CASES])
def test_loopback_step_equals_single_gpu(case):
    import tensorflow as tf
    from openrec_b200.sharded import LoopbackExchange, _dlrm_fetch, dlrm_step_sharded
    R, opt_name, mode, loss_func, thr, D, vocab, idk = case
    B, n_dense = 24, 5
    ref, opt, parts, engines, dense_vars = _ref_and_parts(R, opt_name, mode, loss_func, thr, D, vocab, n_dense)
    xchg = LoopbackExchange()
    rng = np.random.default_rng(R + D)
    try:
        for step in range(1, 4):
            dense = torch.from_numpy(rng.random((R * B, n_dense)).astype(np.float32)).cuda()
            sparse = torch.from_numpy(_ids(rng, vocab, R * B, idk)).cuda()
            label = torch.from_numpy((rng.random(R * B) < 0.4).astype(np.float32)).cuda()
            batches = [(dense[r * B:(r + 1) * B], sparse[r * B:(r + 1) * B].contiguous(), label[r * B:(r + 1) * B])
                       for r in range(R)]
            if step == 1:                       # Z: the single-GPU gather, bit for bit
                Zs = _dlrm_fetch(parts, xchg, [b[1] for b in batches], True)[0]
                want = ref._graph(n_dense).forward(dense, sparse)["Z"]
                assert torch.equal(torch.cat(Zs), want)
            with tf.GradientTape() as tape:
                lv = ref(dense, sparse, label)
            grads = tape.gradient(lv, ref.trainable_variables)
            opt.apply_gradients(zip(grads, ref.trainable_variables))
            want_loss = float(lv.numpy())
            o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, step)
            outs = dlrm_step_sharded(parts, xchg, batches, o)
            for out in outs:
                assert abs(float(out[0]) - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (step, float(out[0]), want_loss)
        tol = TOL[opt_name]
        table = torch.cat([lf.embeddings.t for lf in ref._latent_factors])
        torch.testing.assert_close(_global(parts, None), table, atol=tol, rtol=tol)
        for j, s in enumerate(opt.slots(ref._latent_factors[0].embeddings)):
            if s is not None:
                want = torch.cat([opt.slots(lf.embeddings)[j] for lf in ref._latent_factors])
                torch.testing.assert_close(_global(parts, j), want, atol=tol, rtol=tol)
        for p in parts:
            for k, (var, v) in enumerate(zip(p.dense_vars(), dense_vars)):
                assert torch.equal(var, parts[0].dense_vars()[k]), "Dense replicas differ"
                torch.testing.assert_close(var, v.t, atol=tol, rtol=tol)
                for j, s in enumerate(opt.slots(v)):
                    if s is not None:
                        assert torch.equal(p.dense_slots[k][j], parts[0].dense_slots[k][j])
                        torch.testing.assert_close(p.dense_slots[k][j], s, atol=tol, rtol=tol)
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


@pytest.mark.parametrize("R", [1, 3, 8])
def test_loopback_inference(R):
    from openrec_b200.sharded import LoopbackExchange, dlrm_inference_sharded
    vocab, D = [3, 1, 50, 2, 9], 4
    ref, opt, parts, engines, _ = _ref_and_parts(R, "sgd", "dlrm", "mse", 0.0, D, vocab)
    rng = np.random.default_rng(R)
    try:
        sizes = [0 if r == R - 1 and R > 1 else 5 + r for r in range(R)]       # the last rank has no samples
        batches = [(torch.from_numpy(rng.random((b, 5)).astype(np.float32)).cuda(),
                    torch.from_numpy(_ids(rng, vocab, b, "bad")).cuda()) for b in sizes]
        preds = dlrm_inference_sharded(parts, LoopbackExchange(), batches)
        for (dense, sparse), pred in zip(batches, preds):
            if dense.shape[0] == 0:
                assert pred.numel() == 0
                continue
            torch.testing.assert_close(pred, ref.inference(dense, sparse).t, atol=1e-6, rtol=1e-5)
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


_CLASS = r"""
import os, sys, tempfile
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(0)
dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
import tensorflow as tf
from openrec.tf2.recommenders import DLRM, ShardedDLRM
from openrec_b200.tf2 import checkpoint
vocab, D = [3, 1, 500, 2, 90], 16
kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[32, D], ln_top=[64, 1], interaction_mode="dlrm")
models = [ShardedDLRM(**kw), DLRM(**kw)]
models[0]._build(13); models[1]._graph(13)
for lf, k in zip(models[1]._latent_factors, np.cumsum([0] + vocab[:-1])):
    lf.embeddings.t.copy_(models[0].embedding_shard.t[k:k + lf.embeddings.t.shape[0]])
for a, b in zip(models[0].trainable_variables[1:], models[1].trainable_variables[len(vocab):]):
    b.t.copy_(a.t)
rng = np.random.default_rng(0)
data = [(rng.random((64, 13)).astype(np.float32), np.stack([rng.integers(0, v, 64) for v in vocab], 1).astype(np.int32),
         (rng.random(64) < 0.3).astype(np.float32)) for _ in range(3)]
losses = []
for dlrm_model in models:
    optimizer = tf.keras.optimizers.Adam()

    @tf.function
    def train_step(dense_features, sparse_features, label):
        with tf.GradientTape() as tape:
            loss_value = dlrm_model(dense_features, sparse_features, label)
        gradients = tape.gradient(loss_value, dlrm_model.trainable_variables)
        optimizer.apply_gradients(zip(gradients, dlrm_model.trainable_variables))
        return loss_value

    losses.append([float(train_step(*b).numpy()) for b in data])
    if dlrm_model is models[0]:
        opt0 = optimizer
np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5, atol=1e-6)
table = torch.cat([lf.embeddings.t for lf in models[1]._latent_factors])
torch.testing.assert_close(models[0].embedding_shard.t, table, atol=1e-4, rtol=1e-4)
path = os.path.join(tempfile.mkdtemp(), "rank0.npz")
checkpoint.save(path, models[0], opt0)
before = [v.t.clone() for v in models[0].trainable_variables]
fresh = ShardedDLRM(**kw, seed=5)
opt1 = tf.keras.optimizers.Adam()
fresh._build(13)
checkpoint.load(path, fresh, opt1)
for a, b in zip(before, fresh.trainable_variables):
    assert torch.equal(a, b.t)
assert opt1.iterations == 3
p0 = models[0].inference(data[0][0], data[0][1]).t
torch.testing.assert_close(p0, fresh.inference(data[0][0], data[0][1]).t, atol=0, rtol=0)
dist.destroy_process_group()
print("class ok")
"""


def test_sharded_dlrm_class_one_rank():
    [(rc, out)] = run_ranks(1, _CLASS.format(root=ROOT), "gpu_dlrm_shard class", timeout=600)
    assert rc == 0 and "class ok" in out, out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_dlrm_multi_gpu():
    for rc, out in run_ranks(torch.cuda.device_count(), [os.path.join(ROOT, "tests", "_dlrm_shard_worker.py"), "nccl",
                                                         "adagrad", "dlrm", "mse"], "gpu_dlrm_shard multi", timeout=600):
        assert rc == 0 and "rank ok" in out, out
