"""GPU: the multi-hot row-sharded DLRM.  orx_bag_shard_lookups and orx_bag_segment_sum against numpy; the sharded step
of ShardedDLRM(bag_sizes, pooling)'s parts with R virtual ranks on one device (LoopbackExchange: every rank its own
liborx handle, the multi-GPU code and kernels) against the single-GPU DLRM(bag_sizes) on the global batch; bags of one
id against the one-hot sharded step; sharded inference; ShardedDLRM(bag_sizes) in a one-rank NCCL group with the
reference example's train_step and Keras Adam(), a checkpoint round trip and its refusals; and a worker-process job on
>= 2 GPUs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]

import dlrm_bags_np as NB  # noqa: E402
from _ranks import run_ranks  # noqa: E402
from dlrm_bags_shard_np import bag_segment_sum_np, bag_shard_lookups_np  # noqa: E402
from dlrm_shard_np import lookup_bucket_np  # noqa: E402


@pytest.fixture(scope="module")
def eng():
    from openrec_b200 import native
    return native.engine()


def _bags(rng, vocab, sizes, B, kind):
    """[B, sum(sizes)] int32 bags: uniform / zipf ids in full bags, 'bad' (padding, = vocab, >> vocab, 2^31 - 1 and
    repeated ids among valid ones) or 'ragged' (bag lengths 0 .. L, the rest -1)."""
    cols = []
    for v, L in zip(vocab, sizes):
        if kind == "zipf":
            c = np.minimum(rng.zipf(1.3, (B, L)) - 1, v - 1)
        elif kind == "bad":
            c = rng.choice(np.array([-1, -7, v, v + 1, 2 ** 31 - 1] + list(range(v))), (B, L))
            if L > 1:
                c[:, 1] = np.where(rng.random(B) < 0.3, c[:, 0], c[:, 1])
        else:
            c = rng.integers(0, v, (B, L))
            if kind == "ragged":
                c[np.arange(L)[None, :] >= rng.integers(0, L + 1, B)[:, None]] = -1
        cols.append(c)
    return np.concatenate(cols, 1).astype(np.int32) if cols else np.zeros((B, 0), np.int32)


# ---- orx_bag_shard_lookups ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,Lmax", [(1, 1), (1, 100), (5, 7), (26, 100), (63, 3)])
def test_bag_shard_lookups_exact(eng, T, Lmax):
    rng = np.random.default_rng(T * 1000 + Lmax)
    vocab = list(rng.integers(1, 4, T // 3)) + list(rng.integers(50, 5000, T - T // 3))
    sizes = list(rng.integers(1, Lmax + 1, T))
    sizes[0] = Lmax
    row_off, col_off = NB.col_offsets(vocab), NB.col_offsets(sizes)
    for B in (0, 1, 777):
        sp = _bags(rng, vocab, sizes, B, "bad")
        got = eng.bag_shard_lookups(torch.from_numpy(sp).cuda(), col_off.tolist(), row_off.tolist())
        assert got.shape == (B, col_off[-1])
        np.testing.assert_array_equal(got.cpu().numpy(), bag_shard_lookups_np(sp, col_off, row_off))


def test_bag_shard_lookups_refusals(eng):
    s = torch.zeros(4, 3, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        eng.bag_shard_lookups(s, [0, 1, 3], [0, 2 ** 30, 2 ** 31])        # G > 2^31 - 1
    with pytest.raises(RuntimeError):
        eng.bag_shard_lookups(s, [0, 1, 3], [0, 5, 4])                    # row offsets decrease
    with pytest.raises(RuntimeError):
        eng.bag_shard_lookups(torch.zeros(4, 64, dtype=torch.int32, device="cuda"), list(range(65)), list(range(65)))
    with pytest.raises(ValueError):
        eng.bag_shard_lookups(s, [0, 1, 2], [0, 5, 9])                    # 2 columns for a [4, 3] batch
    with pytest.raises(ValueError):
        eng.bag_shard_lookups(s, [0, 3], [0, 5, 9])                       # T + 1 entries each


# ---- orx_bag_segment_sum --------------------------------------------------------------------------------------------
def _fold_case(eng, rng, vocab, sizes, B, kind, R=1):
    """A batch of bags bucketed as the step buckets it -> (sparse, col_off, slot, grp_off, grp_idx, n_uniq) with the
    device tensors of the bucket tuple."""
    row_off, col_off = NB.col_offsets(vocab), NB.col_offsets(sizes)
    sp = _bags(rng, vocab, sizes, B, kind)
    rows = eng.bag_shard_lookups(torch.from_numpy(sp).cuda(), col_off.tolist(), row_off.tolist())
    bk = eng.lookup_bucket(rows.view(-1, 1), [0, int(row_off[-1])], R)
    return sp, col_off.tolist(), bk, int(bk[0].sum())


def _strided_dz(rng, B, T, D, pad=4):
    buf = torch.from_numpy(rng.standard_normal((B, T * D + pad)).astype(np.float32)).cuda()
    return buf[:, :T * D].unflatten(1, (T, D))


# (D, row padding of dZ): float4 for D % 4 == 0 with a padding of 4; the scalar path for D = 1, 6, and for D = 40 and
# D = 128 at an odd row stride, which take several 32-column chunks with idle lanes in the last one (D = 40)
@pytest.mark.parametrize("D,pad", [(1, 4), (4, 4), (6, 4), (40, 4), (40, 1), (128, 4), (128, 1), (512, 4)])
@pytest.mark.parametrize("mode", [0, 1])
def test_bag_segment_sum(eng, D, pad, mode):
    rng = np.random.default_rng(D * 2 + mode + pad)
    vocab, sizes, B = [2, 3, 900, 40], [100, 1, 7, 33], 300          # table 0: one row with thousands of lookups
    sp, col_off, bk, n_uniq = _fold_case(eng, rng, vocab, sizes, B, "bad", R=3)
    _, _, slot, grp_off, grp_idx = bk
    dz = _strided_dz(rng, B, len(vocab), D, pad)
    assert dz.stride(0) == len(vocab) * D + pad
    out = eng.bag_segment_sum(dz, col_off, mode, slot, grp_off, grp_idx, n_uniq)
    go, gi, sl = grp_off.cpu().numpy(), grp_idx.cpu().numpy(), slot.cpu().numpy()
    z = dz.cpu().numpy().astype(np.float64)
    want = bag_segment_sum_np(z, col_off, mode == 1, sl, go, gi, n_uniq, np.float64)
    scale = bag_segment_sum_np(np.abs(z), col_off, mode == 1, sl, go, gi, n_uniq, np.float64)
    cnt = (go[1:n_uniq + 1] - go[:n_uniq]).max()
    assert cnt >= 2000
    err = np.abs(out.cpu().numpy() - want) / np.maximum(scale, 1e-30)
    assert err.max() <= 2.0 ** -24 * (cnt + mode) * 2, err.max()
    # the documented order (ascending p, a mean divided before the add) in float32: the same bits
    exact = bag_segment_sum_np(dz.cpu().numpy(), col_off, mode == 1, sl, go, gi, n_uniq)
    assert np.array_equal(out.cpu().numpy(), exact)
    for _ in range(3):
        assert torch.equal(eng.bag_segment_sum(dz, col_off, mode, slot, grp_off, grp_idx, n_uniq), out)


def test_bag_segment_sum_no_rows_and_one_hot(eng):
    rng = np.random.default_rng(1)
    vocab, D = [3, 1, 50, 9], 128
    sp = -np.ones((20, 8), np.int32)                                  # every id padding: n_uniq = 0
    rows = eng.bag_shard_lookups(torch.from_numpy(sp).cuda(), [0, 2, 3, 7, 8], NB.col_offsets(vocab).tolist())
    bk = eng.lookup_bucket(rows.view(-1, 1), [0, sum(vocab)], 2)
    assert int(bk[0].sum()) == 0
    dz = _strided_dz(rng, 20, 4, D)
    for mode in (0, 1):
        assert eng.bag_segment_sum(dz, [0, 2, 3, 7, 8], mode, bk[2], bk[3], bk[4], 0).shape == (0, D)
    for D in (1, 6, 128):                                             # every L = 1, sum: orx_rows_segment_sum on dZ
        sp, col_off, bk, n_uniq = _fold_case(eng, rng, vocab, [1] * 4, 500, "bad", R=3)
        dz = torch.from_numpy(rng.standard_normal((500, 4, D)).astype(np.float32)).cuda()
        got = eng.bag_segment_sum(dz, col_off, 0, bk[2], bk[3], bk[4], n_uniq)
        assert torch.equal(got, eng.rows_segment_sum(dz.view(-1, D), bk[3], bk[4], n_uniq))


def test_bag_segment_sum_refusals(eng):
    import ctypes as C
    rng = np.random.default_rng(2)
    sp, col_off, bk, n = _fold_case(eng, rng, [5, 7], [2, 3], 10, "uniform")
    dz = torch.zeros(10, 2, 4, device="cuda")
    ok = dict(dz=dz, ld=8, T=2, dim=4, co=col_off, mode=1, slot=bk[2], B=10, go=bk[3], gi=bk[4], n=n,
              out=torch.empty(n, 4, device="cuda"))

    def call(**kw):
        a = dict(ok, **kw)
        co = (C.c_int32 * len(a["co"]))(*a["co"])
        p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
        return eng.lib.orx_bag_segment_sum(eng.h, p(a["dz"]), a["ld"], a["T"], a["dim"], co, a["mode"], p(a["slot"]),
                                           a["B"], p(a["go"]), p(a["gi"]), a["n"], p(a["out"]), eng.stream())
    assert call() == 0
    for bad in (dict(T=0, co=[0]), dict(T=64, co=list(range(65))), dict(dim=0), dict(B=-1), dict(n=-1), dict(n=51),
                dict(mode=2), dict(ld=7), dict(co=[1, 2, 5]), dict(co=[0, 3, 2]), dict(co=[0, 0, 0]), dict(dz=None),
                dict(go=None), dict(gi=None), dict(out=None), dict(slot=None)):
        assert call(**bad) == -1, bad                                  # ORX_ERR_INVALID
    assert call(slot=None, mode=0) == 0                                # a sum reads no slot
    with pytest.raises(ValueError):
        eng.bag_segment_sum(dz, [0, 2], 0, bk[2], bk[3], bk[4], n)     # T + 1 entries
    with pytest.raises(ValueError):
        eng.bag_segment_sum(dz, col_off, 0, bk[2][:-1], bk[3], bk[4], n)


# ---- loopback: R virtual ranks against the single-GPU DLRM(bag_sizes) ----------------------------------------------
OPTS = {"sgd": 0.1, "adagrad": 0.05, "adam": 0.01, "lazyadam": 0.01}
TOL = {"sgd": 1e-5, "adagrad": 1e-5, "adam": 1e-4, "lazyadam": 1e-5}      # those of tests/test_gpu_dlrm_shard.py

CASES = [  # R, optimizer, pooling, interaction mode, D, vocabularies, bag sizes, id kind
    (1, "adagrad", "sum", "dlrm", 128, [3, 1000, 1, 700], [4, 100, 2, 1], "uniform"),
    (2, "sgd", "mean", "reference", 4, [3, 1, 50, 2, 9], [2, 3, 7, 1, 5], "bad"),
    (3, "lazyadam", "mean", "dlrm", 4, [3, 1, 50, 2, 9], [3, 1, 33, 2, 4], "zipf"),
    (8, "adagrad", "sum", "dlrm", 4, [2, 1, 3], [3, 2, 5], "bad"),                 # G = 6 < R
    (8, "adam", "mean", "reference", 128, [3, 500, 2, 40], [1, 9, 4, 2], "ragged"),
    (3, "adam", "sum", "dlrm", 6, [3, 1, 50, 2, 9], [2, 2, 7, 1, 3], "ragged"),
    (2, "sgd", "sum", "dlrm", 128, [1, 2, 3, 400], [1, 4, 2, 12], "zipf"),
    (1, "lazyadam", "sum", "reference", 16, [5, 300, 2], [3, 8, 1], "bad"),
]


def _ref_and_parts(R, opt_name, D, vocab, sizes, pooling, mode, n_dense=5, one_hot_too=False):
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM
    from openrec_b200 import native
    from openrec_b200.sharded import DLRMShard
    from openrec_b200.tf2.mlp_ops import ACT
    ref = DLRM(m_spa=D, ln_emb=vocab, ln_bot=[16, D], ln_top=[32, 1], interaction_mode=mode, bag_sizes=sizes,
               pooling=pooling)
    ref._graph(n_dense)
    opt = {"sgd": tf.keras.optimizers.SGD, "adagrad": tf.keras.optimizers.Adagrad, "adam": tf.keras.optimizers.Adam,
           "lazyadam": tf.keras.optimizers.LazyAdam}[opt_name](learning_rate=OPTS[opt_name])
    table = torch.cat([lf.embeddings.t for lf in ref._latent_factors])
    dense_vars = ref.trainable_variables[len(vocab):]
    acts = [l.activation for l in ref._mlp_bot.layers + ref._mlp_top.layers]
    engines, sets = [], []
    for col_off in ([ref._col_off, None] if one_hot_too else [ref._col_off]):
        parts = []
        for r in range(R):
            engines.append(native.Engine(0))
            rows = (table.shape[0] - r + R - 1) // R
            t = torch.zeros(max(rows, 1), D, device="cuda")
            t[:rows] = table[r::R]
            slots = [torch.full_like(t, 0.1 if opt_name == "adagrad" else 0.0) if s is not None else None
                     for s in opt.slots(ref._latent_factors[0].embeddings)]
            reps = [v.t.clone() for v in dense_vars]
            dslots = [tuple(x.clone() if x is not None else None for x in opt.slots(v)) for v in dense_vars]
            trip = [(reps[2 * l], reps[2 * l + 1], ACT[acts[l]]) for l in range(len(acts))]
            parts.append(DLRMShard(engines[-1], r, R, vocab, D, trip[:2], trip[2:], t, slots, dslots, mode=mode,
                                   col_off=col_off, pooling=ref._pooling))
        sets.append(parts)
    return ref, opt, sets, engines, dense_vars


def _global(parts, what):
    R, G = parts[0].world, parts[0].G
    out = torch.zeros(G, parts[0].D, device="cuda")
    for p in parts:
        out[p.rank::R] = (p.table if what is None else p.slots[what])[:p.rows]
    return out


def _split(R, B, *xs):
    return [tuple(x[r * B:(r + 1) * B].contiguous() for x in xs) for r in range(R)]


@pytest.mark.parametrize("case", CASES, ids=[f"R{c[0]}-{c[1]}-{c[2]}-{c[3]}-D{c[4]}-{c[7]}" for c in CASES])
def test_loopback_step_equals_single_gpu(case):
    import tensorflow as tf
    from openrec_b200.sharded import LoopbackExchange, _dlrm_fetch, dlrm_step_sharded
    R, opt_name, pooling, mode, D, vocab, sizes, idk = case
    B, n_dense = 24, 5
    ref, opt, (parts,), engines, dense_vars = _ref_and_parts(R, opt_name, D, vocab, sizes, pooling, mode, n_dense)
    xchg = LoopbackExchange()
    rng = np.random.default_rng(R + D)
    try:
        for step in range(1, 4):
            dense = torch.from_numpy(rng.random((R * B, n_dense)).astype(np.float32)).cuda()
            sparse = torch.from_numpy(_bags(rng, vocab, sizes, R * B, idk)).cuda()
            label = torch.from_numpy((rng.random(R * B) < 0.4).astype(np.float32)).cuda()
            batches = _split(R, B, dense, sparse, label)
            if step == 1:                       # Z: the single-GPU pooling, bit for bit
                Zs = _dlrm_fetch(parts, xchg, [b[1] for b in batches], True)[0]
                assert torch.equal(torch.cat(Zs), ref._graph(n_dense).forward(dense, sparse)["Z"])
            with tf.GradientTape() as tape:
                lv = ref(dense, sparse, label)
            opt.apply_gradients(zip(tape.gradient(lv, ref.trainable_variables), ref.trainable_variables))
            want_loss = float(lv.numpy())
            o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, step)
            for out in dlrm_step_sharded(parts, xchg, batches, o):
                got = float(out[0])
                assert abs(got - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (step, got, want_loss)
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


@pytest.mark.parametrize("R,opt_name", [(1, "adagrad"), (1, "adam"), (3, "lazyadam"), (8, "sgd")])
def test_one_id_bags_equal_one_hot_step(R, opt_name):
    """bag_sizes = [1] * T with sum pooling: three steps bit-identical to the one-hot sharded step from the same state.
    Rank r's ids are r modulo R, so no row is in two ranks' batches: an owner's apply then stages no sum of several
    ranks' gradient rows, whose atomic order varies from run to run in either form."""
    from openrec_b200.sharded import LoopbackExchange, dlrm_step_sharded
    vocab, D, B = [3, 1, 50, 2, 9], 4 if R > 1 else 128, 16
    _, opt, (bags, one_hot), engines, _ = _ref_and_parts(R, opt_name, D, vocab, [1] * 5, "sum", "dlrm",
                                                         one_hot_too=True)
    xchg = LoopbackExchange()
    rng = np.random.default_rng(R)
    try:
        for step in range(1, 4):
            dense = torch.from_numpy(rng.random((R * B, 5)).astype(np.float32)).cuda()
            sp = _bags(rng, vocab, [1] * 5, R * B, "bad")
            own = np.repeat(np.arange(R), B)[:, None]
            sp[(sp >= 0) & (sp < np.array(vocab)[None, :]) & (sp % R != own)] = -1
            sparse = torch.from_numpy(sp).cuda()
            label = torch.from_numpy((rng.random(R * B) < 0.4).astype(np.float32)).cuda()
            batches = _split(R, B, dense, sparse, label)
            o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, step)
            a, b = dlrm_step_sharded(bags, xchg, batches, o), dlrm_step_sharded(one_hot, xchg, batches, o)
            assert all(torch.equal(x, y) for x, y in zip(a, b))
        for p, q in zip(bags, one_hot):
            assert torch.equal(p.table, q.table)
            assert all(s is None or torch.equal(s, t) for s, t in zip(p.slots, q.slots))
            assert all(torch.equal(x, y) for x, y in zip(p.dense_vars(), q.dense_vars()))
    finally:
        torch.cuda.synchronize()
        for e in engines:
            e.close()


@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_loopback_inference(R, pooling):
    from openrec_b200.sharded import LoopbackExchange, dlrm_inference_sharded
    vocab, sizes, D = [3, 1, 50, 2, 9], [2, 3, 7, 1, 5], 4
    ref, _, (parts,), engines, _ = _ref_and_parts(R, "sgd", D, vocab, sizes, pooling, "dlrm")
    rng = np.random.default_rng(R)
    try:
        n = [0 if r == R - 1 and R > 1 else 5 + r for r in range(R)]        # the last rank has no samples
        batches = [(torch.from_numpy(rng.random((b, 5)).astype(np.float32)).cuda(),
                    torch.from_numpy(_bags(rng, vocab, sizes, b, "bad")).cuda()) for b in n]
        for (dense, sparse), pred in zip(batches, dlrm_inference_sharded(parts, LoopbackExchange(), batches)):
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
vocab, sizes, D = [3, 1, 500, 2, 90], [2, 1, 20, 3, 4], 16
kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[32, D], ln_top=[64, 1], interaction_mode="dlrm", bag_sizes=sizes,
          pooling="mean")
for bad in (dict(bag_sizes=sizes[:-1]), dict(bag_sizes=[2, 0, 1, 1, 1]), dict(pooling="max")):
    try:
        ShardedDLRM(**dict(kw, **bad))
        raise SystemExit(f"{{bad}} accepted")
    except ValueError:
        pass
models = [ShardedDLRM(**kw), DLRM(**kw)]
models[0]._build(13); models[1]._graph(13)
for lf, k in zip(models[1]._latent_factors, np.cumsum([0] + vocab[:-1])):
    lf.embeddings.t.copy_(models[0].embedding_shard.t[k:k + lf.embeddings.t.shape[0]])
for a, b in zip(models[0].trainable_variables[1:], models[1].trainable_variables[len(vocab):]):
    b.t.copy_(a.t)
rng = np.random.default_rng(0)
def bags(n):
    c = np.concatenate([rng.integers(-1, v + 1, (n, L)) for v, L in zip(vocab, sizes)], 1)
    return c.astype(np.int32)
data = [(rng.random((64, 13)).astype(np.float32), bags(64), (rng.random(64) < 0.3).astype(np.float32))
        for _ in range(3)]
try:
    models[0](data[0][0], data[0][1][:, :5], data[0][2])
    raise SystemExit("sparse width 5 accepted")
except ValueError:
    pass
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
torch.testing.assert_close(models[0].inference(data[0][0], data[0][1]).t, models[1].inference(data[0][0], data[0][1]).t,
                           atol=1e-4, rtol=1e-4)
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


def test_sharded_dlrm_bags_class_one_rank():
    [(rc, out)] = run_ranks(1, _CLASS.format(root=ROOT), "gpu_dlrm_bags_shard class", timeout=600)
    assert rc == 0 and "class ok" in out, out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_dlrm_bags_multi_gpu():
    worker = [os.path.join(ROOT, "tests", "_dlrm_bags_shard_worker.py"), "nccl", "adagrad", "mean", "dlrm"]
    for rc, out in run_ranks(torch.cuda.device_count(), worker, "gpu_dlrm_bags_shard multi", timeout=600):
        assert rc == 0 and "rank ok" in out, out
