"""CPU, world size 2 and 3 over gloo: ShardedGMF / ShardedWRMF through the reference example's step protocol reproduce
the oracle's single-process pointwise step on the valid samples of the concatenated global batch for three steps
(losses, every table row, every optimizer slot, w; tests/_pointwise_shard_worker.py), with the oracle-backed engine and
numpy restatements of tests/pointwise_shard_np.py.  This checks the layout, the exchanges and the step's arithmetic
plan; the kernels are checked in tests/test_gpu_pointwise_shard.py.  Also: the numpy restatements against their
contracts written out sample by sample, and the refusals."""
import os
import sys

import numpy as np
import pytest
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_pointwise_shard_worker.py")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("model,opt", [("gmf", "sgd"), ("gmf", "adagrad"), ("gmf", "lazyadam"), ("gmf", "adam"),
                                       ("wrmf", "adagrad"), ("wrmf_sigmoid", "adam"), ("wrmf", "sgd"),
                                       ("wrmf_sigmoid", "lazyadam")])
def test_sharded_pointwise_equals_oracle(world, model, opt):
    for rc, out in run_ranks(world, [WORKER, "gloo", model, opt], f"pointwise_shard_cpu {model} {opt}"):
        assert rc == 0 and "rank ok" in out, out


_ERRORS = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
import pointwise_shard_np
pointwise_shard_np.install()
dist.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
from openrec.tf2.recommenders import ShardedGMF, ShardedWRMF
import tensorflow as tf
rank = dist.get_rank()
for bad in (lambda: ShardedWRMF(4, 4, 2 ** 30, 2 ** 30), lambda: ShardedGMF(4, 8, 10, 10)):
    try:
        bad()
        raise SystemExit("accepted")
    except ValueError:
        pass
model = ShardedGMF(4, 4, 10, 10)
try:
    model.inference(np.zeros(2, np.int32))
    raise SystemExit("inference accepted")
except NotImplementedError as e:
    assert "Retriever" in str(e)
opt = tf.keras.optimizers.Adagrad(0.05)
B = 4 + rank                                   # unequal local batches: every rank raises
with tf.GradientTape() as tape:
    loss, l2 = model(np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.float32))
grads = tape.gradient((loss, l2), model.trainable_variables)
try:
    opt.apply_gradients(zip(grads, model.trainable_variables))
    raise SystemExit("unequal batches accepted")
except ValueError as e:
    assert "same local batch size" in str(e)
with tf.GradientTape() as tape:
    loss, l2 = model(np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros(4, np.float32))
grads = tape.gradient((loss, l2), model.trainable_variables)
try:
    opt.apply_gradients(list(zip(grads, model.trainable_variables))[:3])
    raise SystemExit("partial gradient set accepted")
except NotImplementedError:
    pass
dist.barrier()
print("rank ok")
"""


def test_sharded_pointwise_refusals():
    for rc, out in run_ranks(2, _ERRORS.format(root=ROOT), "pointwise_shard_cpu errors"):
        assert rc == 0 and "rank ok" in out, out


def test_restatements():
    """tests/pointwise_shard_np against the kernels' contracts written out sample by sample."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from pointwise_shard_np import grad_rows_np, serve_np, shard_lookups_np
    rng = np.random.default_rng(2)
    U, I = 7, 5
    uid, iid = rng.integers(-2, U + 3, 60), rng.integers(-2, I + 3, 60)
    lk = shard_lookups_np(uid, iid, U, I)
    for t in range(60):
        good = 0 <= uid[t] < U and 0 <= iid[t] < I
        assert lk[t].tolist() == ([uid[t], iid[t]] if good else [-1, -1])
    user, item, bias = rng.random((3, 4)), rng.random((2, 4)), rng.random(2)
    req = np.array([0, 2, 3, 4, 5, 6, -1, 1])       # Lu = 4: rows 4, 5 are items 0, 1; 3 and 6 belong to no table
    rows, ul, il = serve_np(user, item, bias, 3, 2, 4, req, 8)
    assert ul.tolist() == [0, 2, -1, -1, -1, -1, -1, 1] and il.tolist() == [-1, -1, -1, 0, 1, -1, -1, -1]
    np.testing.assert_allclose(rows[[0, 1, 7], :4], user[[0, 2, 1]], rtol=1e-6)
    np.testing.assert_allclose(rows[[3, 4], :4], item, rtol=1e-6)
    np.testing.assert_allclose(rows[[3, 4], 4], bias, rtol=1e-6)
    assert not rows[[2, 5, 6]].any() and not rows[:, 5:].any() and not rows[[0, 1, 7], 4].any()
    # grad rows: GMF by hand, one valid and one skipped sample, w terms on
    D = 3
    fetched = rng.random((2, D + 4))
    w = rng.random(D)
    d, gw, (loss, l2) = grad_rows_np(0, fetched, D, np.array([0, 1, -1, -1]), np.array([1.0, 0.0]), w, 0.5,
                                     c_loss=2.0, c_l2=0.3, add_w_terms=True)
    u, it, bi = fetched[0, :D], fetched[1, :D], fetched[1, D]
    z = (u * w * it).sum() + bi
    g = 2.0 * (1 / (1 + np.exp(-z)) - 1.0) * 0.5
    np.testing.assert_allclose(d[0, :D], g * w * it + 0.3 * u)
    np.testing.assert_allclose(d[1, :D], g * w * u + 0.3 * it)
    np.testing.assert_allclose(d[1, D], g)
    assert not d[2:].any() and not d[0, D:].any() and not d[1, D + 1:].any()
    np.testing.assert_allclose(gw, g * u * it + 0.3 * w)
    np.testing.assert_allclose(loss, (max(z, 0) - z + np.log1p(np.exp(-abs(z)))) * 0.5)
    np.testing.assert_allclose(l2, 0.5 * ((u * u).sum() + (it * it).sum() + (w * w).sum()))
