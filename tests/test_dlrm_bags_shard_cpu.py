"""CPU, world size 2 and 3 over gloo: a multi-hot ShardedDLRM(bag_sizes, pooling) through the reference example's step
protocol reproduces the float64 multi-hot oracle step (tests/dlrm_bags_np.train_step) on the concatenated global batch
for three steps (losses, every table row, every Dense weight; tests/_dlrm_bags_shard_worker.py), with the oracle-backed
engine of tests/fake_engine.py and the numpy restatements of tests/dlrm_bags_shard_np.py.  This checks the layout, the
exchanges and the step's arithmetic plan; the kernels are checked in tests/test_gpu_dlrm_bags_shard.py.  Also: the
restatements against a direct definition, and the constructor refusals."""
import os
import sys

import numpy as np
import pytest
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_dlrm_bags_shard_worker.py")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("opt,pooling,mode", [("adagrad", "sum", "dlrm"), ("adam", "mean", "reference"),
                                              ("sgd", "mean", "dlrm"), ("lazyadam", "sum", "dlrm")])
def test_sharded_bags_equal_oracle(world, opt, pooling, mode):
    salt = f"dlrm_bags_shard_cpu {opt} {pooling} {mode}"
    for rc, out in run_ranks(world, [WORKER, "gloo", opt, pooling, mode], salt):
        assert rc == 0 and "rank ok" in out, out


_ERRORS = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
import dlrm_bags_shard_np, fake_engine
fake_engine.install()
dlrm_bags_shard_np.install(fake_engine.FakeEngine)
dist.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
from openrec.tf2.recommenders import ShardedDLRM
import tensorflow as tf
rank = dist.get_rank()
kw = dict(m_spa=8, ln_emb=[10, 20], ln_bot=[8, 8], ln_top=[4, 1])
for bad in (dict(bag_sizes=[1]), dict(bag_sizes=[2, 0]), dict(bag_sizes=[1, -3]), dict(bag_sizes=[1, 1], pooling="max"),
            dict(pooling="sqrtn"), dict(bag_sizes=[1] * 64, ln_emb=[10] * 64)):
    try:
        ShardedDLRM(**dict(kw, **bad))
        raise SystemExit(f"{{bad}} accepted")
    except ValueError:
        pass
model = ShardedDLRM(**kw, bag_sizes=[3, 2], pooling="mean")
for width in (2, 4, 6):
    try:
        model(np.zeros((4, 3), np.float32), np.zeros((4, width), np.int32), np.zeros(4, np.float32))
        raise SystemExit(f"sparse width {{width}} != 5 accepted")
    except ValueError:
        pass
B = 4 + rank                                   # unequal local batches: every rank raises, naming B, not B * C
opt = tf.keras.optimizers.Adagrad(0.05)
with tf.GradientTape() as tape:
    loss = model(np.zeros((B, 3), np.float32), np.zeros((B, 5), np.int32), np.zeros(B, np.float32))
grads = tape.gradient(loss, model.trainable_variables)
try:
    opt.apply_gradients(zip(grads, model.trainable_variables))
    raise SystemExit("unequal batches accepted")
except ValueError as e:
    assert "same local batch size" in str(e) and "[4, 5]" in str(e), str(e)
dist.barrier()
print("rank ok")
"""


def test_sharded_bags_refusals():
    for rc, out in run_ranks(2, _ERRORS.format(root=ROOT), "dlrm_bags_shard_cpu errors"):
        assert rc == 0 and "rank ok" in out, out


def test_restatements():
    """tests/dlrm_bags_shard_np against the contracts written out lookup by lookup: the lookups, and the fold against
    np.add.at of the IndexedSlices of tests/dlrm_bags_np.bag_slices."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dlrm_bags_np as NB
    from dlrm_bags_shard_np import bag_segment_sum_np, bag_shard_lookups_np
    from dlrm_shard_np import lookup_bucket_np
    rng = np.random.default_rng(5)
    vocab, sizes, B, D = [3, 1, 50, 9], [2, 1, 7, 4], 30, 3
    row_off, col_off = NB.col_offsets(vocab), NB.col_offsets(sizes)
    sp = np.concatenate([rng.integers(-2, V + 3, (B, L)) for L, V in zip(sizes, vocab)], 1).astype(np.int32)
    sp[0, 3:10] = -1
    rows = bag_shard_lookups_np(sp, col_off, row_off)
    for b in range(B):
        for c in range(col_off[-1]):
            k = int(np.searchsorted(col_off, c, side="right") - 1)
            idv = sp[b, c]
            assert rows[b, c] == (row_off[k] + idv if 0 <= idv < vocab[k] else -1)
    dz = rng.standard_normal((B, len(vocab), D))
    for R in (1, 3):
        _, _, slot, grp_off, grp_idx = lookup_bucket_np(rows.reshape(-1, 1), [0, row_off[-1]], R)
        uniq = np.unique(rows[rows >= 0])
        order = sorted(uniq, key=lambda g: (g % R, g // R))
        for mean in (False, True):
            got = bag_segment_sum_np(dz, col_off, mean, slot, grp_off, grp_idx, len(order), np.float64)
            ref = np.zeros((row_off[-1], D))
            for k in range(len(vocab)):
                ids, vals = NB.bag_slices(sp, col_off, k, vocab[k], dz[:, k], mean)
                np.add.at(ref, ids + row_off[k], vals)
            np.testing.assert_allclose(got, ref[order], atol=1e-12)
