"""CPU, world size 2 and 3 over gloo: ShardedDLRM through the reference example's step protocol reproduces the oracle's
single-process DLRM step on the concatenated global batch for three steps (losses, every table row, every Dense weight;
tests/_dlrm_shard_worker.py), with the oracle-backed engine of tests/fake_engine.py and the numpy restatements of tests/dlrm_shard_np.py.  This checks the layout, the
exchanges and the step's arithmetic plan; the kernels are checked in tests/test_gpu_dlrm_shard.py.  Also: the numpy
restatement of orx_lookup_bucket against a direct definition, and the argument checks."""
import os
import sys

import numpy as np
import pytest
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_dlrm_shard_worker.py")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("opt,mode,loss", [("adagrad", "dlrm", "mse"), ("adam", "reference", "bce"),
                                           ("sgd", "dlrm", "bce"), ("lazyadam", "dlrm", "mse")])
def test_sharded_dlrm_equals_oracle(world, opt, mode, loss):
    for rc, out in run_ranks(world, [WORKER, "gloo", opt, mode, loss], f"dlrm_shard_cpu {opt} {mode} {loss}"):
        assert rc == 0 and "rank ok" in out, out


_ERRORS = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
import dlrm_shard_np, fake_engine
fake_engine.install()
dlrm_shard_np.install(fake_engine.FakeEngine)
dist.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
from openrec.tf2.recommenders import ShardedDLRM
import tensorflow as tf
rank = dist.get_rank()
try:
    ShardedDLRM(4, [2 ** 30, 2 ** 30], [8, 4], [8, 1])
    raise SystemExit("G >= 2^31 accepted")
except ValueError:
    pass
model = ShardedDLRM(4, [5, 7, 3], [8, 4], [8, 1])
try:
    model(np.zeros((4, 3), np.float32), np.zeros((4, 2), np.int32), np.zeros(4, np.float32))
    raise SystemExit("sparse width != T accepted")
except ValueError:
    pass
B = 4 + rank                                   # unequal local batches: every rank raises
opt = tf.keras.optimizers.Adagrad(0.05)
with tf.GradientTape() as tape:
    loss = model(np.zeros((B, 3), np.float32), np.zeros((B, 3), np.int32), np.zeros(B, np.float32))
grads = tape.gradient(loss, model.trainable_variables)
try:
    opt.apply_gradients(zip(grads, model.trainable_variables))
    raise SystemExit("unequal batches accepted")
except ValueError as e:
    assert "same local batch size" in str(e)
dist.barrier()
print("rank ok")
"""


def test_sharded_dlrm_refusals():
    for rc, out in run_ranks(2, _ERRORS.format(root=ROOT), "dlrm_shard_cpu errors"):
        assert rc == 0 and "rank ok" in out, out


def test_lookup_bucket_restatement():
    """tests/dlrm_shard_np.lookup_bucket_np against the contract written out lookup by lookup."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dlrm_shard_np import lookup_bucket_np
    rng = np.random.default_rng(3)
    vocab = [3, 1, 50, 0, 9]
    off = np.concatenate([[0], np.cumsum(vocab)])
    sparse = np.stack([rng.integers(-2, v + 3, 40) for v in vocab], 1)
    for R in (1, 2, 3, 8, 64):
        counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(sparse, off, R)
        rows = {}
        for i, idv in enumerate(sparse.reshape(-1)):
            k = i % len(vocab)
            if 0 <= idv < vocab[k]:
                rows.setdefault(int(off[k] + idv), []).append(i)
        order = sorted(rows, key=lambda g: (g % R, g // R))
        assert counts.tolist() == [sum(1 for g in order if g % R == r) for r in range(R)]
        assert send_local.tolist() == [g // R for g in order]
        want_slot = np.full(sparse.size, -1)
        for j, g in enumerate(order):
            want_slot[rows[g]] = j
            assert grp_idx[grp_off[j]:grp_off[j + 1]].tolist() == rows[g]
        assert slot.tolist() == want_slot.tolist()
        assert grp_off[len(order)] == sum(len(v) for v in rows.values())
