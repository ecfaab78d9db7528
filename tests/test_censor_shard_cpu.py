"""CPU, world size 2 and 3 over gloo: ShardedUCML.censor_vec and the sharded tables' LatentFactor.censor are collective
calls, and after them the gathered tables equal the oracle's UCML.censor_vec / LatentFactor.censor on the gathered
tables and the concatenation of every rank's ids.  The engine is the oracle-backed one of tests/fake_engine.py with a
test-local censor_shard that restates orx_censor_shard in numpy (each rank censors the ids it owns), so this checks the
decomposition and the collective plumbing; the kernel is checked in tests/test_gpu_censor_shard.py."""
import os

import numpy as np
import pytest
import torch
from _ranks import run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _censor_shard(self, tab, total_rows, world, rank, ids, n_per_block, block_stride, n_blocks, first=0,
                  min_norm=0.1):
    """orx_censor_shard in numpy: the owned ids among the n_blocks blocks, each row once, on local row id // world."""
    from oracle import openrec_oracle as O
    a = ids.numpy().astype(np.int64)
    g = np.concatenate([np.zeros(0, np.int64)] + [a[first + b * block_stride:first + b * block_stride + n_per_block]
                                                  for b in range(n_blocks)])
    mine = g[(g >= 0) & (g < total_rows) & (g % world == rank)]
    if len(mine):
        O.censor(tab.numpy(), mine // world, min_norm)


def _gather(var, total, world, rank):
    """The global table from every rank's shard: row r = local row r // world of rank r % world."""
    import torch.distributed as dist
    t = var.t
    per = (total + world - 1) // world
    own = (total - rank + world - 1) // world
    pad = torch.zeros(per, t.shape[1])
    pad[:own] = t[:own]
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.stack(parts, 1).reshape(per * world, -1)[:total].numpy().copy()


def _valid(a, total):
    return a[(a >= 0) & (a < total)]


def _worker(world):
    import torch.distributed as dist
    import fake_engine
    from oracle import openrec_oracle as O
    fake_engine.FakeEngine.censor_shard = _censor_shard
    fake_engine.install()
    from openrec.tf2.recommenders import ShardedUCML
    rank = int(os.environ["RANK"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(11)                 # the same draws on every rank
    U, I, D, B = 17, 29, 6, 12                      # U, I not multiples of the world size; rows of norm < 0.1 grow x10
    model = ShardedUCML(D, D, U, I, seed=4)
    user0, item0 = (_gather(v, n, world, rank) for v, n in zip(model.variables[:2], (U, I)))
    for step in range(2):
        ids = [rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
        ids[2][:B // 2] = ids[1][B // 2:B]          # items in both p and n, across ranks: censored twice, p first
        ids[0][1], ids[1][2], ids[2][3] = -1, I, 2 ** 31 - 1     # out of range: skipped
        mine = [a[rank * B:(rank + 1) * B] for a in ids]
        out = model.censor_vec(*mine)
        assert out[0] is model.user_latent_factor.embeddings and out[1] is out[2] is model.item_latent_factor.embeddings
        O.ucml_censor_vec(user0, item0, _valid(ids[0], U), _valid(ids[1], I), _valid(ids[2], I))
    got = [_gather(v, n, world, rank) for v, n in zip(model.variables[:2], (U, I))]
    # one table's censor with a different number of ids per rank (rank 1 passes none)
    counts = [3 + 5 * r if r != 1 else 0 for r in range(world)]
    cids = rng.integers(-2, I + 2, sum(counts)).astype(np.int32)
    off = int(np.sum(counts[:rank]))
    ret = model.item_latent_factor.censor(cids[off:off + counts[rank]])
    assert ret is model.item_latent_factor.embeddings
    O.censor(item0, _valid(cids, I))
    got_item = _gather(model.variables[1], I, world, rank)
    if rank == 0:
        np.testing.assert_array_equal(got[0], user0)
        np.testing.assert_array_equal(got_item, item0)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_censor_equals_oracle(world):
    paths = [os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "tests")]
    code = (f"import sys; sys.path[:0] = {paths!r}\n"
            f"import test_censor_shard_cpu as t\nt._worker({world})\nprint('rank ok')\n")
    for rc, out in run_ranks(world, code, "censor_shard_cpu"):
        assert rc == 0 and "rank ok" in out, out
