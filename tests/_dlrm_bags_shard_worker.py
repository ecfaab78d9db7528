"""Worker of tests/test_dlrm_bags_shard_cpu.py (gloo, the oracle-backed engine of tests/fake_engine.py) and of
tests/test_gpu_dlrm_bags_shard.py (NCCL, one process per GPU): one rank of a multi-hot ShardedDLRM job.

    python _dlrm_bags_shard_worker.py <gloo|nccl> <sgd|adagrad|adam|lazyadam> <sum|mean> <reference|dlrm>

Every rank draws the same global batches of bags (padding, ids = vocab and beyond, ragged lengths, repeated ids) and
trains on its slice for three steps through the reference example's GradientTape / apply_gradients protocol.  Every
rank also runs the float64 multi-hot oracle step (tests/dlrm_bags_np.train_step) on the whole global batch from the
same starting tables and weights, and checks the loss of every step, every table row and every Dense weight, and that
its Dense replicas equal rank 0's.  Prints 'rank ok'."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]

VOCAB = [3, 1, 40, 17, 2]          # tiny tables and one of a single row: G = 63
BAGS = [2, 1, 5, 3, 4]
D, N_DENSE, B = 4, 5, 6
BOT, TOP = [8, D], [16, 1]
LR = {"sgd": 0.1, "adagrad": 0.05, "adam": 0.01, "lazyadam": 0.01}


def gather_rows(t, G, rank, world):
    """The global [G, D] table from every rank's shard (row g = local row g // world of rank g % world)."""
    per = (G + world - 1) // world
    n = (G - rank + world - 1) // world
    pad = torch.zeros(per, t.shape[1], dtype=t.dtype, device=t.device)
    pad[:n] = t[:n]
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.stack(parts, 1).reshape(per * world, -1)[:G].cpu().numpy()


def draw_bags(rng, n):
    """[n, sum(BAGS)] bags: ragged lengths (the rest -1), ids = vocab and beyond, repeated ids."""
    cols = []
    for L, V in zip(BAGS, VOCAB):
        ids = rng.integers(0, V, (n, L))
        ids[rng.random((n, L)) < 0.1] = V + rng.integers(0, 3)
        if L > 1:
            ids[:, 1] = np.where(rng.random(n) < 0.3, ids[:, 0], ids[:, 1])
        length = rng.integers(0, L + 1, n)
        ids[np.arange(L)[None, :] >= length[:, None]] = -1
        cols.append(ids)
    return np.concatenate(cols, 1).astype(np.int32)


def main(backend, opt_name, pooling, mode):
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    if backend == "gloo":
        import dlrm_bags_shard_np
        import fake_engine
        fake_engine.install()
        dlrm_bags_shard_np.install(fake_engine.FakeEngine)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        atol = 1e-5
    else:
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        atol = 1e-4 if opt_name == "adam" else 1e-5
    import tensorflow as tf
    import dlrm_bags_np as NB
    from oracle import openrec_oracle as O
    from openrec.tf2.recommenders import ShardedDLRM
    from openrec_b200.sharded import row_offsets
    off = row_offsets(VOCAB)
    col_off = NB.col_offsets(BAGS)
    G, T = off[-1], len(VOCAB)
    model = ShardedDLRM(D, VOCAB, BOT, TOP, interaction_mode=mode, seed=1, bag_sizes=BAGS, pooling=pooling)
    model._build(N_DENSE)
    opt = {"sgd": tf.keras.optimizers.SGD, "adagrad": tf.keras.optimizers.Adagrad, "adam": tf.keras.optimizers.Adam,
           "lazyadam": tf.keras.optimizers.LazyAdam}[opt_name](learning_rate=LR[opt_name])
    kind = opt._kind
    table = gather_rows(model.embedding_shard.t, G, rank, world).astype(np.float64)
    dense_vars = model.trainable_variables[1:]
    weights = [v.numpy().astype(np.float64) for v in dense_vars]
    fill = 0.1 if opt_name == "adagrad" else 0.0
    slots = [np.full_like(table, fill), np.full_like(table, fill)]
    st = [(slots[0][off[k]:off[k + 1]], slots[1][off[k]:off[k + 1]]) for k in range(T)]
    st += [(np.full_like(w, fill), np.full_like(w, fill)) for w in weights]
    tabs = [table[off[k]:off[k + 1]] for k in range(T)]
    rng = np.random.default_rng(11)
    for step in range(1, 4):
        dense = rng.random((world * B, N_DENSE)).astype(np.float32)
        sparse = draw_bags(rng, world * B)
        label = (rng.random(world * B) < 0.5).astype(np.float32)
        mine = slice(rank * B, (rank + 1) * B)
        with tf.GradientTape() as tape:
            loss = model(dense[mine], sparse[mine], label[mine])
        grads = tape.gradient(loss, model.trainable_variables)
        opt.apply_gradients(zip(grads, model.trainable_variables))
        got = float(loss.numpy())
        want = NB.train_step(kind, tabs, weights, st, step, LR[opt_name], dense.astype(np.float64),
                             sparse.astype(np.int64), label.astype(np.float64), col_off, pooling == "mean", mode,
                             len(BOT))
        assert abs(got - want) <= atol * max(1.0, abs(want)), (step, got, want)
    got_table = gather_rows(model.embedding_shard.t, G, rank, world)
    np.testing.assert_allclose(got_table, table, atol=atol, rtol=atol)
    flat = torch.cat([v.t.reshape(-1) for v in dense_vars])
    ref = flat.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(flat, ref), "Dense replicas differ from rank 0's"
    for v, w in zip(dense_vars, weights):
        np.testing.assert_allclose(v.numpy(), w, atol=atol, rtol=atol, err_msg=v.name)
    dist.barrier()
    dist.destroy_process_group()
    print("rank ok")


if __name__ == "__main__":
    main(*sys.argv[1:5])
