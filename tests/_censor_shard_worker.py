"""Worker of tests/test_gpu_censor_shard.py: one rank of a world_size-R NCCL job (one process per GPU).  Trains ShardedUCML
with UCML's loop (GradientTape, Adagrad, then censor_vec) for three steps; rank 0 trains UCML from the same initial
tables on the global batch (every rank's triplets, concatenated) and compares losses and tables.  Then
item_latent_factor.censor with a different number of ids per rank against UCML's item_latent_factor.censor of all of
them."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]


def gather(t, total, world, rank):
    """The global table from every rank's shard (row r = local row r // world of rank r % world)."""
    per = (total + world - 1) // world
    own = (total - rank + world - 1) // world
    pad = torch.zeros(per, t.shape[1], device=t.device)
    pad[:own] = t[:own]
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.stack(parts, 1).reshape(per * world, -1)[:total].cpu().numpy()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import tensorflow as tf
    from openrec.tf2.recommenders import UCML, ShardedUCML
    rng = np.random.default_rng(8)                              # the same draws on every rank
    U, I, D, B = 1201, 3001, 64, 512
    model = ShardedUCML(D, D, U, I, seed=5)
    for v in model.variables[:2]:                               # rows in +-0.4, so that the censor has work
        v.t.mul_(8.0)
    init = [gather(v.t, n, world, rank) for v, n in zip(model.variables, (U, I, I))]
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    ref = ref_opt = None
    if rank == 0:
        ref = UCML(D, D, U, I)
        for v, t in zip(ref.trainable_variables, init):
            v.assign(t)
        ref_opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    for _ in range(3):
        ids = [rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
        ids[2][:B // 4] = ids[1][B // 4:B // 2]                 # items in both p and n
        with tf.GradientTape() as tape:
            out = model(*[a[rank * B:(rank + 1) * B] for a in ids])
        grads = tape.gradient(out, model.trainable_variables)
        opt.apply_gradients(zip(grads, model.trainable_variables))
        model.censor_vec(*[a[rank * B:(rank + 1) * B] for a in ids])
        loss = [float(x) for x in out]
        if rank == 0:
            with tf.GradientTape() as tape:
                want = ref(*ids)
            g = tape.gradient(want, ref.trainable_variables)
            ref_opt.apply_gradients(zip(g, ref.trainable_variables))
            ref.censor_vec(*ids)
            np.testing.assert_allclose(loss, [float(x) for x in want], rtol=1e-5)
    model.check()
    counts = [100 + 37 * r for r in range(world)]
    cids = rng.integers(-3, I + 3, sum(counts)).astype(np.int32)
    off = sum(counts[:rank])
    model.item_latent_factor.censor(cids[off:off + counts[rank]])
    got = [gather(v.t, n, world, rank) for v, n in zip(model.variables, (U, I, I))]
    if rank == 0:
        valid = cids[(cids >= 0) & (cids < I)]
        ref.item_latent_factor.censor(valid)
        for a, v, name in zip(got, ref.trainable_variables, ("user", "item", "bias")):
            np.testing.assert_allclose(a, v.t.cpu().numpy(), atol=1e-6, err_msg=name)
        norms = np.linalg.norm(got[1][np.unique(valid)], axis=1)
        assert np.abs(norms - 1).max() < 1e-5                   # censored rows lie on the unit sphere
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("censor ok")


if __name__ == "__main__":
    main()
