"""Worker of tests/test_gpu_score_topk_shard.py: one rank of a world_size-R NCCL job (one process per GPU).  Trains
ShardedBPR and ShardedUCML for three Adagrad steps, calls Retriever.recommend on every rank, and on rank 0 compares with
Retriever on BPR / UCML holding the gathered tables (orx_score_topk on one device): items equal, scores bit for bit, and
every rank's result bit-identical to rank 0's."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import tensorflow as tf
    from openrec.tf2.recommenders import BPR, UCML, Retriever, ShardedBPR, ShardedUCML
    from _score_rank_shard_worker import datasets
    rng = np.random.default_rng(5)                              # the same problem on every rank
    U, I, D, B = 1201, 16981, 64, 512
    train, _ = datasets(rng, U, I)
    users = np.concatenate([np.arange(U), [0, 5, U - 1]]).astype(np.int64)   # every user, some twice
    for sharded_cls, cls in ((ShardedBPR, BPR), (ShardedUCML, UCML)):
        model = sharded_cls(D, D, U, I, seed=3)
        opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
        for _ in range(3):
            ids = [rng.integers(0, n, B * world).astype(np.int32)[rank * B:(rank + 1) * B] for n in (U, I, I)]
            with tf.GradientTape() as tape:
                out = model(*ids)
            grads = tape.gradient(out, model.trainable_variables)
            opt.apply_gradients(zip(grads, model.trainable_variables))
        model.check()
        for k in (10, 100):
            ret = Retriever(excl_datasets=[train], k=k, batch_size=500)
            items, scores = ret.recommend(model, users)
            got = [items.numpy(), scores.numpy().view(np.int32)]
            assert got[0].shape == (len(users), k)
            everyone = [None] * world
            dist.all_gather_object(everyone, got)
            tables = [t.cpu().numpy() for t in model._impl.gather_global()]
            if rank == 0:
                for r, theirs in enumerate(everyone):
                    for x, y in zip(got, theirs):
                        np.testing.assert_array_equal(x, y, err_msg=f"rank {r}")
                ref = cls(D, D, U, I)
                for v, t in zip(ref.trainable_variables, tables):
                    v.assign(t)
                want_items, want_scores = Retriever(excl_datasets=[train], k=k, batch_size=500).recommend(ref, users)
                np.testing.assert_array_equal(got[0], want_items.numpy(), err_msg=f"{cls.__name__} k={k}")
                np.testing.assert_array_equal(got[1], want_scores.numpy().view(np.int32), err_msg=cls.__name__)
                seen = {u: set(train.datastore.get_positive_items(u)) for u in range(50)}
                assert all(not seen[u] & set(got[0][u].tolist()) for u in range(50))
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("retrieval ok")


if __name__ == "__main__":
    main()
