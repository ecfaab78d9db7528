"""Worker of tests/test_gpu_score_rank_listed_shard.py: one rank of a world_size-R NCCL job (one process per GPU).
Trains ShardedBPR and ShardedUCML for three Adagrad steps, evaluates them with CandidateEvaluator on a dataset with
100 listed negatives per user on every rank, and on rank 0 compares with BPR / UCML holding the gathered tables
(orx_score_rank_listed on one device): AUC and Recall bit for bit, NDCG within one float32 ulp, and every rank's
results bit-identical to rank 0's."""
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
    from openrec.tf2.data import Dataset
    from openrec.tf2.metrics import CandidateEvaluator
    from openrec.tf2.recommenders import BPR, UCML, ShardedBPR, ShardedUCML
    from test_gpu_score_rank import check_equal
    rng = np.random.default_rng(5)                              # the same problem on every rank
    U, I, D, B = 1201, 16981, 64, 512
    tr, va = [], []
    for u in range(U):
        items = rng.choice(I, 45, replace=False)
        if u % 7:
            va += [(u, i) for i in items[:1 + u % 5]]
        if u % 11:
            tr += [(u, i) for i in items[5:5 + int(rng.integers(1, 41))]]

    def mk(pairs, **kw):
        raw = np.empty(len(pairs), dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = np.array(pairs).T
        return Dataset(raw_data=raw, total_users=U, total_items=I, **kw)
    np.random.seed(3)                                           # the Dataset's negative draw, the same on every rank
    train, val = mk(tr), mk(va, num_negatives=100)
    at = [10, 50]
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
        ev = CandidateEvaluator(val, excl_datasets=[train], at=at, batch_size=300)
        res = ev.evaluate(model)
        got = [res[k].numpy() for k in ("AUC", "NDCG", "Recall")]
        assert len(got[0]) == len(ev.warm_users) > 300
        everyone = [None] * world
        dist.all_gather_object(everyone, got)
        tables = [t.cpu().numpy() for t in model._impl.gather_global()]
        if rank == 0:
            for r, theirs in enumerate(everyone):
                for x, y in zip(got, theirs):
                    np.testing.assert_array_equal(x.view(np.int32), y.view(np.int32), err_msg=f"rank {r}")
            ref = cls(D, D, U, I)
            for v, t in zip(ref.trainable_variables, tables):
                v.assign(t)
            res_ref = CandidateEvaluator(val, excl_datasets=[train], at=at, batch_size=300).evaluate(ref)
            check_equal([torch.from_numpy(x) for x in got],
                        [torch.from_numpy(res_ref[k].numpy()) for k in ("AUC", "NDCG", "Recall")], cls.__name__)
            assert 0.3 < np.nanmean(got[0]) < 0.7, np.nanmean(got[0])
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("evaluation ok")


if __name__ == "__main__":
    main()
