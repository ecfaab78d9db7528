"""Worker of tests/test_pointwise_shard_cpu.py (gloo, the oracle-backed engine of tests/pointwise_shard_np.py) and of
tests/test_gpu_pointwise_shard.py (NCCL, one process per GPU): one rank of a ShardedGMF / ShardedWRMF job.

    python _pointwise_shard_worker.py <gloo|nccl> <gmf|wrmf|wrmf_sigmoid> <sgd|adagrad|adam|lazyadam>

Every rank draws the same global batches (repeated rows, out-of-range ids, among them an id in [U, R * ceil(U / R)))
and trains on its slice for three steps through the reference example's GradientTape / apply_gradients protocol.  Rank
0 runs the oracle's single-process step (oracle/openrec_oracle.py pointwise_train_step) on the valid samples of the
whole global batch from the same starting state -- GMF's loss stays the mean over the full global batch, as
orx_pointwise_step's is over its B -- and checks every loss, every table row, every optimizer slot and w.  Every rank
checks that its w replica equals rank 0's.  Prints 'rank ok'."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]

U, I, D, B = 11, 7, 4, 6
LR = {"sgd": 0.1, "adagrad": 0.05, "adam": 0.01, "lazyadam": 0.01}


def gather_rows(t, total, rank, world):
    """The global [total, cols] table from every rank's shard (row r = local row r // world of rank r % world)."""
    per = (total + world - 1) // world
    n = (total - rank + world - 1) // world
    pad = torch.zeros(per, t.shape[1], dtype=t.dtype, device=t.device)
    pad[:n] = t[:n]
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.stack(parts, 1).reshape(per * world, -1)[:total].cpu().numpy()


def main(backend, model_name, opt_name):
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    if backend == "gloo":
        import pointwise_shard_np
        pointwise_shard_np.install()
        dist.init_process_group("gloo", rank=rank, world_size=world)
        atol = 1e-5
    else:
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        atol = 1e-4 if opt_name == "adam" else 1e-5
    import tensorflow as tf
    from oracle import openrec_oracle as O
    from openrec.tf2.recommenders import ShardedGMF, ShardedWRMF
    gmf = model_name == "gmf"
    a, b, sig = (1.0, 1.0, False) if gmf else (1.0, 0.05, model_name == "wrmf_sigmoid")
    model = ShardedGMF(D, D, U, I, seed=1) if gmf else ShardedWRMF(D, D, U, I, a=a, b=b, seed=1)
    if sig:
        model.pointwise_mse_loss._sigmoid = True
    opt = {"sgd": tf.keras.optimizers.SGD, "adagrad": tf.keras.optimizers.Adagrad, "adam": tf.keras.optimizers.Adam,
           "lazyadam": tf.keras.optimizers.LazyAdam}[opt_name](learning_rate=LR[opt_name])
    kind = opt._kind
    vs = model.trainable_variables
    totals = (U, I, I)
    tabs = [gather_rows(v.t, n, rank, world).astype(np.float64) for v, n in zip(vs[:3], totals)]
    w = vs[3].numpy().astype(np.float64) if gmf else None
    fill = 0.1 if opt_name == "adagrad" else 0.0
    state = {k: (np.full_like(t, fill), np.full_like(t, fill)) for k, t in zip(("user", "item", "bias"), tabs)}
    if gmf:
        state["w"] = (np.full_like(w, fill), np.full_like(w, fill))
    c_loss, c_l2 = (1.0, 1.0) if opt_name == "sgd" else (1.5, 0.25)
    rng = np.random.default_rng(5)
    for step in range(1, 4):
        n = world * B
        uid = rng.integers(0, U, n).astype(np.int32)
        iid = rng.integers(0, I, n).astype(np.int32)
        uid[1], iid[4], uid[7 % n], iid[9 % n] = U, I + 2, -1, -3        # out of range: whole samples skipped
        label = (rng.random(n) < 0.5).astype(np.float32)
        mine = slice(rank * B, (rank + 1) * B)
        with tf.GradientTape() as tape:
            loss, l2 = model(uid[mine], iid[mine], label[mine])
        obj = (loss, l2) if opt_name == "sgd" else c_loss * loss + c_l2 * l2
        grads = tape.gradient(obj, model.trainable_variables)
        opt.apply_gradients(zip(grads, model.trainable_variables))
        got = (float(loss.numpy()), float(l2.numpy()))
        ok = (uid >= 0) & (uid < U) & (iid >= 0) & (iid < I)
        scale = ok.sum() / n if gmf else 1.0                             # GMF: the mean over all n samples
        want = O.pointwise_train_step("gmf" if gmf else "wrmf", *tabs, w, uid[ok], iid[ok], label[ok].astype(np.float64),
                                      kind, state, step, LR[opt_name], a, b, sig, c_loss * scale, c_l2)
        want = (float(want[0]) * scale, float(want[1]))
        for g_, w_ in zip(got, want):
            assert abs(g_ - w_) <= atol * max(1.0, abs(w_)), (step, got, want)
    for k, (v, total) in enumerate(zip(vs[:3], totals)):
        name = ("user", "item", "bias")[k]
        np.testing.assert_allclose(gather_rows(v.t, total, rank, world), tabs[k], atol=atol, rtol=atol, err_msg=name)
        for j, s in enumerate(opt.slots(v)):
            if s is not None:
                np.testing.assert_allclose(gather_rows(s, total, rank, world), state[name][j], atol=atol, rtol=atol,
                                           err_msg=f"{name} slot {j}")
    if gmf:
        wt = vs[3].t.reshape(-1)
        ref = wt.clone()
        dist.broadcast(ref, 0)
        assert torch.equal(wt, ref), "w replicas differ from rank 0's"
        np.testing.assert_allclose(vs[3].numpy(), w, atol=atol, rtol=atol, err_msg="w")
        for j, s in enumerate(opt.slots(vs[3])):
            if s is not None:
                np.testing.assert_allclose(s.cpu().numpy(), state["w"][j], atol=atol, rtol=atol, err_msg=f"w slot {j}")
    dist.barrier()
    dist.destroy_process_group()
    print("rank ok")


if __name__ == "__main__":
    main(*sys.argv[1:4])
