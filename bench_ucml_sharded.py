"""Row-sharded UCML benchmark: UCML's training loop -- the step, then censor_vec of its batch -- with the user table (1M
rows), item table (1M x N rows) and item bias row-sharded over N GPUs, D = 128, B = 65 536 triplets PER RANK (weak
scaling), uniform ids, Adagrad.  Prints one JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N bench_ucml_sharded.py [--window 1.0]

A step is ShardedUCML + tf.GradientTape + Adagrad.apply_gradients, then ShardedUCML.censor_vec.  Reported (CUDA events,
slowest rank, windows of at least --window seconds): ms/step with and without censor_vec; censor_vec alone, split into
the id all-gather and the three orx_censor_shard launches; the id bytes all-gathered per rank; the card name and power
limit read in the same run.  At N = 1, before timing, one step + censor_vec is checked against the single-GPU UCML from
the same tables (a mismatch exits non-zero); the plain UCML loop (step + three orx_censor) is then timed in alternation
with the sharded one, and orx_censor_shard against orx_censor on the same ids.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")]
from bench_eval import card  # noqa: E402
from bench_eval_sharded import slowest, timed  # noqa: E402
from openrec_b200.sharded import censor_gathered  # noqa: E402

U, I_PER_GPU, D, B, LR = 1_000_000, 1_000_000, 128, 65_536, 0.05


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ucml_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
    import tensorflow as tf
    from openrec.tf2.recommenders import UCML, ShardedUCML
    I = I_PER_GPU * world
    model = ShardedUCML(D, D, U, I, seed=1)
    opt = tf.keras.optimizers.Adagrad(learning_rate=LR)
    rng = np.random.default_rng(100 + rank)
    data = [tuple(torch.from_numpy(rng.integers(0, n, B).astype(np.int32)).cuda() for n in (U, I, I)) for _ in range(4)]

    def make_step(m, o, censor):
        def train_step(u, p, n):
            with tf.GradientTape() as tape:
                loss, l2 = m(u, p, n)
            g = tape.gradient((loss, l2), m.trainable_variables)
            o.apply_gradients(zip(g, m.trainable_variables))
            if censor:
                m.censor_vec(u, p, n)
            return loss
        return train_step

    sharded_step, sharded_nocensor = make_step(model, opt, True), make_step(model, opt, False)
    plain = check = None
    if world == 1:                   # the single-GPU UCML on the same tables, checked on one step + censor_vec
        plain = UCML(D, D, U, I)
        for a, b in zip(model.trainable_variables, plain.trainable_variables):
            b.t.copy_(a.t)
        plain_step = make_step(plain, tf.keras.optimizers.Adagrad(learning_rate=LR), True)
        ls, lp = float(sharded_step(*data[0]).numpy()), float(plain_step(*data[0]).numpy())
        u, p, n = (x.long() for x in data[0])
        it = torch.cat([p, n])
        va, vb = model.trainable_variables, plain.trainable_variables
        diffs = [float((va[0].t[u] - vb[0].t[u]).abs().max()), float((va[1].t[it] - vb[1].t[it]).abs().max()),
                 float((va[2].t[it] - vb[2].t[it]).abs().max())]
        check = {"loss_sharded": ls, "loss_plain": lp, "max_abs_diff_user_item_bias": diffs,
                 "passed": abs(ls - lp) <= 1e-5 * max(1.0, abs(lp)) and max(diffs) <= 1e-5}
        if not check["passed"]:
            print(json.dumps({"error": "step + censor_vec does not match the single-GPU UCML", "check": check}))
            sys.exit(1)
    cnt = {"k": 0}

    def runner(step):
        def run():
            step(*data[cnt["k"] % 4])
            cnt["k"] += 1
        return run

    run_sharded, run_nocensor = runner(sharded_step), runner(sharded_nocensor)
    run_plain = runner(plain_step) if plain is not None else None
    for _ in range(3):
        run_sharded()
        run_nocensor()
        if plain is not None:
            run_plain()
    ms, ms_nocensor, ms_plain = [], [], []
    for _ in range(2):               # alternate the loops
        ms.append(slowest(timed(run_sharded, args.window)))
        ms_nocensor.append(slowest(timed(run_nocensor, args.window)))
        if plain is not None:
            torch.cuda.synchronize()
            ms_plain.append(timed(run_plain, args.window))

    # censor_vec alone, split: pack + all-gather of the ids, then the three orx_censor_shard launches
    eng = model._eng
    user, item = model.user_latent_factor.embeddings.t, model.item_latent_factor.embeddings.t
    n_split, t_gather, t_launch = 50, 0.0, 0.0
    for i in range(n_split):
        u, p, n = data[i % 4]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        ids = torch.empty(world * 3 * B, dtype=torch.int32, device="cuda")
        dist.all_gather_into_tensor(ids, torch.stack([u, p, n]).reshape(-1))
        ev[1].record()
        censor_gathered(eng, user, item, U, I, world, rank, ids, B)
        ev[2].record()
        ev[2].synchronize()
        t_gather += ev[0].elapsed_time(ev[1]) / n_split
        t_launch += ev[1].elapsed_time(ev[2]) / n_split
    censor_only = slowest(timed(lambda: model.censor_vec(*data[cnt["k"] % 4]), args.window))
    split = {"censor_vec_ms": censor_only, "allgather_ms": slowest(t_gather), "three_launches_ms": slowest(t_launch)}

    kernels = None
    if world == 1:                   # orx_censor_shard against orx_censor: the same p ids on the same item table
        p = data[1][1]
        kernels = {}
        for _ in range(2):
            kernels.setdefault("orx_censor_shard_ms", []).append(
                timed(lambda: eng.censor_shard(item, I, 1, 0, p, B, B, 1), args.window))
            kernels.setdefault("orx_censor_ms", []).append(timed(lambda: eng.censor(item, p), args.window))
    name, watts = card()
    best = min(ms)
    line = {"metric": "ucml_sharded_triplets_per_sec", "value": world * B / (best * 1e-3), "unit": "triplets/s",
            "gpus": world, "ms_per_step_slowest_rank": best, "ms_per_step_windows": ms,
            "ms_per_step_without_censor_windows": ms_nocensor, "censor_vec_split_slowest_rank": split,
            "per_rank_batch": B, "tables": f"user {U} x {D}, item {I} x {D}", "ids": "uniform",
            "optimizer": f"Adagrad lr {LR}", "censor_ids_bytes_sent_per_rank": 12 * B,
            "censor_ids_bytes_received_per_rank": 12 * world * B, "card": name, "power_limit_w": watts, "check": check}
    if plain is not None:
        line["single_gpu_ucml_ms_per_step_windows"] = ms_plain
        line["ratio_vs_single_gpu"] = best / min(ms_plain)
        line["censor_kernels_ms_windows"] = kernels
    if rank == 0:
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
