"""Row-sharded GMF benchmark: GMF with its user table (1M rows), item table (1M x N rows) and item bias row-sharded over N
GPUs, D = 128, B = 65 536 samples PER RANK (weak scaling).  Prints one JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N bench_pointwise_sharded.py [--window 1.0] [--zipf A]

A step is ShardedGMF + tf.GradientTape + Adagrad.apply_gradients (the reference example's train_step).  Ids are uniform,
or Zipf(A) clipped to the table with --zipf.  Reported: global samples/s and ms/step of the slowest rank (CUDA events
over a window of at least --window seconds), a per-phase split of the step (CUDA events between the phases of
openrec_b200.sharded.pointwise_step_sharded over a few extra steps), the unique rows and exchange bytes per rank per
step, and the card name and power limit read in the same run.  At N = 1, before timing, one step is checked against the
single-GPU GMF step from the same tables and w (a mismatch exits non-zero), and then the plain GMF step on the same
tables is timed in alternation with the sharded one.  Nothing is written to disk."""
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
from openrec_b200.sharded import pointwise_step_sharded  # noqa: E402

U, I_PER_GPU, D, B, LR = 1_000_000, 1_000_000, 128, 65_536, 0.05
PHASES = ["bucket", "counts", "ids", "owner_serve", "rows", "grad_rows", "segment_sum", "grad_xchg", "owner_apply",
          "dense_allreduce"]


def batches(rng, zipf, I, n=4):
    out = []
    for _ in range(n):
        if zipf:
            u, i = np.minimum(rng.zipf(zipf, B) - 1, U - 1), np.minimum(rng.zipf(zipf, B) - 1, I - 1)
        else:
            u, i = rng.integers(0, U, B), rng.integers(0, I, B)
        out.append((torch.from_numpy(u.astype(np.int32)).cuda(), torch.from_numpy(i.astype(np.int32)).cuda(),
                    torch.from_numpy((rng.random(B) < 0.25).astype(np.float32)).cuda()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    ap.add_argument("--zipf", type=float, default=0.0, help="Zipf exponent of the ids (0: uniform)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pointwise_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
    import tensorflow as tf
    from openrec.tf2.recommenders import GMF, ShardedGMF
    I = I_PER_GPU * world
    model = ShardedGMF(D, D, U, I, seed=1)
    opt = tf.keras.optimizers.Adagrad(learning_rate=LR)
    data = batches(np.random.default_rng(100 + rank), args.zipf, I)

    def make_step(m, o):
        def train_step(u, i, y):
            with tf.GradientTape() as tape:
                loss, l2 = m(u, i, y)
            g = tape.gradient((loss, l2), m.trainable_variables)
            o.apply_gradients(zip(g, m.trainable_variables))
            return loss
        return train_step

    sharded_step = make_step(model, opt)
    plain = None
    check = None
    if world == 1:                   # the single-GPU GMF on the same tables and w, checked on one step
        plain = GMF(D, D, U, I)
        for a, b in zip(model.trainable_variables, plain.trainable_variables):
            b.t.copy_(a.t)
        popt = tf.keras.optimizers.Adagrad(learning_rate=LR)
        plain_step = make_step(plain, popt)
        ls, lp = float(sharded_step(*data[0]).numpy()), float(plain_step(*data[0]).numpy())
        uid, iid = data[0][0].long(), data[0][1].long()
        va, vb = model.trainable_variables, plain.trainable_variables
        diffs = [float((va[0].t[uid] - vb[0].t[uid]).abs().max()), float((va[1].t[iid] - vb[1].t[iid]).abs().max()),
                 float((va[2].t[iid] - vb[2].t[iid]).abs().max()), float((va[3].t - vb[3].t).abs().max())]
        check = {"loss_sharded": ls, "loss_plain": lp, "max_abs_diff_user_item_bias_w": diffs,
                 "passed": abs(ls - lp) <= 1e-5 * max(1.0, abs(lp)) and max(diffs) <= 1e-5}
        if not check["passed"]:
            print(json.dumps({"error": "the sharded step does not match the single-GPU GMF step", "check": check}))
            sys.exit(1)
    cnt = {"k": 0}

    def run_sharded():
        sharded_step(*data[cnt["k"] % 4])
        cnt["k"] += 1

    def run_plain():
        plain_step(*data[cnt["k"] % 4])
        cnt["k"] += 1

    for _ in range(3):
        run_sharded()
        if plain is not None:
            run_plain()
    ms, ms_plain = [], []
    for _ in range(2):               # alternate the two steps at N = 1
        ms.append(slowest(timed(run_sharded, args.window)))
        if plain is not None:
            torch.cuda.synchronize()
            ms_plain.append(timed(run_plain, args.window))

    # per-phase split: pointwise_step_sharded on the model's own state with CUDA events between the phases
    part = model._part(opt)
    sums = {p: 0.0 for p in PHASES}
    n_ph = 5
    for i in range(n_ph):
        ev = [torch.cuda.Event(enable_timing=True)]
        ev[0].record()

        def timer(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.append(e)
        opt.iterations += 1
        o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, opt.iterations)
        pointwise_step_sharded([part], model._xchg, [data[i % 4]], o, timer=timer)
        torch.cuda.synchronize()
        for name, a, b in zip(PHASES, ev[:-1], ev[1:]):
            sums[name] += a.elapsed_time(b) / n_ph
    uniq, served = part.last["uniq"], part.last["served"]
    phase_ms = {k: slowest(v) for k, v in sums.items()}
    row_bytes = part.W * 4
    exchange = {"ids_bytes_sent": 4 * uniq, "ids_bytes_received": 4 * served,
                "rows_bytes_received": row_bytes * uniq, "rows_bytes_sent": row_bytes * served,
                "grad_rows_bytes_sent": row_bytes * uniq, "grad_rows_bytes_received": row_bytes * served,
                "allreduce_bytes": 4 * (D + 2)}
    name, watts = card()
    best = min(ms)
    line = {"metric": "gmf_sharded_samples_per_sec", "value": world * B / (best * 1e-3), "unit": "samples/s",
            "gpus": world, "ms_per_step_slowest_rank": best, "ms_per_step_windows": ms, "per_rank_batch": B,
            "tables": f"user {U} x {D}, item {I} x {D}", "ids": f"zipf({args.zipf})" if args.zipf else "uniform",
            "optimizer": f"Adagrad lr {LR}", "phase_ms_slowest_rank": phase_ms, "unique_rows_per_rank_step": uniq,
            "lookups_per_rank_step": 2 * B, "exchange_per_rank_step": exchange, "card": name, "power_limit_w": watts,
            "check": check}
    if plain is not None:
        line["single_gpu_gmf_ms_per_step_windows"] = ms_plain
        line["ratio_vs_single_gpu"] = best / min(ms_plain)
    if rank == 0:
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
