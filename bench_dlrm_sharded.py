"""Row-sharded DLRM benchmark: bench.py's DLRM workload (26 tables x 1M rows x 128, the same MLPs, interaction_mode='dlrm',
Adagrad) with the tables row-sharded over N GPUs and B = 32 768 samples PER RANK (weak scaling).  Prints one JSON line
from rank 0.

    python -m torch.distributed.run --nproc-per-node N bench_dlrm_sharded.py [--window 1.0] [--zipf A]

A step is ShardedDLRM + tf.GradientTape + Adagrad.apply_gradients (the reference example's train_step).  Ids are uniform
per table, or Zipf(A) clipped to the vocabulary with --zipf.  Reported: global samples/s and ms/step of the slowest rank
(CUDA events over a window of at least --window seconds), a per-phase split of the step (CUDA events between the phases
of openrec_b200.sharded.dlrm_step_sharded over a few extra steps), the unique rows and exchange bytes per rank per step,
and the card name and power limit read in the same run.  At N = 1, before timing, one step is checked against the
single-GPU DLRM step from the same tables and weights (a mismatch exits non-zero), and then the plain DLRM step on the
same tables is timed in alternation with the sharded one.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")]
from bench import D, DLRM_B, DLRM_BOT, DLRM_DENSE, DLRM_LR, DLRM_T, DLRM_TOP, DLRM_VOCAB  # noqa: E402
from bench_eval import card  # noqa: E402
from bench_eval_sharded import slowest, timed  # noqa: E402
from openrec_b200.sharded import dlrm_step_sharded  # noqa: E402

PHASES = ["bucket", "counts", "ids", "owner_serve", "rows", "fwd_bwd", "segment_sum", "grad_xchg", "owner_apply",
          "dense_allreduce"]


def batches(rng, zipf, n=4):
    out = []
    for _ in range(n):
        if zipf:
            sparse = np.minimum(rng.zipf(zipf, (DLRM_B, DLRM_T)) - 1, DLRM_VOCAB - 1)
        else:
            sparse = rng.integers(0, DLRM_VOCAB, (DLRM_B, DLRM_T))
        out.append((torch.from_numpy(np.log1p(rng.integers(0, 100, (DLRM_B, DLRM_DENSE))).astype(np.float32)).cuda(),
                    torch.from_numpy(sparse.astype(np.int32)).cuda(),
                    torch.from_numpy((rng.random(DLRM_B) < 0.25).astype(np.float32)).cuda()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    ap.add_argument("--zipf", type=float, default=0.0, help="Zipf exponent of the ids (0: uniform)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dlrm_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM, ShardedDLRM
    vocab = [DLRM_VOCAB] * DLRM_T
    model = ShardedDLRM(m_spa=D, ln_emb=vocab, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm", seed=1)
    model._build(DLRM_DENSE)
    opt = tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)
    data = batches(np.random.default_rng(100 + rank), args.zipf)

    def make_step(m, o):
        def train_step(d, s, y):
            with tf.GradientTape() as tape:
                loss = m(d, s, y)
            g = tape.gradient(loss, m.trainable_variables)
            o.apply_gradients(zip(g, m.trainable_variables))
            return loss
        return train_step

    sharded_step = make_step(model, opt)
    plain = None
    check = None
    if world == 1:                   # the single-GPU DLRM on the same tables and weights, checked on one step
        plain = DLRM(m_spa=D, ln_emb=vocab, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm")
        plain._graph(DLRM_DENSE)
        for k, lf in enumerate(plain._latent_factors):
            lf.embeddings.t.copy_(model.embedding_shard.t[k * DLRM_VOCAB:(k + 1) * DLRM_VOCAB])
        for a, b in zip(model.trainable_variables[1:], plain.trainable_variables[DLRM_T:]):
            b.t.copy_(a.t)
        popt = tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)
        plain_step = make_step(plain, popt)
        ls, lp = float(sharded_step(*data[0]).numpy()), float(plain_step(*data[0]).numpy())
        ids = data[0][1][:, 0].long()
        drow = float((model.embedding_shard.t[ids] - plain._latent_factors[0].embeddings.t[ids]).abs().max())
        dw = max(float((a.t - b.t).abs().max()) for a, b in zip(model.trainable_variables[1:],
                                                                 plain.trainable_variables[DLRM_T:]))
        check = {"loss_sharded": ls, "loss_plain": lp, "max_abs_diff_table0_rows": drow, "max_abs_diff_dense": dw,
                 "passed": abs(ls - lp) <= 1e-5 * max(1.0, abs(lp)) and drow <= 1e-5 and dw <= 1e-5}
        if not check["passed"]:
            print(json.dumps({"error": "the sharded step does not match the single-GPU DLRM step", "check": check}))
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

    # per-phase split: dlrm_step_sharded on the model's own state with CUDA events between the phases
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
        dlrm_step_sharded([part], model._xchg, [data[i % 4]], o, timer=timer)
        torch.cuda.synchronize()
        for name, a, b in zip(PHASES, ev[:-1], ev[1:]):
            sums[name] += a.elapsed_time(b) / n_ph
    uniq, served = part.last["uniq"], part.last["served"]
    phase_ms = {k: slowest(v) for k, v in sums.items()}
    row_bytes = D * 4
    exchange = {"ids_bytes_sent": 4 * uniq, "ids_bytes_received": 4 * served,
                "rows_bytes_received": row_bytes * uniq, "rows_bytes_sent": row_bytes * served,
                "grad_rows_bytes_sent": row_bytes * uniq, "grad_rows_bytes_received": row_bytes * served,
                "dense_allreduce_bytes": 4 * (sum(v.t.numel() for v in model.trainable_variables[1:]) + 1)}
    name, watts = card()
    best = min(ms)
    line = {"metric": "dlrm_sharded_samples_per_sec", "value": world * DLRM_B / (best * 1e-3), "unit": "samples/s",
            "gpus": world, "ms_per_step_slowest_rank": best, "ms_per_step_windows": ms,
            "per_rank_batch": DLRM_B, "tables": f"{DLRM_T} x {DLRM_VOCAB} x {D}", "ids": f"zipf({args.zipf})" if args.zipf
            else "uniform", "optimizer": f"Adagrad lr {DLRM_LR}", "phase_ms_slowest_rank": phase_ms,
            "unique_rows_per_rank_step": uniq, "lookups_per_rank_step": DLRM_B * DLRM_T,
            "exchange_per_rank_step": exchange, "card": name, "power_limit_w": watts, "check": check}
    if plain is not None:
        line["single_gpu_dlrm_ms_per_step_windows"] = ms_plain
        line["overhead_vs_single_gpu"] = best / min(ms_plain) - 1.0
    if rank == 0:
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
