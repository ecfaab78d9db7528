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
same tables is timed in alternation with the sharded one.  Nothing is written to disk.

    ... bench_dlrm_sharded.py --bags mlperf [--ragged]

runs the multi-hot model instead: ShardedDLRM(bag_sizes=...) with the MLPerf DLRM-DCNv2 bag sizes of
bench_dlrm_multihot.py (214 ids per sample), full bags pooled by a sum, or with --ragged bag lengths uniform in 1 .. L_k
pooled by a mean.  At N = 1 the single-GPU DLRM(bag_sizes) is checked and timed against it in the same way.  Its line
adds the unique rows against the valid lookups; orx_bag_segment_sum's kernel time, the least bytes it must move (every
pooled gradient row read once, its index and offset arrays, its output rows, and for a mean the slot block and the bag
counts) over that time, and that against the H100 SXM data-sheet HBM3 figure (3.35 TB/s); the bytes its lookups request
(one gradient row per valid lookup, most of them L2 hits); and the device memory in use after the timed and per-phase
steps.  That stands in for the peak: torch's caching allocator is never emptied and liborx's scratch buffers only grow,
so both still hold their high-water marks."""
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
from bench_dlrm_multihot import BAGS, HBM_GBS, draw, make_step  # noqa: E402
from bench_eval_sharded import slowest, timed  # noqa: E402
from openrec_b200 import native as N  # noqa: E402
from openrec_b200.sharded import dlrm_step_sharded  # noqa: E402

PHASE_STEPS = 5   # steps of the per-phase split; part.last then describes batch data[(PHASE_STEPS - 1) % 4]
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
    ap.add_argument("--bags", choices=["mlperf"], default=None, help="multi-hot features with the MLPerf bag sizes")
    ap.add_argument("--ragged", action="store_true", help="with --bags: ragged bags pooled by a mean")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dlrm_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world,
                            device_id=torch.device("cuda", torch.cuda.current_device()))
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM, ShardedDLRM
    vocab = [DLRM_VOCAB] * DLRM_T
    kw = dict(m_spa=D, ln_emb=vocab, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm")
    rng = np.random.default_rng(100 + rank)
    if args.bags:
        pooling = "mean" if args.ragged else "sum"
        kw.update(bag_sizes=BAGS, pooling=pooling)
        data, col_off = draw(rng, args.ragged)
        checked, row_key = (0, 20), "max_abs_diff_rows_tables_0_20"     # a 3-id and the 100-id table
    else:
        data, col_off = batches(rng, args.zipf), list(range(DLRM_T + 1))
        checked, row_key = (0,), "max_abs_diff_table0_rows"
    model = ShardedDLRM(**kw, seed=1)
    model._build(DLRM_DENSE)
    opt = tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)
    sharded_step = make_step(tf, model, opt)
    plain = None
    check = None
    if world == 1:                   # the single-GPU DLRM on the same tables and weights, checked on one step
        plain = DLRM(**kw)
        plain._graph(DLRM_DENSE)
        for k, lf in enumerate(plain._latent_factors):
            lf.embeddings.t.copy_(model.embedding_shard.t[k * DLRM_VOCAB:(k + 1) * DLRM_VOCAB])
        for a, b in zip(model.trainable_variables[1:], plain.trainable_variables[DLRM_T:]):
            b.t.copy_(a.t)
        plain_step = make_step(tf, plain, tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR))
        ls, lp = float(sharded_step(*data[0]).numpy()), float(plain_step(*data[0]).numpy())
        drow = 0.0
        for k in checked:            # the rows the step touched
            ids = data[0][1][:, col_off[k]:col_off[k + 1]]
            ids = ids[ids >= 0].long()
            drow = max(drow, float((model.embedding_shard.t[k * DLRM_VOCAB + ids]
                                    - plain._latent_factors[k].embeddings.t[ids]).abs().max()))
        dw = max(float((a.t - b.t).abs().max()) for a, b in zip(model.trainable_variables[1:],
                                                                 plain.trainable_variables[DLRM_T:]))
        check = {"loss_sharded": ls, "loss_plain": lp, row_key: drow, "max_abs_diff_dense": dw,
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

    part = model._part(opt)
    phase_ms = phase_split(part, model._xchg, opt, data)
    uniq, served = part.last["uniq"], part.last["served"]
    row_bytes = D * 4
    exchange = {"ids_bytes_sent": 4 * uniq, "ids_bytes_received": 4 * served,
                "rows_bytes_received": row_bytes * uniq, "rows_bytes_sent": row_bytes * served,
                "grad_rows_bytes_sent": row_bytes * uniq, "grad_rows_bytes_received": row_bytes * served,
                "dense_allreduce_bytes": 4 * (sum(v.t.numel() for v in model.trainable_variables[1:]) + 1)}
    name, watts = card()
    best = min(ms)
    if args.bags:
        line = {"metric": "dlrm_sharded_multihot_samples_per_sec"}
        ids = "ragged, lengths uniform in 1 .. L" if args.ragged else "full bags, uniform ids"
    else:
        line = {"metric": "dlrm_sharded_samples_per_sec"}
        ids = f"zipf({args.zipf})" if args.zipf else "uniform"
    line.update({"value": world * DLRM_B / (best * 1e-3), "unit": "samples/s",
                 "gpus": world, "ms_per_step_slowest_rank": best, "ms_per_step_windows": ms,
                 "per_rank_batch": DLRM_B, "tables": f"{DLRM_T} x {DLRM_VOCAB} x {D}", "ids": ids,
                 "optimizer": f"Adagrad lr {DLRM_LR}", "phase_ms_slowest_rank": phase_ms,
                 "unique_rows_per_rank_step": uniq, "lookups_per_rank_step": DLRM_B * int(col_off[-1]),
                 "exchange_per_rank_step": exchange})
    if args.bags:
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()       # before segment_sum_time's own buffers
        reserved = torch.cuda.max_memory_reserved()
        seg = segment_sum_time(N.engine(), part, data[(PHASE_STEPS - 1) % len(data)], args.window)   # part.last's batch
        line.update({"bag_sizes": BAGS, "pooling": kw["pooling"],
                     "valid_lookups_per_rank_step": seg["valid_lookups"], **{k: v for k, v in seg.items()
                                                                             if k != "valid_lookups"},
                     "hbm_peak_gbs_datasheet": HBM_GBS,
                     "device_memory_in_use_after_steps_gb": (total - free) / 1e9, "device_memory_total_gb": total / 1e9,
                     "torch_max_reserved_gb": reserved / 1e9})
    line.update({"card": name, "power_limit_w": watts, "check": check})
    if plain is not None:
        line["single_gpu_dlrm_ms_per_step_windows"] = ms_plain
        line["overhead_vs_single_gpu"] = best / min(ms_plain) - 1.0
    if rank == 0:
        print(json.dumps(line))
    dist.barrier()
    dist.destroy_process_group()

def phase_split(part, xchg, opt, data, n_ph=PHASE_STEPS):
    """ms per phase of dlrm_step_sharded on the model's own state, CUDA events between the phases, averaged over n_ph
    steps on data[0], data[1], ..., the slowest rank's."""
    sums = {p: 0.0 for p in PHASES}
    for i in range(n_ph):
        ev = [torch.cuda.Event(enable_timing=True)]
        ev[0].record()

        def timer(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.append(e)
        opt.iterations += 1
        o = (opt._kind, opt.learning_rate, opt.epsilon, opt.beta_1, opt.beta_2, opt.iterations)
        dlrm_step_sharded([part], xchg, [data[i % len(data)]], o, timer=timer)
        torch.cuda.synchronize()
        for name, a, b in zip(PHASES, ev[:-1], ev[1:]):
            sums[name] += a.elapsed_time(b) / n_ph
    return {k: slowest(v) for k, v in sums.items()}


def segment_sum_time(eng, part, batch, window):
    """orx_bag_segment_sum alone on this rank's bucket of one batch -> its kernel time, and bytes over that time.

    The least bytes it must move: every pooled gradient row that has a valid lookup, read once; the grp_idx entry of
    every valid lookup; the grp_off entry and the output row of every unique row; for a mean also the slot block, the
    bag counts written and each read once.  The request bytes count one gradient row per valid lookup instead: a row is
    requested by every lookup of its bag, and most of those repeats are L2 hits (at N = 1 the unique rows are folded in
    global-row order, one table's 16.8 MB dZ slice at a time), so they are no measure of HBM traffic."""
    _, sp, _ = batch
    B, T, D = sp.shape[0], part.T, part.D
    rows = eng.bag_shard_lookups(sp, part.col_off, part.row_off)
    bk = eng.lookup_bucket(rows.view(-1, 1), [0, part.G], part.world)
    n_uniq = int(bk[0].sum())
    hit = bk[2].view(B, -1) >= 0
    valid = int(hit.sum())
    bags_read = sum(int(hit[:, part.col_off[k]:part.col_off[k + 1]].any(1).sum()) for k in range(T))
    dZ = torch.randn(B, T, D, device="cuda") * 1e-3
    out = torch.empty(n_uniq, D, device="cuda")
    ms = timed(lambda: eng.bag_segment_sum(dZ, part.col_off, part.pooling, bk[2], bk[3], bk[4], n_uniq, out), window)
    rest = 4 * valid + 4 * (n_uniq + 1) + 4 * D * n_uniq
    if part.pooling:
        rest += 4 * sp.numel() + 4 * B * T + 4 * bags_read
    least, requested = 4 * D * bags_read + rest, 4 * D * valid + rest
    gbs = least / (ms * 1e-3) / 1e9
    return {"valid_lookups": valid, "bag_segment_sum_ms": ms, "bag_segment_sum_least_bytes": least,
            "bag_segment_sum_gbs": gbs, "bag_segment_sum_share_of_hbm_peak": gbs / HBM_GBS,
            "bag_segment_sum_request_bytes_incl_l2_hits": requested}

if __name__ == "__main__":
    main()
