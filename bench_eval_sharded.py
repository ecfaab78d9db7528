"""Sharded catalogue-evaluation benchmark: orx_score_rank_shard's four phases with an NCCL all-reduce between them, BPR
dot + item bias, one rank per GPU.  Prints one JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N bench_eval_sharded.py [--window 1.0] [--shapes 1m,8m]

Shapes: "1m" I = 1 000 000 and "8m" I = 8 000 000, D = 128, 1 024 users per call, positives ~ Poisson(20) and
exclusions ~ Poisson(100) per user (the problem generator of bench_eval.py, rows r % N of the tables on rank r).
Before timing, rank 0 checks the 1m shape against orx_score_rank on the gathered tables (AUC and Recall bit for bit,
NDCG within one float32 ulp); a mismatch exits non-zero.  A call is timed with CUDA events on every rank and the
slowest rank's time is reported, with a per-phase split (each phase's C call and the all-reduce after it).  At N = 1
the plain orx_score_rank on the same tables is timed in alternation with the phased call.  Nothing is written to
disk."""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_eval import FP32_DATASHEET_TFLOPS, card, problem  # noqa: E402
from openrec_b200 import native as N  # noqa: E402
from openrec_b200.sharded import all_reduce_sum, score_rank_sharded  # noqa: E402

SHAPES = {"1m": (1_000_000, 128, 1024), "8m": (8_000_000, 128, 1024)}
AT = (50, 100)


def slowest(ms):
    t = torch.tensor([ms], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def timed(fn, window):
    """ms per call on this rank: CUDA events around enough calls to fill `window` seconds (the count agreed by all
    ranks, so the collectives line up)."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    n = max(3, math.ceil(window * 1e3 / max(slowest(a.elapsed_time(b)), 1e-3)))
    dist.barrier()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--shapes", default="1m,8m")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
    eng = N.engine()
    name, watts = card()
    reduce = all_reduce_sum()
    out = {"metric": "sharded_eval_users_per_s", "gpu": name, "power_limit_w": watts, "gpus": world,
           "kind": "BPR dot + item bias", "at": list(AT), "shapes": []}
    for shape in args.shapes.split(","):
        I, D, Bu = SHAPES[shape]
        p = problem(np.random.default_rng(0), I, D, Bu)     # same problem on every rank; keep this rank's rows
        del p["pos_mask"], p["excl_mask"]
        g = N.rowshard(world, rank, Bu, I)
        user, item, bias = (p[k][rank::world].contiguous() for k in ("user", "item", "bias"))
        full = (p["user"], p["item"], p["bias"]) if world == 1 or shape == "1m" else None
        if world > 1 and shape != "1m":
            del p["user"], p["item"], p["bias"]
        torch.cuda.empty_cache()
        part = (eng, N.ORX_SCORE_DOT, user, item, bias, g)
        lists = (p["uid"], p["pos_off"], p["pos_items"], p["excl_off"], p["excl_items"], p["max_pos"])

        def phased():
            return score_rank_sharded([part], reduce, *lists, at=AT)[0]

        def plain():
            return eng.score_rank(N.ORX_SCORE_DOT, full[0], p["uid"], full[1], full[2], *lists[1:], at=AT)

        if shape == "1m":
            got = [t.cpu().numpy() for t in phased()]
            if rank == 0:
                want = [t.cpu().numpy() for t in plain()]
                ok = all(np.array_equal(got[k].view(np.int32), want[k].view(np.int32)) for k in (0, 2))
                try:
                    np.testing.assert_array_max_ulp(got[1], want[1], maxulp=1)
                except AssertionError:
                    ok = False
                if not ok:
                    print(json.dumps({"error": "sharded and single-device outputs differ"}), flush=True)
                    os._exit(1)
            dist.barrier()
        t_sh, t_plain = [], []
        for _ in range(2):
            t_sh.append(slowest(timed(phased, args.window)))
            if world == 1:
                t_plain.append(timed(plain, args.window))
        # per-phase split: each phase's C call, then the all-reduce of what it wrote, each between two events
        n3 = eng.score_rank_shard_sizes(Bu, D, p["max_pos"])
        bufs = (torch.empty(n3[0], dtype=torch.int32, device="cuda"), torch.empty(n3[1], dtype=torch.int32, device="cuda"),
                torch.empty(n3[2], dtype=torch.int64, device="cuda"))
        reps = 5
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(8)] for _ in range(reps)]
        dist.barrier()
        for k in range(reps):
            for ph in range(4):
                ev[k][2 * ph].record()
                eng.score_rank_shard(N.ORX_SCORE_DOT, ph, g, user, item, bias, p["uid"], *lists[1:], *bufs, at=AT)
                ev[k][2 * ph + 1].record()
                if ph < 3:
                    reduce([bufs[ph]])
        torch.cuda.synchronize()
        split = {}
        names = ["phase0_user_rows", "phase1_pos_scores", "phase2_local_pass", "phase3_finish"]
        for ph in range(4):
            split[names[ph]] = slowest(min(e[2 * ph].elapsed_time(e[2 * ph + 1]) for e in ev))
            if ph < 3:
                split[f"allreduce{ph}"] = slowest(min(e[2 * ph + 1].elapsed_time(e[2 * ph + 2]) for e in ev))
        rec = [r for r in eng.debug_dispatch_log() if r.op == N.ORX_OP_SCORE_RANK_SHARD]
        ms = min(t_sh)
        local_rate = 2.0 * Bu * g.local_items * D / (split["phase2_local_pass"] * 1e-3) / 1e12
        row = {"shape": shape, "I": I, "D": D, "users_per_call": Bu, "max_pos": p["max_pos"],
               "ms_per_call": round(ms, 4), "ms_windows": [round(x, 4) for x in t_sh],
               "users_per_s": round(Bu / (ms * 1e-3), 1),
               "phase_ms": {k: round(v, 4) for k, v in split.items()},
               "exchange_bytes_per_call": 4 * Bu * D + 4 * Bu * (p["max_pos"] + 1) + 8 * Bu * (p["max_pos"] + 1),
               "local_pass_fp32_equiv_tflops": round(local_rate, 2),
               "local_pass_share_of_fp32_datasheet": round(local_rate / FP32_DATASHEET_TFLOPS, 3),
               "local_variant": "smem" if rec and rec[-1].variant == N.ORX_VARIANT_RANK_SMEM else "global",
               "item_splits": rec[-1].s if rec else None}
        if world == 1:
            row["plain_score_rank_ms"] = round(min(t_plain), 4)
            row["plain_ms_windows"] = [round(x, 4) for x in t_plain]
            row["phased_overhead"] = round(ms / min(t_plain) - 1.0, 4)
        out["shapes"].append(row)
        del p, part, full, user, item, bias, bufs
        torch.cuda.empty_cache()
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
