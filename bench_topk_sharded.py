"""Sharded top-K retrieval benchmark: orx_score_topk_shard's three phases with an NCCL all-reduce between them, BPR dot
+ item bias, one rank per GPU.  Prints one JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N bench_topk_sharded.py [--window 1.0] [--shapes 1m_k100,...]

Shapes: I = 1 000 000 ("1m") and 8 000 000 ("8m"), D = 128, 1 024 users per call, k = 100 and k = 1 000, exclusions
~ Poisson(100) per user (the problem generator of bench_topk.py, rows r % N of the tables on rank r).  Before timing,
rank 0 checks each 1m shape against orx_score_topk on the gathered tables (items equal, scores bit for bit); a mismatch
exits non-zero.  A call is timed with CUDA events on every rank and the slowest rank's time is reported, with a
per-phase split (each phase's C call and the all-reduce after it).  At N = 1 the plain orx_score_topk on the same
tables is timed in alternation with the phased call.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_eval import FP32_DATASHEET_TFLOPS, card  # noqa: E402
from bench_eval_sharded import slowest, timed  # noqa: E402
from bench_topk import problem  # noqa: E402
from openrec_b200 import native as N  # noqa: E402
from openrec_b200.sharded import all_reduce_sum, score_topk_sharded  # noqa: E402

SHAPES = {"1m_k100": (1_000_000, 128, 1024, 100), "1m_k1000": (1_000_000, 128, 1024, 1000),
          "8m_k100": (8_000_000, 128, 1024, 100), "8m_k1000": (8_000_000, 128, 1024, 1000)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_topk_sharded.py needs a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
    eng = N.engine()
    name, watts = card()
    reduce = all_reduce_sum()
    out = {"metric": "sharded_topk_users_per_s", "gpu": name, "power_limit_w": watts, "gpus": world,
           "kind": "BPR dot + item bias", "shapes": []}
    for shape in args.shapes.split(","):
        I, D, Bu, k = SHAPES[shape]
        p = problem(np.random.default_rng(0), I, D, Bu)     # same problem on every rank; keep this rank's rows
        del p["mask"], p["excl"]
        g = N.rowshard(world, rank, Bu, I)
        user, item, bias = (p[key][rank::world].contiguous() for key in ("user", "item", "bias"))
        checked = shape.startswith("1m")
        full = (p["user"], p["item"], p["bias"]) if world == 1 or checked else None
        if full is None:
            del p["user"], p["item"], p["bias"]
        torch.cuda.empty_cache()
        part = (eng, N.ORX_SCORE_DOT, user, item, bias, g)
        lists = (p["uid"], p["excl_off"], p["excl_items"])

        def phased():
            return score_topk_sharded([part], reduce, *lists, k)[0]

        def plain():
            return eng.score_topk(N.ORX_SCORE_DOT, full[0], p["uid"], full[1], full[2], *lists[1:], k)

        if checked:
            got = [t.cpu().numpy() for t in phased()]
            if rank == 0:
                want = [t.cpu().numpy() for t in plain()]
                if not (np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.int32),
                                                                           want[1].view(np.int32))):
                    print(json.dumps({"error": f"{shape}: sharded and single-device top-K differ"}), flush=True)
                    os._exit(1)
            dist.barrier()
        t_sh, t_plain = [], []
        for _ in range(2):
            t_sh.append(slowest(timed(phased, args.window)))
            if world == 1:
                t_plain.append(timed(plain, args.window))
        # per-phase split: each phase's C call, then the all-reduce of what it wrote, each between two events
        bufs = (torch.empty(Bu * D, dtype=torch.int32, device="cuda"),
                torch.empty(Bu * world * k, dtype=torch.int64, device="cuda"))
        reps = 5
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(6)] for _ in range(reps)]
        dist.barrier()
        for r in range(reps):
            for ph in range(3):
                ev[r][2 * ph].record()
                eng.score_topk_shard(N.ORX_SCORE_DOT, ph, g, user, item, bias, *lists, k, *bufs)
                ev[r][2 * ph + 1].record()
                if ph < 2:
                    reduce([bufs[ph]])
        torch.cuda.synchronize()
        split = {}
        names = ["phase0_user_rows", "phase1_local_pass", "phase2_merge"]
        for ph in range(3):
            split[names[ph]] = slowest(min(e[2 * ph].elapsed_time(e[2 * ph + 1]) for e in ev))
            if ph < 2:
                split[f"allreduce{ph}"] = slowest(min(e[2 * ph + 1].elapsed_time(e[2 * ph + 2]) for e in ev))
        rec = [r for r in eng.debug_dispatch_log() if r.op == N.ORX_OP_SCORE_TOPK_SHARD]
        ms = min(t_sh)
        local_rate = 2.0 * Bu * g.local_items * D / (split["phase1_local_pass"] * 1e-3) / 1e12
        row = {"shape": shape, "I": I, "D": D, "users_per_call": Bu, "k": k, "checked": checked,
               "ms_per_call": round(ms, 4), "ms_windows": [round(x, 4) for x in t_sh],
               "users_per_s": round(Bu / (ms * 1e-3), 1),
               "phase_ms": {key: round(v, 4) for key, v in split.items()},
               "exchange_bytes_per_call": 4 * Bu * D + 8 * Bu * world * k,
               "local_pass_fp32_equiv_tflops": round(local_rate, 2),
               "local_pass_share_of_fp32_datasheet": round(local_rate / FP32_DATASHEET_TFLOPS, 3),
               "item_splits": rec[-1].s if rec else None}
        if world == 1:
            row["plain_score_topk_ms"] = round(min(t_plain), 4)
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
