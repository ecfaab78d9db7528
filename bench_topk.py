"""Catalogue top-K retrieval benchmark: the fused orx_score_topk against what a user writes today, orx_score_all ->
masked_fill(-inf) over the exclusions -> torch.topk, BPR DOT with item bias, on the same device-resident inputs.
Prints one JSON line.

    python bench_topk.py [--window 1.0] [--shapes catalogue_k100,catalogue_k1000,example_k100]

Shapes: "catalogue" I = 1 000 000, D = 128, 1 024 users per call, k = 100 and k = 1 000; "example" I = 16 980, D = 50,
1 000 users, k = 100 (the reference example's evaluation).  Exclusions ~ Poisson(100) per user.  Before timing, the
fused result is compared with orx_score_all plus the oracle order (tests/topk_oracle.py) on a fixed sample of rows; a
mismatch exits non-zero.  Each path is warmed up, then timed with CUDA events over enough calls to fill --window
seconds, twice, alternating the paths; the faster window of each is reported.  The catalogue shape at k = 100 is also
timed once with scores rising with item id (every tile compacts every row's candidate list: the worst case).  Nothing
is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, "tests")]
from bench_eval import FP32_DATASHEET_TFLOPS, card, timed  # noqa: E402
from openrec_b200 import native as N  # noqa: E402
from topk_oracle import topk as oracle_topk  # noqa: E402

SHAPES = {"catalogue_k100": (1_000_000, 128, 1024, 100), "catalogue_k1000": (1_000_000, 128, 1024, 1000),
          "example_k100": (16_980, 50, 1000, 100)}
SAMPLE_ROWS = 16


def problem(rng, I, D, Bu):
    user = torch.from_numpy(rng.uniform(-0.1, 0.1, (Bu, D)).astype(np.float32)).cuda()
    item = torch.from_numpy(rng.uniform(-0.1, 0.1, (I, D)).astype(np.float32)).cuda()
    bias = torch.from_numpy(rng.uniform(-0.1, 0.1, I).astype(np.float32)).cuda()
    excl = [np.unique(rng.integers(0, I, rng.poisson(100))) for _ in range(Bu)]
    off = np.concatenate([[0], np.cumsum([len(r) for r in excl])]).astype(np.int64)
    excl_off = torch.from_numpy(off).cuda()
    excl_items = torch.from_numpy(np.concatenate(excl).astype(np.int32)).cuda()
    uid = torch.arange(Bu, dtype=torch.int32, device="cuda")
    mask = torch.zeros((Bu, I), dtype=torch.bool, device="cuda")
    mask[torch.repeat_interleave(torch.arange(Bu, device="cuda"), excl_off[1:] - excl_off[:-1]), excl_items.long()] = True
    return dict(user=user, item=item, bias=bias, uid=uid, excl_off=excl_off, excl_items=excl_items, mask=mask,
                excl=excl)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_topk.py needs a CUDA device")
    eng = N.engine()
    name, watts = card()
    out = {"metric": "topk_users_per_s", "gpu": name, "power_limit_w": watts, "kind": "BPR dot + item bias",
           "shapes": []}
    for shape in args.shapes.split(","):
        I, D, Bu, k = SHAPES[shape]
        p = problem(np.random.default_rng(0), I, D, Bu)

        def fused():
            return eng.score_topk(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"], p["excl_off"],
                                  p["excl_items"], k)

        def unfused():
            pred = eng.score_all(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"])
            pred.masked_fill_(p["mask"], float("-inf"))
            return torch.topk(pred, k, dim=1)

        items, scores = (t.cpu().numpy() for t in fused())
        rows = np.random.default_rng(1).choice(Bu, SAMPLE_ROWS, replace=False)
        pred = eng.score_all(N.ORX_SCORE_DOT, p["user"], p["uid"][rows].contiguous(), p["item"], p["bias"])
        excl = np.zeros((SAMPLE_ROWS, I), bool)
        for j, b in enumerate(rows):
            excl[j, p["excl"][b]] = True
        want_i, want_s = oracle_topk(pred.cpu().numpy(), excl, k)
        del pred
        if not (np.array_equal(items[rows], want_i) and np.array_equal(scores[rows], want_s)):
            print(json.dumps({"error": f"{shape}: fused top-K differs from orx_score_all + the oracle order"}))
            sys.exit(1)
        t_f, t_u, n_f, n_u = [], [], 0, 0
        for _ in range(2):
            ms, n_f = timed(fused, args.window)
            t_f.append(ms)
            ms, n_u = timed(unfused, args.window)
            t_u.append(ms)
        tf_, tu_ = min(t_f), min(t_u)
        rec = [r for r in eng.debug_dispatch_log() if r.op == N.ORX_OP_SCORE_TOPK]
        splits = rec[-1].s if rec else None
        rate = 2.0 * Bu * I * D / (tf_ * 1e-3) / 1e12
        entry = {
            "shape": shape, "I": I, "D": D, "users_per_call": Bu, "k": k,
            "fused_ms": round(tf_, 4), "unfused_ms": round(tu_, 4),
            "fused_ms_windows": [round(x, 4) for x in t_f], "unfused_ms_windows": [round(x, 4) for x in t_u],
            "calls_per_window": [n_f, n_u],
            "fused_users_per_s": round(Bu / (tf_ * 1e-3), 1), "unfused_users_per_s": round(Bu / (tu_ * 1e-3), 1),
            "speedup": round(tu_ / tf_, 3), "fused_fp32_equiv_tflops": round(rate, 2),
            "fused_share_of_fp32_datasheet": round(rate / FP32_DATASHEET_TFLOPS, 3), "item_splits": splits,
            "fused_scratch_bytes": 8 * Bu * splits * (k + 1024) + 4 * Bu * splits if splits else None,
            "unfused_score_matrix_bytes": 4 * Bu * I}
        if shape == "catalogue_k100":
            # worst case: scores rise with item id, so every item beats every row's threshold
            p["bias"] = torch.arange(I, dtype=torch.float32, device="cuda")
            ms, _ = timed(fused, args.window)
            entry["rising_scores_fused_ms"] = round(ms, 4)
        out["shapes"].append(entry)
        del p
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
