"""Listed-candidate evaluation benchmark: orx_score_rank_listed (each user ranked against its listed items only)
against the path users have without it -- dense masks pos = P, excl = ~(P u L) u E scattered on the device from the
same CSR rows, then orx_score_all + orx_rank_metrics over the whole catalogue.  BPR DOT with item bias.  Prints one
JSON line.

    python bench_eval_listed.py [--window 1.0] [--shapes catalogue,example]

Shapes: "catalogue" I = 1 000 000, D = 128, 1 024 users per call; "example" I = 16 980, D = 50, 1 000 users.
Positives ~ Poisson(20), 100 listed items per user drawn uniformly from its non-positives, exclusions ~ Poisson(100),
all from a fixed seed.  Before timing, the two paths' outputs are compared (AUC and Recall bit for bit, NDCG within one
float32 ulp); a mismatch exits non-zero.  Each path is warmed up, then timed with CUDA events over enough calls to fill
--window seconds, twice, alternating the paths; the faster window of each is reported.  The listed call's algorithmic
bytes are one item row (4 * D bytes) and one bias per positive and listed item, plus the user rows and the three CSR
lists; their rate is reported against the 3.35 TB/s data-sheet HBM3 figure.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_eval import card, timed  # noqa: E402
from openrec_b200 import native as N  # noqa: E402

HBM_DATASHEET_TBPS = 3.35           # H100 SXM HBM3, data sheet
SHAPES = {"catalogue": (1_000_000, 128, 1024), "example": (16_980, 50, 1000)}
N_LISTED = 100


def problem(rng, I, D, Bu):
    user = torch.from_numpy(rng.uniform(-0.1, 0.1, (Bu, D)).astype(np.float32)).cuda()
    item = torch.from_numpy(rng.uniform(-0.1, 0.1, (I, D)).astype(np.float32)).cuda()
    bias = torch.from_numpy(rng.uniform(-0.1, 0.1, I).astype(np.float32)).cuda()
    pos, neg, excl = [], [], []
    for _ in range(Bu):
        p = np.unique(rng.integers(0, I, rng.poisson(20)))
        n = set()
        while len(n) < N_LISTED:
            n |= set(rng.integers(0, I, N_LISTED - len(n)).tolist()) - set(p.tolist())
        pos.append(p), neg.append(np.array(sorted(n))), excl.append(np.unique(rng.integers(0, I, rng.poisson(100))))

    def csr(rows):
        off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
        return torch.from_numpy(off).cuda(), torch.from_numpy(np.concatenate(rows).astype(np.int32)).cuda()
    lists = [csr(r) for r in (pos, neg, excl)]
    max_pos = max(len(r) for r in pos)
    uid = torch.arange(Bu, dtype=torch.int32, device="cuda")
    n_rows = sum(len(r) for r in pos) + sum(len(r) for r in neg)
    list_bytes = sum(o.numel() * 8 + it.numel() * 4 for o, it in lists)
    return dict(user=user, item=item, bias=bias, uid=uid, lists=lists, max_pos=max_pos,
                bytes=n_rows * (4 * D + 4) + Bu * 4 * D + list_bytes, rows=n_rows)


def masks(p, I):
    """The dense masks of Dataset.evaluation for explicit negatives, scattered on the device from the CSR rows."""
    Bu = p["uid"].numel()

    def scatter(m, off, items, value):
        rows = torch.repeat_interleave(torch.arange(Bu, device="cuda"), off[1:] - off[:-1])
        m[rows, items.long()] = value
    (po, pi), (no, ni), (eo, ei) = p["lists"]
    pos = torch.zeros((Bu, I), dtype=torch.uint8, device="cuda")
    excl = torch.ones((Bu, I), dtype=torch.uint8, device="cuda")
    scatter(pos, po, pi, 1)
    scatter(excl, po, pi, 0)
    scatter(excl, no, ni, 0)
    scatter(excl, eo, ei, 1)
    return pos, excl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--shapes", default="catalogue,example")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval_listed.py needs a CUDA device")
    eng = N.engine()
    name, watts = card()
    at = (10, 50)
    out = {"metric": "listed_eval_users_per_s", "gpu": name, "power_limit_w": watts, "kind": "BPR dot + item bias",
           "at": list(at), "listed_per_user": N_LISTED, "shapes": []}
    for shape in args.shapes.split(","):
        I, D, Bu = SHAPES[shape]
        p = problem(np.random.default_rng(0), I, D, Bu)
        (po, pi), (no, ni), (eo, ei) = p["lists"]

        def listed():
            return eng.score_rank_listed(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"], po, pi, no, ni,
                                         eo, ei, p["max_pos"], at=at)

        def dense():
            pos, excl = masks(p, I)
            pred = eng.score_all(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"])
            return eng.rank_metrics(pred, pos, excl, at=at)

        got, want = ([t.cpu().numpy() for t in f()] for f in (listed, dense))
        agree = (np.array_equal(got[0].view(np.int32), want[0].view(np.int32))
                 and np.array_equal(got[2].view(np.int32), want[2].view(np.int32)))
        try:
            np.testing.assert_array_max_ulp(got[1], want[1], maxulp=1)
        except AssertionError:
            agree = False
        if not agree:
            print(json.dumps({"error": f"{shape}: listed and dense-mask outputs differ"}))
            sys.exit(1)
        t_l, t_d, n_l, n_d = [], [], 0, 0
        for _ in range(2):
            ms, n_l = timed(listed, args.window)
            t_l.append(ms)
            ms, n_d = timed(dense, args.window)
            t_d.append(ms)
        tl, td = min(t_l), min(t_d)
        bw = p["bytes"] / (tl * 1e-3) / 1e12
        out["shapes"].append({
            "shape": shape, "I": I, "D": D, "users_per_call": Bu, "max_pos": p["max_pos"], "item_rows": p["rows"],
            "listed_ms": round(tl, 4), "dense_ms": round(td, 4),
            "listed_ms_windows": [round(x, 4) for x in t_l], "dense_ms_windows": [round(x, 4) for x in t_d],
            "calls_per_window": [n_l, n_d],
            "listed_users_per_s": round(Bu / (tl * 1e-3), 1), "dense_users_per_s": round(Bu / (td * 1e-3), 1),
            "speedup": round(td / tl, 1), "listed_algorithmic_mb": round(p["bytes"] / 1e6, 2),
            "listed_tbps": round(bw, 3), "listed_share_of_hbm_datasheet": round(bw / HBM_DATASHEET_TBPS, 3)})
        del p
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
