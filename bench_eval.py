"""Catalogue-scale evaluation benchmark: the fused orx_score_rank against orx_score_all + orx_rank_metrics, BPR DOT
with item bias, on the same device-resident inputs (the two-kernel path's dense masks are scattered on the device from
the same CSR rows).  Prints one JSON line.

    python bench_eval.py [--window 1.0] [--shapes catalogue,example]

Shapes: "catalogue" I = 1 000 000, D = 128, 1 024 users per call; "example" I = 16 980, D = 50, 1 000 users (the
reference example's evaluation).  Positives ~ Poisson(20), exclusions ~ Poisson(100) per user.  Before timing, the two
paths' outputs are compared (AUC and Recall bit for bit, NDCG within one float32 ulp); a mismatch exits non-zero.
Each path is warmed up, then timed with CUDA events over enough calls to fill --window seconds, twice, alternating
the paths; the faster window of each is reported.  Nothing is written to disk."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from openrec_b200 import native as N  # noqa: E402

FP32_DATASHEET_TFLOPS = 67.0        # H100 SXM dense FP32, at up to 700 W
SHAPES = {"catalogue": (1_000_000, 128, 1024), "example": (16_980, 50, 1000)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, watts = [s.strip() for s in out.strip().split(",")[:2]]
        return name, float(watts)
    except Exception:
        return torch.cuda.get_device_name(), None


def problem(rng, I, D, Bu):
    user = torch.from_numpy(rng.uniform(-0.1, 0.1, (Bu, D)).astype(np.float32)).cuda()
    item = torch.from_numpy(rng.uniform(-0.1, 0.1, (I, D)).astype(np.float32)).cuda()
    bias = torch.from_numpy(rng.uniform(-0.1, 0.1, I).astype(np.float32)).cuda()
    pos, excl = [], []
    for _ in range(Bu):
        n_p, n_e = rng.poisson(20), rng.poisson(100)
        c = np.unique(rng.integers(0, I, n_p + n_e))
        rng.shuffle(c)
        pos.append(np.sort(c[:n_p])), excl.append(np.sort(c[n_p:]))

    def csr(rows):
        off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
        return (torch.from_numpy(off).cuda(), torch.from_numpy(np.concatenate(rows).astype(np.int32)).cuda(),
                max(len(r) for r in rows))
    pos_off, pos_items, max_pos = csr(pos)
    excl_off, excl_items, _ = csr(excl)
    uid = torch.arange(Bu, dtype=torch.int32, device="cuda")

    def dense(off, items):
        m = torch.zeros((Bu, I), dtype=torch.uint8, device="cuda")
        rows = torch.repeat_interleave(torch.arange(Bu, device="cuda"), off[1:] - off[:-1])
        m[rows, items.long()] = 1
        return m
    return dict(user=user, item=item, bias=bias, uid=uid, pos_off=pos_off, pos_items=pos_items, excl_off=excl_off,
                excl_items=excl_items, max_pos=max_pos, pos_mask=dense(pos_off, pos_items),
                excl_mask=dense(excl_off, excl_items))


def timed(fn, window):
    """ms per call: CUDA events around enough calls to fill `window` seconds."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    n = max(3, math.ceil(window * 1e3 / max(a.elapsed_time(b), 1e-3)))
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--shapes", default="catalogue,example")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval.py needs a CUDA device")
    eng = N.engine()
    name, watts = card()
    at = (50, 100)
    out = {"metric": "eval_users_per_s", "gpu": name, "power_limit_w": watts, "kind": "BPR dot + item bias",
           "at": list(at), "shapes": []}
    for shape in args.shapes.split(","):
        I, D, Bu = SHAPES[shape]
        p = problem(np.random.default_rng(0), I, D, Bu)

        def fused():
            return eng.score_rank(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"], p["pos_off"],
                                  p["pos_items"], p["excl_off"], p["excl_items"], p["max_pos"], at=at)

        def two_kernel():
            pred = eng.score_all(N.ORX_SCORE_DOT, p["user"], p["uid"], p["item"], p["bias"])
            return eng.rank_metrics(pred, p["pos_mask"], p["excl_mask"], at=at)

        got, want = ([t.cpu().numpy() for t in f()] for f in (fused, two_kernel))
        agree = (np.array_equal(got[0].view(np.int32), want[0].view(np.int32))
                 and np.array_equal(got[2].view(np.int32), want[2].view(np.int32)))
        try:
            np.testing.assert_array_max_ulp(got[1], want[1], maxulp=1)
        except AssertionError:
            agree = False
        if not agree:
            print(json.dumps({"error": f"{shape}: fused and two-kernel outputs differ"}))
            sys.exit(1)
        t_f, t_r, n_f, n_r = [], [], 0, 0
        for _ in range(2):
            ms, n_f = timed(fused, args.window)
            t_f.append(ms)
            ms, n_r = timed(two_kernel, args.window)
            t_r.append(ms)
        tf_, tr_ = min(t_f), min(t_r)
        rate = 2.0 * Bu * I * D / (tf_ * 1e-3) / 1e12
        rec = [r for r in eng.debug_dispatch_log() if r.op == N.ORX_OP_SCORE_RANK]
        out["shapes"].append({
            "shape": shape, "I": I, "D": D, "users_per_call": Bu, "max_pos": p["max_pos"],
            "fused_ms": round(tf_, 4), "two_kernel_ms": round(tr_, 4),
            "fused_ms_windows": [round(x, 4) for x in t_f], "two_kernel_ms_windows": [round(x, 4) for x in t_r],
            "calls_per_window": [n_f, n_r],
            "fused_users_per_s": round(Bu / (tf_ * 1e-3), 1), "two_kernel_users_per_s": round(Bu / (tr_ * 1e-3), 1),
            "speedup": round(tr_ / tf_, 3), "fused_fp32_equiv_tflops": round(rate, 2),
            "fused_share_of_fp32_datasheet": round(rate / FP32_DATASHEET_TFLOPS, 3),
            "fused_variant": "smem" if rec and rec[-1].variant == N.ORX_VARIANT_RANK_SMEM else "global",
            "item_splits": rec[-1].s if rec else None})
        del p
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
