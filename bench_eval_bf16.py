"""Scoring bf16 tables in place against today's upcast-then-fp32 path and against fp32 tables, BPR DOT with item bias,
I = 1 000 000 items, D = 128.  Prints one JSON line.

    python bench_eval_bf16.py [--window 1.0] [--rounds 2]

Calls timed, each on three paths with the same values (the fp32 tables are the exact upcast of the bf16 ones):
  bf16      the call on the bf16 tables (orx_score_*_bf16, picked by native.Engine from the dtype);
  upcast    user.float() and item.float() of the bf16 tables, then the fp32 call: what one request that is a single
            batch cost before (evaluate / recommend upcast once per call, so over several batches it was amortized);
  fp32      the fp32 call on fp32 tables held beforehand.
Shapes: orx_score_rank with 1 024 users and cut-offs 50 / 100 (positives ~ Poisson(20), exclusions ~ Poisson(100), as
bench_eval.py draws them); orx_score_topk with 1 024 users and with 64 users (a serving batch), k = 100, excluding the
same rows; orx_score_rank_listed with 100 listed items per user.  The user table has 1 000 000 rows, so the upcast path
copies both 1M x 128 tables.  Before timing, each call's bf16 outputs must equal its fp32 outputs bit for bit; a
mismatch exits non-zero.  The three paths run alternated, round after round, each over a window of at least --window
seconds timed with CUDA events; the fastest round of each is reported.

Model level, on a bf16 BPR of 100 000 users x 1M items: RankingEvaluator.evaluate (batch 1 024, about 18 batches) and
Retriever.recommend (2 000 users, batch 64, 32 batches), scoring the stored tables (in place) and scoring an fp32
upcast made once per call (before: the model's scoring operands upcast, as BPR._score_operands did).  For each, the
peak rise of torch.cuda.max_memory_allocated() and the wall time of the whole call (host clock around calls that end
in a device synchronise, the two paths alternated, fastest of --rounds).

The card's name and power limit are read in the same run.  Nothing is written to disk."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from openrec_b200 import native as N  # noqa: E402

U = I = 1_000_000
D = 128
AT = (50, 100)
K = 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, watts = [s.strip() for s in out.strip().split(",")[:2]]
        return name, float(watts)
    except Exception:
        return torch.cuda.get_device_name(), None


def csr(rows):
    """rows of users 0 .. len(rows) - 1; the users after them, up to U, have empty rows"""
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    off = np.concatenate([off, np.full(U - len(rows), off[-1], np.int64)])
    return (torch.from_numpy(off).cuda(), torch.from_numpy(np.concatenate(rows).astype(np.int32)).cuda(),
            max(len(r) for r in rows))


def lists(rng, Bu):
    """Users 0 .. Bu - 1: positives ~ Poisson(20), exclusions ~ Poisson(100) (bench_eval.py's draws), 100 listed."""
    pos, excl, neg = [], [], []
    for _ in range(Bu):
        n_p, n_e = rng.poisson(20), rng.poisson(100)
        c = np.unique(rng.integers(0, I, n_p + n_e + 100))
        rng.shuffle(c)
        pos.append(np.sort(c[:n_p])), excl.append(np.sort(c[n_p:n_p + n_e])), neg.append(np.sort(c[-100:]))
    return csr(pos), csr(excl), csr(neg)


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
    return a.elapsed_time(b) / n


def bits(out):
    return [t.contiguous().view(torch.int32).cpu() if t.dtype == torch.float32 else t.cpu() for t in out]


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def model_level(rng, rounds):
    """Peak allocation rise (bytes) of evaluate + recommend on a bf16 BPR, scoring in place and via an fp32 upcast."""
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tf2.data.dataset import Dataset
    from openrec_b200.tf2.metrics.evaluator import RankingEvaluator
    Um = 100_000
    model = Rm.BPR(D, D, Um, I, embedding_dtype="bfloat16")

    def mk(n):
        raw = np.empty(n, dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = rng.integers(0, Um, n), rng.integers(0, I, n)
        return Dataset(raw_data=raw, total_users=Um, total_items=I)
    train, val = mk(400_000), mk(20_000)
    ev = RankingEvaluator(val, excl_datasets=[train], at=list(AT), batch_size=1024)
    ret = Rm.Retriever(excl_datasets=[train], k=K, batch_size=64)
    users = np.arange(0, Um, 50, dtype=np.int32)

    class Upcast:   # the model's scoring operands with the tables upcast for the call, as scoring bf16 tables did
        def _score_operands(self):
            kind, user, item, bias, scale = model._score_operands()
            return kind, user.float(), item.float(), bias, scale

    out = {"users": Um, "items": I, "dim": D, "bf16_table_bytes": 2 * D * (Um + I)}
    paths = (("in_place", model), ("upcast", Upcast()))
    for name, m in paths:
        out[f"evaluate_peak_rise_bytes_{name}"] = peak(lambda: ev.evaluate(m))
        out[f"recommend_peak_rise_bytes_{name}"] = peak(lambda: ret.recommend(m, users))
    t = {f"{what}_ms_{name}": [] for what in ("evaluate", "recommend") for name, _ in paths}
    for _ in range(rounds):
        for name, m in paths:
            t[f"evaluate_ms_{name}"].append(wall_ms(lambda: ev.evaluate(m)))
            t[f"recommend_ms_{name}"].append(wall_ms(lambda: ret.recommend(m, users)))
    out.update({k: round(min(v), 3) for k, v in t.items()})
    out["evaluate_batches"] = -(-len(ev.warm_users) // 1024)
    out["recommend_batches"] = -(-len(users) // 64)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per timed window")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval_bf16.py needs a CUDA device")
    eng = N.engine()
    name, watts = card()
    rng = np.random.default_rng(0)
    ub = torch.empty(U, D, device="cuda")
    ib = torch.empty(I, D, device="cuda")
    bias = torch.empty(I, device="cuda")
    for k, t in enumerate((ub, ib, bias)):
        eng.fill_uniform(t, -0.1, 0.1, 100 + k)
    ub, ib = ub.to(torch.bfloat16), ib.to(torch.bfloat16)
    uf, itf = ub.float(), ib.float()
    (po, pi, mp), (eo, ei, _), (no, ni, _) = lists(rng, 1024)
    uid = {Bu: torch.arange(Bu, dtype=torch.int32, device="cuda") for Bu in (1024, 64)}
    dot = N.ORX_SCORE_DOT

    calls = {
        "score_rank_1024": lambda u, i: eng.score_rank(dot, u, uid[1024], i, bias, po, pi, eo, ei, mp, at=AT),
        "score_topk_1024": lambda u, i: eng.score_topk(dot, u, uid[1024], i, bias, eo, ei, K),
        "score_topk_64": lambda u, i: eng.score_topk(dot, u, uid[64], i, bias, eo, ei, K),
        "score_rank_listed_1024": lambda u, i: eng.score_rank_listed(dot, u, uid[1024], i, bias, po, pi, no, ni, eo,
                                                                     ei, mp, at=AT),
    }
    paths = {"bf16": lambda f: f(ub, ib), "upcast": lambda f: f(ub.float(), ib.float()), "fp32": lambda f: f(uf, itf)}
    out = {"metric": "bf16_scoring_ms", "gpu": name, "power_limit_w": watts, "kind": "BPR dot + item bias", "I": I,
           "U": U, "D": D, "at": list(AT), "k": K, "calls": []}
    for cname, f in calls.items():
        got, want = bits(paths["bf16"](f)), bits(paths["fp32"](f))
        if not all(torch.equal(a, b) for a, b in zip(got, want)):
            print(json.dumps({"error": f"{cname}: bf16 and fp32 outputs differ"}))
            sys.exit(1)
        t = {p: [] for p in paths}
        for _ in range(args.rounds):
            for p, run in paths.items():
                t[p].append(timed(lambda: run(f), args.window))
        best = {p: min(v) for p, v in t.items()}
        out["calls"].append({"call": cname, **{f"{p}_ms": round(v, 4) for p, v in best.items()},
                             **{f"{p}_ms_rounds": [round(x, 4) for x in v] for p, v in t.items()},
                             "bf16_over_upcast": round(best["bf16"] / best["upcast"], 3),
                             "bf16_over_fp32": round(best["bf16"] / best["fp32"], 3), "bit_equal": True})
    del ub, ib, uf, itf, bias
    torch.cuda.empty_cache()
    out["model"] = model_level(rng, max(args.rounds, 3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
