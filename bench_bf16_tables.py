"""fp32 against bf16 user / item tables on the fused BPR step, under SGD, RowwiseAdagrad and Adagrad.

    python bench_bf16_tables.py [--rounds 3] [--window 1.0]
    python bench_bf16_tables.py --quality [--steps 400]

bench.py's BPR (1M users x 1M items, D = 128, B = 65 536, uniform ids, rotating batches, each batch's index prefetched
while the previous step runs): the six configurations run alternated, round after round, each in a window of at least
--window seconds timed with CUDA events; the time reported is the median over rounds.  Before anything is timed, one
bf16 step of each optimizer at a small shape is judged by the bar of tests/test_gpu_bf16_tables.py (the float64 step's
value and float32 tolerance, through the stochastic rounding's random bits), and one step of each configuration at the
bench shape must give a finite loss; a failure exits non-zero.

Bytes per triplet (BYTES): the algorithmic model of DESIGN section 4 -- 12 bytes of ids, each of a triplet's three rows
read and written once in the table's storage (4 or 2 bytes per element) with its optimizer state (Adagrad one float
per element, row-wise one float per row, SGD none), the two item biases read and written with their state.  GB/s is that
over the step time, and the share of the 3.35 TB/s HBM3 data-sheet figure of an H100 SXM.  Device memory is the bytes
of the tables plus their slots.

--quality: a planted-low-rank dataset (users and items with true rank-16 factors; each user's positives are its top
items under them), BPR trained on its loss with fp32 and with bf16 tables under the same optimizer (Adagrad, Keras
Adam), start (the bf16 model's tables are the fp32 start rounded to nearest) and batches for --steps steps, then
RankingEvaluator's AUC / Recall@50 on held-out positives.  Reported, not asserted.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import B, D, I, LR, N_BATCHES, U  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
OPTS = ("sgd", "rowwise", "adagrad")


def bytes_per_triplet(opt, elem):
    """ids + 3 rows (r+w) + 2 biases (r+w) + optimizer state (r+w)."""
    state = {"sgd": 0, "rowwise": 3 * 4, "adagrad": 3 * D * 4}[opt]
    bias_state = 0 if opt == "sgd" else 2 * 4
    return 12 + 2 * (3 * D * elem + state) + 2 * (2 * 4 + bias_state)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=60)
    name, power = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
    return name, power


def kind_of(N, opt):
    return {"sgd": N.ORX_OPT_SGD, "rowwise": N.ORX_OPT_ROWWISE_ADAGRAD, "adagrad": N.ORX_OPT_ADAGRAD}[opt]


def make_path(eng, torch, N, opt, dtype):
    dev = torch.device("cuda", 0)
    kind = kind_of(N, opt)
    tu, ti, tb = torch.empty(U, D, device=dev), torch.empty(I, D, device=dev), torch.empty(I, 1, device=dev)
    for k, t in enumerate((tu, ti, tb)):
        eng.fill_uniform(t, -0.05, 0.05, 1000 + k)
    if dtype == "bf16":
        tu, ti = tu.to(torch.bfloat16), ti.to(torch.bfloat16)
    if opt == "adagrad":
        acc = [torch.full(t.shape, 0.1, device=dev) for t in (tu, ti, tb)]
    elif opt == "rowwise":
        acc = [torch.full((U,), 0.1, device=dev), torch.full((I,), 0.1, device=dev), torch.full_like(tb, 0.1)]
    else:
        acc = [None, None, None]
    make = N.table_bf16 if dtype == "bf16" else N.table
    tabs = (make(tu, acc[0], kind=kind), make(ti, acc[1], kind=kind), N.table(tb, acc[2]))
    mem = sum(t.numel() * t.element_size() for t in (tu, ti, tb, *acc) if t is not None)
    return dict(kind=kind, dtype=dtype, t=(tu, ti, tb), acc=acc, tabs=tabs, mem=mem, step=0)


def run_steps(eng, N, p, batches, out4, n, start=0):
    """n steps over the rotating batches, each step's successor prefetched under it (as bench.py's loop)."""
    step = eng.pairwise_step_bf16 if p["dtype"] == "bf16" else eng.pairwise_step
    for i in range(start, start + n):
        b = batches[i % N_BATCHES]
        p["step"] += 1
        o = N.opt(p["kind"], LR, step=p["step"])
        if p["dtype"] == "bf16":
            step(N.ORX_PAIR_BPR, *p["tabs"], *b, o, 7, out4)
        else:
            step(N.ORX_PAIR_BPR, *p["tabs"], *b, o, out4)
        nb = batches[(i + 1) % N_BATCHES]
        eng.pairwise_prefetch(p["tabs"][0], p["tabs"][1], *nb, p["kind"], ids_ready=True)


def time_window(eng, torch, N, p, batches, out4, seconds):
    def run(n):
        eng.pairwise_prefetch(p["tabs"][0], p["tabs"][1], *batches[0], p["kind"], ids_ready=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run_steps(eng, N, p, batches, out4, n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3
    t = run(20)
    n = max(20, int(np.ceil(seconds / (t / 20))))
    return run(n) / n


def check_bf16_paths():
    """One bf16 step per optimizer at a small shape under the bar of tests/test_gpu_bf16_tables.py."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_bf16_tables as T
    from openrec_b200 import native as N
    eng = N.engine()
    out = {}
    for opt, k in (("sgd", T.SGD), ("rowwise", T.ROWWISE), ("adagrad", T.ADAGRAD)):
        c, bar = T.make_case("bpr", k, D, 4096, 11)
        d = T.Dev(c)
        out4 = T.launch(eng, c, d)
        T.judge(c, bar, d.got(), out4, f"bench check {opt}")   # raises on a miss
        out[opt] = "ok"
    return out


def quality(torch, steps):
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow as tf
    from openrec.tf2.recommenders import BPR
    from openrec_b200.tf2.data.dataset import Dataset
    from openrec_b200.tf2.metrics.evaluator import RankingEvaluator
    Uq, Iq, Dq, Bq, R, POS = 4000, 6000, 64, 1024, 16, 30
    rng = np.random.default_rng(0)
    pu, pi = rng.standard_normal((Uq, R)), rng.standard_normal((Iq, R))
    top = np.argsort(-(pu @ pi.T), axis=1)[:, :POS]
    tr, va = top[:, :POS - 5], top[:, POS - 5:]

    def ds(items):
        raw = np.empty(items.size, dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = np.repeat(np.arange(Uq), items.shape[1]), items.reshape(-1)
        return Dataset(raw_data=raw, total_users=Uq, total_items=Iq)
    train, val = ds(tr), ds(va)
    brng = np.random.default_rng(1)
    batches = []
    for _ in range(32):
        u = brng.integers(0, Uq, Bq)
        batches.append((u.astype(np.int32), tr[u, brng.integers(0, tr.shape[1], Bq)].astype(np.int32),
                        brng.integers(0, Iq, Bq).astype(np.int32)))
    res = {"shape": {"users": Uq, "items": Iq, "dim": Dq, "batch": Bq, "planted_rank": R, "steps": steps}}
    # the loss alone (no L2 term) and optimizers that normalise BPR's 1/B-scaled gradient, so that the planted signal
    # is learnt within --steps steps
    for opt_name, mk in (("adagrad", lambda: tf.keras.optimizers.Adagrad(learning_rate=0.02,
                                                                          initial_accumulator_value=1e-6)),
                         ("adam", lambda: tf.keras.optimizers.Adam(learning_rate=0.002))):
        for dtype in ("float32", "bfloat16"):
            model = BPR(Dq, Dq, Uq, Iq, embedding_dtype=dtype, rounding_seed=3)
            if dtype == "bfloat16":   # the same start as the fp32 model: its tables rounded to bf16
                ref = res.get(f"_{opt_name}_start")
                for v, a in zip(model.variables, ref):
                    v.assign(a)
            else:
                res[f"_{opt_name}_start"] = [v.numpy() for v in model.variables]
            opt = mk()
            for s in range(steps):
                u, p, n = (tf.constant(x) for x in batches[s % len(batches)])
                with tf.GradientTape() as tape:
                    loss = model(u, p, n)
                opt.apply_gradients(zip(tape.gradient(loss[0], model.trainable_variables), model.trainable_variables))
            ev = RankingEvaluator(val, excl_datasets=[train], at=[50])
            r = ev.evaluate(model)
            res[f"{opt_name}_{dtype}"] = {"AUC": float(np.nanmean(r["AUC"].numpy())),
                                          "Recall@50": float(np.nanmean(r["Recall"].numpy())),
                                          "final_loss": float(loss[0].numpy())}
    for k in [k for k in res if k.startswith("_")]:
        del res[k]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--steps", type=int, default=400)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_bf16_tables.py measures on the GPU; no CUDA device")
    from openrec_b200 import native as N
    name, power = card()
    torch.cuda.set_device(0)
    if args.quality:
        print(json.dumps({"card": name, "power_limit": power, "quality": quality(torch, args.steps)}))
        return
    checks = check_bf16_paths()
    eng = N.engine(torch.device("cuda", 0))
    g = torch.Generator(device="cpu").manual_seed(1)
    batches = [tuple(torch.randint(0, n, (B,), generator=g, dtype=torch.int32).cuda() for n in (U, I, I))
               for _ in range(N_BATCHES)]
    out4 = torch.zeros(4, device="cuda")
    res = {"card": name, "power_limit": power, "bf16_step_checks": checks, "bpr": {}}
    times = {}
    for opt in OPTS:   # one optimizer's two configurations at a time: six tables of 1M x 128 would not all fit with slots
        paths = {f"{opt}_{dt}": make_path(eng, torch, N, opt, dt) for dt in ("fp32", "bf16")}
        for k, p in paths.items():
            run_steps(eng, N, p, batches, out4, 1)
            torch.cuda.synchronize()
            if not np.isfinite(out4.cpu().numpy()).all():
                raise SystemExit(f"{k}: non-finite step output {out4.cpu().numpy()}")
            times[k] = []
        for _ in range(args.rounds):
            for k, p in paths.items():
                times[k].append(time_window(eng, torch, N, p, batches, out4, args.window))
        for k, p in paths.items():
            t = float(np.median(times[k]))
            bpt = bytes_per_triplet(opt, 2 if p["dtype"] == "bf16" else 4)
            res["bpr"][k] = {"step_ms": t * 1e3, "triplets_per_sec": B / t, "bytes_per_triplet": bpt,
                             "GB_per_s": B * bpt / t / 1e9, "share_of_3.35TBps": B * bpt / t / HBM_BYTES_PER_S,
                             "table_and_slot_bytes": p["mem"], "rounds_step_ms": [x * 1e3 for x in times[k]]}
        del paths
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
