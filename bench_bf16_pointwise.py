"""fp32 against bf16 user / item tables on the fused GMF and WRMF step, under SGD, RowwiseAdagrad and Adagrad.

    python bench_bf16_pointwise.py [--rounds 3] [--window 1.0]
    python bench_bf16_pointwise.py --quality [--steps 400]

Shape: 1M users x 1M items, D = 128, B = 65 536 samples, uniform ids and labels (1 with probability 1/2) drawn from a
seed, rotating batches.  One optimizer's four configurations (GMF and WRMF, fp32 and bf16 tables) run alternated, round
after round, each in a window of at least --window seconds timed with CUDA events; the time reported is the median
over rounds.  Before anything is timed, one bf16 step of each optimizer at a small shape is judged by the bar of
tests/test_gpu_bf16_pointwise.py (the float64 step's value and float32 tolerance, through the stochastic rounding's
random bits), and one step of each configuration at the bench shape must give a finite loss; a failure exits non-zero.

Bytes per sample (bytes_per_sample): the algorithmic model of DESIGN section 4 -- 12 bytes of ids and label, the
user and item rows read and written once in the table's storage (4 or 2 bytes per element) with their optimizer state
(Adagrad one float per element, row-wise one float per row, SGD none), the item bias read and written with its state.
GMF's per-block traffic on w is left out.  GB/s is that over the step time.

--quality: a planted-low-rank dataset (users and items with true rank-16 factors; each user's positives are its top
items under them), GMF trained with Keras Adagrad on batches of positives (label 1) and uniform negatives (label 0), with
fp32 and with bf16 tables from one start (the bf16 model's tables are the fp32 start rounded to nearest) over the same
batches for --steps steps, then RankingEvaluator's AUC / Recall@50 on held-out positives.  Reported, not asserted.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

U = I = 1_000_000
D = 128
B = 65_536
N_BATCHES = 16
LR = 0.05
OPTS = ("sgd", "rowwise", "adagrad")
KINDS = ("gmf", "wrmf")


def bytes_per_sample(opt, elem, dim=D):
    """ids + label, 2 rows (r+w) with their optimizer state (r+w), the item bias (r+w) with its state (r+w)."""
    state = {"sgd": 0, "rowwise": 2 * 4, "adagrad": 2 * dim * 4}[opt]
    bias_state = 0 if opt == "sgd" else 4
    return 12 + 2 * (2 * dim * elem + state) + 2 * (4 + bias_state)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=60)
    name, power = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
    return name, power


def kind_of(N, opt):
    return {"sgd": N.ORX_OPT_SGD, "rowwise": N.ORX_OPT_ROWWISE_ADAGRAD, "adagrad": N.ORX_OPT_ADAGRAD}[opt]


def make_path(eng, torch, N, kind, opt, dtype):
    dev = torch.device("cuda", 0)
    okind = kind_of(N, opt)
    tu, ti, tb = torch.empty(U, D, device=dev), torch.empty(I, D, device=dev), torch.empty(I, 1, device=dev)
    w = torch.empty(D, 1, device=dev)
    for k, t in enumerate((tu, ti, tb, w)):
        eng.fill_uniform(t, -0.05, 0.05, 1000 + k)
    if dtype == "bf16":
        tu, ti = tu.to(torch.bfloat16), ti.to(torch.bfloat16)
    if opt == "adagrad":
        acc = [torch.full(t.shape, 0.1, device=dev) for t in (tu, ti, tb, w)]
    elif opt == "rowwise":   # one accumulator per table row; the bias and w keep element-wise ones
        acc = [torch.full((U,), 0.1, device=dev), torch.full((I,), 0.1, device=dev), torch.full_like(tb, 0.1),
               torch.full_like(w, 0.1)]
    else:
        acc = [None] * 4
    make = N.table_bf16 if dtype == "bf16" else N.table
    tabs = (make(tu, acc[0], kind=okind), make(ti, acc[1], kind=okind), N.table(tb, acc[2]))
    wt = N.OrxTable(w.data_ptr(), acc[3].data_ptr() if acc[3] is not None else None, None, 1, D) \
        if kind == "gmf" else None
    mem = sum(t.numel() * t.element_size() for t in (tu, ti, tb, *acc[:3]) if t is not None)
    return dict(kind=N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF, opt=okind, dtype=dtype,
                t=(tu, ti, tb, w), acc=acc, tabs=tabs, w=wt, mem=mem, step=0)


def run_steps(eng, N, p, batches, out4, n):
    for i in range(n):
        uid, iid, lab = batches[i % N_BATCHES]
        p["step"] += 1
        o = N.opt(p["opt"], LR, step=p["step"])
        if p["dtype"] == "bf16":
            eng.pointwise_step_bf16(p["kind"], *p["tabs"], p["w"], uid, iid, lab, o, 7, out4)
        else:
            eng.pointwise_step(p["kind"], *p["tabs"], p["w"], uid, iid, lab, o, out4)


def time_window(eng, torch, N, p, batches, out4, seconds):
    def run(n):
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
    """One bf16 GMF and WRMF step per optimizer at a small shape under the bar of tests/test_gpu_bf16_pointwise.py."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_bf16_pointwise as T
    from openrec_b200 import native as N
    eng = N.engine()
    out = {}
    for opt, k in (("sgd", T.SGD), ("rowwise", T.ROWWISE), ("adagrad", T.ADAGRAD)):
        for kind in KINDS:
            c, bar = T.make_case(kind, k, D, 4096, 11)
            d = T.Dev(c)
            out4 = T.launch(eng, c, d)
            T.judge(c, bar, d.got(), out4, f"bench check {kind} {opt}")   # raises on a miss
            out[f"{kind}_{opt}"] = "ok"
    return out


def quality(torch, steps):
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow as tf
    from openrec.tf2.recommenders import GMF
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
    for _ in range(32):   # half positives, half uniform negatives
        u = brng.integers(0, Uq, Bq)
        h = Bq // 2
        it = np.r_[tr[u[:h], brng.integers(0, tr.shape[1], h)], brng.integers(0, Iq, Bq - h)]
        batches.append((u.astype(np.int32), it.astype(np.int32), np.r_[np.ones(h), np.zeros(Bq - h)].astype(np.float32)))
    res = {"shape": {"users": Uq, "items": Iq, "dim": Dq, "batch": Bq, "planted_rank": R, "steps": steps}}
    start = None
    for dtype in ("float32", "bfloat16"):
        model = GMF(Dq, Dq, Uq, Iq, embedding_dtype=dtype, rounding_seed=3)
        if start is None:
            start = [v.numpy() for v in model.variables]
        else:                 # the same start as the fp32 model: its tables rounded to bf16
            for v, a in zip(model.variables, start):
                v.assign(a)
        opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
        for s in range(steps):
            u, i, lab = (tf.constant(x) for x in batches[s % len(batches)])
            with tf.GradientTape() as tape:
                loss = model(u, i, lab)
            opt.apply_gradients(zip(tape.gradient(loss[0], model.trainable_variables), model.trainable_variables))
        r = RankingEvaluator(val, excl_datasets=[train], at=[50]).evaluate(model)
        res[f"adagrad_{dtype}"] = {"AUC": float(np.nanmean(r["AUC"].numpy())),
                                   "Recall@50": float(np.nanmean(r["Recall"].numpy())),
                                   "final_loss": float(loss[0].numpy())}
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
        raise SystemExit("bench_bf16_pointwise.py measures on the GPU; no CUDA device")
    from openrec_b200 import native as N
    name, power = card()
    torch.cuda.set_device(0)
    if args.quality:
        print(json.dumps({"card": name, "power_limit": power, "quality": quality(torch, args.steps)}))
        return
    checks = check_bf16_paths()
    eng = N.engine(torch.device("cuda", 0))
    g = torch.Generator(device="cpu").manual_seed(1)
    batches = [(torch.randint(0, U, (B,), generator=g, dtype=torch.int32).cuda(),
                torch.randint(0, I, (B,), generator=g, dtype=torch.int32).cuda(),
                (torch.rand(B, generator=g) < 0.5).float().cuda()) for _ in range(N_BATCHES)]
    out4 = torch.zeros(4, device="cuda")
    res = {"card": name, "power_limit": power, "shape": {"users": U, "items": I, "dim": D, "batch": B},
           "bf16_step_checks": checks, "gmf": {}, "wrmf": {}}
    times = {}
    for opt in OPTS:   # one optimizer's four configurations at a time
        paths = {(kind, f"{opt}_{dt}"): make_path(eng, torch, N, kind, opt, dt) for kind in KINDS
                 for dt in ("fp32", "bf16")}
        for k, p in paths.items():
            run_steps(eng, N, p, batches, out4, 1)
            torch.cuda.synchronize()
            if not np.isfinite(out4.cpu().numpy()).all():
                raise SystemExit(f"{k}: non-finite step output {out4.cpu().numpy()}")
            times[k] = []
        for _ in range(args.rounds):
            for k, p in paths.items():
                times[k].append(time_window(eng, torch, N, p, batches, out4, args.window))
        for (kind, key), p in paths.items():
            t = float(np.median(times[(kind, key)]))
            bps = bytes_per_sample(opt, 2 if p["dtype"] == "bf16" else 4)
            res[kind][key] = {"step_ms": t * 1e3, "samples_per_sec": B / t, "bytes_per_sample": bps,
                              "GB_per_s": B * bps / t / 1e9, "table_and_slot_bytes": p["mem"],
                              "rounds_step_ms": [x * 1e3 for x in times[(kind, key)]]}
        del paths
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
