"""SGD with momentum and Nesterov momentum against SGD and Adagrad on the fused BPR step, and against Adagrad on the
Criteo-shape DLRM.

    python bench_momentum.py [--rounds 3] [--window 1.0] [--dlrm-steps 20] [--no-dlrm]

BPR at bench.py's shape (1M users x 1M items, D = 128, B = 65 536, uniform ids): the four optimizers' steps run
alternated, round after round, each in a window of at least --window seconds timed with CUDA events; the rate reported
is the median over rounds.  Each path first runs one step checked against a float64 step on a fixed sample of its rows
(value and optimizer slot); a mismatch exits non-zero before anything is timed.  Bytes per triplet are the algorithmic
model (ids, and each of a triplet's three rows plus its two item biases read and written once with their optimizer
state: one slot for Adagrad and both momentum forms, none for SGD); GB/s is that over the measured step time, and the
share of the 3.35 TB/s HBM3 data-sheet figure of an H100 SXM.

DLRM at the Criteo shape of bench.py (26 tables x 1M rows x 128): the Keras step (tape + apply_gradients) under Adagrad
and under SGD(momentum=0.9), one model after the other.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import B, D, DLRM_B, DLRM_BOT, DLRM_DENSE, DLRM_LR, DLRM_T, DLRM_TOP, DLRM_VOCAB, I, LR, N_BATCHES, U  # noqa

HBM_BYTES_PER_S = 3.35e12
SAMPLE = 2048            # checked rows per table
MOMENTUM = 0.9
# bytes per triplet: 12 of ids; the three rows and two biases (3D + 2 floats) read and written, plus per optimizer the
# state read and written with them: one float per element for Adagrad and both momentum forms, none for SGD
BYTES = {"sgd": 12 + 4 * (3 * D + 2) * 2, "momentum": 12 + 4 * (3 * D + 2) * 4, "nesterov": 12 + 4 * (3 * D + 2) * 4,
         "adagrad": 12 + 4 * (3 * D + 2) * 4}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=60)
    name, power = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
    return name, power


def bpr_paths(eng, torch, N):
    dev = torch.device("cuda", 0)
    paths = {}
    for name, kind in (("sgd", N.ORX_OPT_SGD), ("momentum", N.ORX_OPT_MOMENTUM), ("nesterov", N.ORX_OPT_NESTEROV),
                       ("adagrad", N.ORX_OPT_ADAGRAD)):
        tu, ti, tb = torch.empty(U, D, device=dev), torch.empty(I, D, device=dev), torch.empty(I, 1, device=dev)
        for k, t in enumerate((tu, ti, tb)):
            eng.fill_uniform(t, -0.05, 0.05, 1000 + k)
        if kind == N.ORX_OPT_ADAGRAD:
            acc = [torch.full_like(t, 0.1) for t in (tu, ti, tb)]
        elif kind == N.ORX_OPT_SGD:
            acc = [None, None, None]
        else:                     # a nonzero velocity, so that the check sees its decay
            acc = [torch.empty_like(t) for t in (tu, ti, tb)]
            for k, a in enumerate(acc):
                eng.fill_uniform(a, -0.01, 0.01, 2000 + k)
        tabs = tuple(N.table(t, a) for t, a in zip((tu, ti, tb), acc))
        paths[name] = dict(kind=kind, t=(tu, ti, tb), acc=acc, tabs=tabs, o=N.opt(kind, LR, beta1=MOMENTUM))
    return paths


def check_step(eng, torch, N, p, ids, out4):
    """One step of path p on batch ids against float64 on SAMPLE user and item rows: -> max relative error."""
    tu, ti, tb = p["t"]
    u_id, p_id, n_id = (x.long() for x in ids)
    pre = [x.double().cpu().numpy() for x in (tu[u_id], ti[p_id], ti[n_id], tb[p_id, 0], tb[n_id, 0])]
    uid, pid, nid = (x.cpu().numpy() for x in ids)
    rng = np.random.default_rng(7)
    rows = {"user": rng.choice(np.unique(uid), SAMPLE, replace=False),
            "item": rng.choice(np.unique(np.r_[pid, nid]), SAMPLE, replace=False)}
    tabs = {"user": tu, "item": ti}
    old = {k: tabs[k][torch.from_numpy(r).to(tu.device).long()].double().cpu().numpy() for k, r in rows.items()}
    old_acc = {k: None if p["acc"][j] is None else
               p["acc"][j][torch.from_numpy(r).to(tu.device).long()].double().cpu().numpy()
               for j, (k, r) in enumerate(rows.items())}
    eng.pairwise_step(N.ORX_PAIR_BPR, *p["tabs"], *ids, p["o"], out4)
    torch.cuda.synchronize()
    u, pv, nv, bp, bn = pre
    x = (u * pv).sum(1) + bp - (u * nv).sum(1) - bn
    y = np.maximum(x, -30.0)
    g = (-(1.0 / B) / (1.0 + np.exp(y)) * (x >= -30.0))[:, None]
    contrib = {"user": [(uid, g * (pv - nv) + u)], "item": [(pid, g * u + pv), (nid, -g * u + nv)]}
    worst = 0.0
    for j, k in enumerate(("user", "item")):
        r = rows[k]
        pos = {int(v): q for q, v in enumerate(r)}
        G = np.zeros((len(r), D))
        for ids_k, val in contrib[k]:
            sel = np.array([int(v) in pos for v in ids_k])
            np.add.at(G, np.array([pos[int(v)] for v in ids_k[sel]], dtype=np.int64), val[sel])
        if p["kind"] == N.ORX_OPT_SGD:
            want, want_acc = old[k] - LR * G, None
        elif p["kind"] == N.ORX_OPT_ADAGRAD:
            want_acc = old_acc[k] + G * G
            want = old[k] - LR * G / (np.sqrt(want_acc) + 1e-7)
        else:
            m = float(np.float32(MOMENTUM))
            want_acc = m * old_acc[k] - LR * G
            want = old[k] + (m * want_acc - LR * G if p["kind"] == N.ORX_OPT_NESTEROV else want_acc)
        idx = torch.from_numpy(r).to(tu.device).long()
        got = tabs[k][idx].double().cpu().numpy()
        worst = max(worst, float((np.abs(got - want) / (np.abs(want - old[k]) + 1e-5)).max()))
        if want_acc is not None:
            got_acc = p["acc"][j][idx].double().cpu().numpy()
            worst = max(worst, float((np.abs(got_acc - want_acc) / (np.abs(want_acc) + 1e-5)).max()))
    return worst


def time_window(eng, torch, N, p, batches, out4, seconds):
    def run(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            eng.pairwise_step(N.ORX_PAIR_BPR, *p["tabs"], *batches[i % N_BATCHES], p["o"], out4)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3
    t = run(20)
    n = max(20, int(np.ceil(seconds / (t / 20))))
    return run(n) / n


def dlrm(torch, steps):
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(0)
    host = [(np.log1p(rng.integers(0, 100, (DLRM_B, DLRM_DENSE))).astype(np.float32),
             rng.integers(0, DLRM_VOCAB, (DLRM_B, DLRM_T)).astype(np.int32),
             (rng.random(DLRM_B) < 0.25).astype(np.float32)) for _ in range(4)]
    out = {}
    for name, mk in (("adagrad", lambda: tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)),
                     ("momentum", lambda: tf.keras.optimizers.SGD(learning_rate=DLRM_LR, momentum=MOMENTUM))):
        model = DLRM(m_spa=D, ln_emb=[DLRM_VOCAB] * DLRM_T, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm")
        opt = mk()
        data = [tuple(tf.constant(a) for a in b) for b in host]

        def step(i):
            with tf.GradientTape() as tape:
                loss = model(*data[i % 4])
            opt.apply_gradients(zip(tape.gradient(loss, model.trainable_variables), model.trainable_variables))
            return loss

        for i in range(3):
            step(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            loss = step(i)
        e1.record()
        torch.cuda.synchronize()
        lv = float(loss)
        if not np.isfinite(lv):
            raise SystemExit(f"DLRM {name}: loss {lv}")
        out[name] = {"step_ms": e0.elapsed_time(e1) / steps, "peak_allocated_bytes": torch.cuda.max_memory_allocated(),
                     "loss": lv}
        del model, opt, data
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--dlrm-steps", type=int, default=20)
    ap.add_argument("--no-dlrm", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_momentum.py measures on the GPU; no CUDA device")
    from openrec_b200 import native as N
    name, power = card()
    torch.cuda.set_device(0)
    eng = N.engine(torch.device("cuda", 0))
    g = torch.Generator(device="cpu").manual_seed(1)
    batches = [tuple(torch.randint(0, n, (B,), generator=g, dtype=torch.int32).cuda() for n in (U, I, I))
               for _ in range(N_BATCHES)]
    out4 = torch.zeros(4, device="cuda")
    paths = bpr_paths(eng, torch, N)
    checks = {k: check_step(eng, torch, N, p, batches[0], out4) for k, p in paths.items()}
    bad = {k: v for k, v in checks.items() if not v <= 1e-3}
    if bad:
        print(json.dumps({"error": "step check failed", "max_rel_err": checks}))
        raise SystemExit(1)
    times = {k: [] for k in paths}
    for _ in range(args.rounds):
        for k, p in paths.items():
            times[k].append(time_window(eng, torch, N, p, batches, out4, args.window))
    res = {"card": name, "power_limit": power, "bpr": {}}
    for k, ts in times.items():
        t = float(np.median(ts))
        res["bpr"][k] = {"step_ms": t * 1e3, "triplets_per_sec": B / t, "bytes_per_triplet": BYTES[k],
                         "GB_per_s": B * BYTES[k] / t / 1e9, "share_of_3.35TBps": B * BYTES[k] / t / HBM_BYTES_PER_S,
                         "check_max_rel_err": checks[k], "rounds_step_ms": [x * 1e3 for x in ts]}
    del paths
    torch.cuda.empty_cache()
    res["dlrm"] = "not measured" if args.no_dlrm else dlrm(torch, args.dlrm_steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
