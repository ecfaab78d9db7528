"""Multi-hot DLRM benchmark: bench.py's DLRM workload (26 tables x 1M rows x 128, B = 32 768, the same MLPs,
interaction_mode='dlrm', Adagrad) with the MLPerf DLRM-DCNv2 multi-hot bag sizes (214 ids per sample).  Prints one JSON
line.

    python bench_dlrm_multihot.py [--window 1.0]

A step is DLRM(bag_sizes=...) + tf.GradientTape + Adagrad.apply_gradients.  Two id draws: "full" (uniform ids, every bag
full, pooling 'sum') and "ragged" (bag lengths uniform in 1 .. L_k, the rest -1 padding, pooling 'mean').  Reported per
draw: samples/s and ms/step (CUDA events over windows of at least --window seconds); orx_bag_gather's kernel time, its
achieved GB/s from the bytes it must move (valid lookups x D x 4 + the id block + Z) and that over the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s); the time of the 26 orx_bag_sparse_apply calls.  The one-hot DLRM step of
bench.py is timed in alternation with the multi-hot one, and the card name and power limit are read in the same run.
Before timing, one step of the full draw is checked against the float64 oracle on the touched rows of three tables, the
Dense layers and the loss (a mismatch exits non-zero).  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]
from bench import D, DLRM_B, DLRM_BOT, DLRM_DENSE, DLRM_LR, DLRM_T, DLRM_TOP, DLRM_VOCAB  # noqa: E402
from bench_eval import card  # noqa: E402

BAGS = [3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1]
HBM_GBS = 3350.0
CHECKED = (0, 9, 20)


def timed(fn, window):
    """ms per call: CUDA events around enough calls to fill `window` seconds."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    n = max(3, int(np.ceil(window * 1e3 / max(a.elapsed_time(b), 1e-3))))
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def draw(rng, ragged, n=4):
    col_off = np.concatenate([[0], np.cumsum(BAGS)])
    out = []
    for _ in range(n):
        sp = rng.integers(0, DLRM_VOCAB, (DLRM_B, col_off[-1]))
        if ragged:
            for k, L in enumerate(BAGS):
                length = rng.integers(1, L + 1, DLRM_B)
                sp[:, col_off[k]:col_off[k + 1]][np.arange(L)[None, :] >= length[:, None]] = -1
        out.append((torch.from_numpy(np.log1p(rng.integers(0, 100, (DLRM_B, DLRM_DENSE))).astype(np.float32)).cuda(),
                    torch.from_numpy(sp.astype(np.int32)).cuda(),
                    torch.from_numpy((rng.random(DLRM_B) < 0.25).astype(np.float32)).cuda()))
    return out, col_off


def make_step(tf, m, o):
    def train_step(d, s, y):
        with tf.GradientTape() as tape:
            loss = m(d, s, y)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
        return loss
    return train_step


def check_step(tf, model, opt, batch, col_off):
    """One step against the float64 oracle on the touched rows of CHECKED, the Dense layers and the loss."""
    import dlrm_bags_np as NB
    from oracle import openrec_oracle as O
    dense, sp_t, label = (t.cpu().numpy() for t in batch)
    sp = sp_t.astype(np.int64)
    tv = model.trainable_variables
    rows, csp, tabs = {}, np.zeros_like(sp), []
    for k in range(DLRM_T):                          # the touched rows of every table, as a compact problem
        cols = sp[:, col_off[k]:col_off[k + 1]]
        r = np.unique(cols[cols >= 0])
        rows[k] = r
        csp[:, col_off[k]:col_off[k + 1]] = np.where(cols >= 0, np.searchsorted(r, cols), -1)
        tabs.append(tv[k].t[torch.from_numpy(r).cuda()].cpu().numpy().astype(np.float64))
    dvars = [v.numpy().astype(np.float64) for v in tv[DLRM_T:]]
    loss = float(make_step(tf, model, opt)(*batch).numpy())
    st = [(np.full_like(v, 0.1) if k in CHECKED or k >= DLRM_T else None, None) for k, v in enumerate(tabs + dvars)]
    rl = NB.train_step(O.OPT_ADAGRAD, tabs, dvars, st, 1, DLRM_LR, dense.astype(np.float64), csp, label, col_off,
                       model._pooling == 1, "dlrm", len(DLRM_BOT), apply_tables=CHECKED)
    err_t = max(float(np.abs(tv[k].t[torch.from_numpy(rows[k]).cuda()].cpu().numpy() - tabs[k]).max()) for k in CHECKED)
    err_d = max(float(np.abs(v.numpy() - r).max()) for v, r in zip(tv[DLRM_T:], dvars))
    return {"loss": loss, "loss_oracle": float(rl), "max_abs_err_tables": err_t, "max_abs_err_dense": err_d,
            "passed": abs(loss - rl) <= 2e-6 + 1e-5 * abs(rl) and err_t <= 2e-5 and err_d <= 2e-5}


def kernel_parts(model, opt, batch, col_off, window):
    """orx_bag_gather alone (ms, bytes it must move) and the 26 orx_bag_sparse_apply calls (ms), with Adagrad."""
    from openrec_b200 import native as N
    eng = N.engine()
    _, sp, _ = batch
    tabs = [lf.embeddings.t for lf in model._latent_factors]
    Z = torch.empty(DLRM_B, DLRM_T * D, device="cuda")
    ms_gather = timed(lambda: eng.bag_gather(tabs, sp, col_off, model._pooling, Z), window)
    valid = int(((sp >= 0) & (sp < DLRM_VOCAB)).sum())
    nbytes = valid * D * 4 + sp.numel() * 4 + Z.numel() * 4
    dZ = torch.randn(DLRM_B, DLRM_T, D, device="cuda") * 1e-3
    o = N.opt(N.ORX_OPT_ADAGRAD, DLRM_LR)

    def applies():
        for k, lf in enumerate(model._latent_factors):
            eng.bag_sparse_apply(opt.table(lf.embeddings), sp, col_off[k], BAGS[k], dZ[:, k, :],
                                 model._pooling, o)
    ms_apply = timed(applies, window)
    return ms_gather, nbytes, valid, ms_apply


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dlrm_multihot.py needs a CUDA device")
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM
    vocab = [DLRM_VOCAB] * DLRM_T
    rng = np.random.default_rng(7)
    one = DLRM(m_spa=D, ln_emb=vocab, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm")
    one._graph(DLRM_DENSE)
    one_step = make_step(tf, one, tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR))
    one_data = [(d, torch.from_numpy(rng.integers(0, DLRM_VOCAB, (DLRM_B, DLRM_T)).astype(np.int32)).cuda(), y)
                for d, _, y in draw(rng, False, 2)[0]]
    result = {"metric": "dlrm_multihot_samples_per_sec", "unit": "samples/s", "gpus": 1, "batch": DLRM_B,
              "tables": f"{DLRM_T} x {DLRM_VOCAB} x {D}", "bag_sizes": BAGS, "ids_per_sample": sum(BAGS),
              "optimizer": f"Adagrad lr {DLRM_LR}", "hbm_peak_gbs_datasheet": HBM_GBS}
    check = None
    for name, ragged, pooling in (("full", False, "sum"), ("ragged", True, "mean")):
        model = DLRM(m_spa=D, ln_emb=vocab, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm",
                     bag_sizes=BAGS, pooling=pooling)
        model._graph(DLRM_DENSE)
        opt = tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)
        data, col_off = draw(rng, ragged)
        if not ragged:
            check = check_step(tf, model, opt, data[0], col_off)
            if not check["passed"]:
                print(json.dumps({"error": "the multi-hot step does not match the oracle", "check": check}))
                sys.exit(1)
        step = make_step(tf, model, opt)
        cnt = {"k": 0}

        def run(fn, batches):
            def go():
                fn(*batches[cnt["k"] % len(batches)])
                cnt["k"] += 1
            return go
        for _ in range(3):
            run(step, data)()
            run(one_step, one_data)()
        ms, ms_one = [], []
        for _ in range(3):          # alternate the multi-hot and the one-hot step
            ms.append(timed(run(step, data), args.window))
            ms_one.append(timed(run(one_step, one_data), args.window))
        ms_g, nbytes, valid, ms_a = kernel_parts(model, opt, data[0], col_off, args.window)
        best = min(ms)
        result[name] = {"pooling": pooling, "samples_per_sec": DLRM_B / (best * 1e-3), "ms_per_step": best,
                        "ms_per_step_windows": ms, "valid_lookups_per_step": valid,
                        "bag_gather_ms": ms_g, "bag_gather_bytes": nbytes,
                        "bag_gather_gbs": nbytes / (ms_g * 1e-3) / 1e9,
                        "bag_gather_share_of_hbm_peak": nbytes / (ms_g * 1e-3) / 1e9 / HBM_GBS,
                        "bag_sparse_apply_26_tables_ms": ms_a,
                        "one_hot_dlrm_ms_per_step_windows": ms_one,
                        "one_hot_dlrm_samples_per_sec": DLRM_B / (min(ms_one) * 1e-3)}
        del model, opt, step, data
        torch.cuda.empty_cache()
    result["value"] = result["full"]["samples_per_sec"]
    result["check"] = check
    result["card"], result["power_limit_w"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
