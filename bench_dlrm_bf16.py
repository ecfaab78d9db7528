"""bf16 embedding tables for DLRM: bench.py's DLRM (26 tables x 1M rows x 128, B = 32 768, the same MLPs,
interaction_mode='dlrm') with fp32 and bf16 tables.  Prints one JSON line.

    python bench_dlrm_bf16.py [--window 1.0]
    python bench_dlrm_bf16.py --quality

Cases: one-hot ids, and the MLPerf DLRM-DCNv2 multi-hot bags of bench_dlrm_multihot.py (full draw, pooling 'sum'); each
with Adagrad and RowwiseAdagrad.  For each (ids, optimizer) an fp32 and a bf16 model are built and their steps
alternated in windows of at least --window seconds (CUDA events), three rounds; the median is reported.  Before timing,
one step of the bf16 model is checked against the fp32 model holding its upcast tables: loss and Dense variables
bit-equal, every row of tables 0 and 20 touched once equal to orx_debug_round_bf16 of the fp32 row (a mismatch exits
non-zero).  Reported per configuration: step time and samples/s; the gather (orx_bag_gather, or the 26
orx_gather_strided calls) alone, with the bytes it must move (valid lookups x D x bytes per element + ids + Z) over
its time and as a share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s); the 26 applies alone; the bytes of
tables plus optimizer slots.  The card name and power limit are read in the same run.

--quality: a seeded synthetic click task (a planted logistic teacher over four small tables and 13 dense features).
DLRM with fp32 and with bf16 tables, from the same start and on the same batches, trained with Adagrad and with Keras
Adam(); reports held-out AUC (the Keras AUC metric) and the final training loss.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]
from bench import D, DLRM_B, DLRM_BOT, DLRM_DENSE, DLRM_LR, DLRM_T, DLRM_TOP, DLRM_VOCAB  # noqa: E402
from bench_dlrm_multihot import BAGS, HBM_GBS, make_step, timed  # noqa: E402
from bench_eval import card  # noqa: E402

CHECKED = (0, 20)


def batches(rng, multihot, n=3):
    C = sum(BAGS) if multihot else DLRM_T
    return [(torch.from_numpy(np.log1p(rng.integers(0, 100, (DLRM_B, DLRM_DENSE))).astype(np.float32)).cuda(),
             torch.from_numpy(rng.integers(0, DLRM_VOCAB, (DLRM_B, C)).astype(np.int32)).cuda(),
             torch.from_numpy((rng.random(DLRM_B) < 0.25).astype(np.float32)).cuda()) for _ in range(n)]


def touch_counts(sp, k, multihot):
    c = np.concatenate([[0], np.cumsum(BAGS)]) if multihot else np.arange(DLRM_T + 1)
    ids = sp[:, c[k]:c[k + 1]].reshape(-1)
    return np.bincount(ids[ids >= 0], minlength=DLRM_VOCAB)


def check_step(tf, bf, fp, opt_bf, opt_fp, batch, multihot):
    """One step of the bf16 model against the fp32 model on its upcast tables."""
    from openrec_b200 import native as N
    from openrec_b200.tf2.recommenders.dlrm import table_rounding_seed
    l_bf = float(make_step(tf, bf, opt_bf)(*batch).numpy())
    l_fp = float(make_step(tf, fp, opt_fp)(*batch).numpy())
    tb, tf_ = bf.trainable_variables, fp.trainable_variables
    dense_ok = all(torch.equal(a.t, b.t) for a, b in zip(tb[DLRM_T:], tf_[DLRM_T:]))
    sp = batch[1].cpu().numpy()
    rows_ok, n_rows = True, 0
    for k in CHECKED:
        once = torch.from_numpy(np.flatnonzero(touch_counts(sp, k, multihot) == 1)).cuda()
        n_rows += int(once.numel())
        r = N.engine().debug_round_bf16(tf_[k].t, 0, D, 0, table_rounding_seed(bf.rounding_seed, k), opt_bf.iterations)
        rows_ok = rows_ok and torch.equal(tb[k].t[once].view(torch.int16), r[once].view(torch.int16))
        del r
    return {"loss_bf16": l_bf, "loss_fp32": l_fp, "dense_bit_equal": dense_ok, "rows_touched_once_checked": n_rows,
            "rows_equal_rounded_fp32": rows_ok, "passed": l_bf == l_fp and dense_ok and rows_ok}


def parts(model, opt, batch, multihot, window, sr):
    """The gather alone (ms, bytes it must move, valid lookups) and the 26 applies alone (ms)."""
    from openrec_b200 import native as N
    from openrec_b200.tf2.recommenders.dlrm import table_rounding_seed
    eng = N.engine()
    _, sp, _ = batch
    tabs = [lf.embeddings.t for lf in model._latent_factors]
    esz = tabs[0].element_size()
    Z = torch.empty(DLRM_B, DLRM_T, D, device="cuda")
    col_off = [int(c) for c in np.concatenate([[0], np.cumsum(BAGS)])]
    if multihot:
        ms_g = timed(lambda: eng.bag_gather(tabs, sp, col_off, 0, Z.view(DLRM_B, DLRM_T * D)), window)
    else:
        ms_g = timed(lambda: [eng.gather_strided(t, sp, k, Z[:, k, :]) for k, t in enumerate(tabs)], window)
    valid = int((sp >= 0).sum())
    nbytes = valid * D * esz + sp.numel() * 4 + Z.numel() * 4
    dZ = torch.randn(DLRM_B, DLRM_T, D, device="cuda") * 1e-3
    o = opt.opt_struct()

    def applies():
        for k, lf in enumerate(model._latent_factors):
            kw = {"sr_seed": table_rounding_seed(0, k)} if sr else {}
            if multihot:
                eng.bag_sparse_apply(opt.table(lf.embeddings), sp, col_off[k], BAGS[k], dZ[:, k, :], 0, o, **kw)
            else:
                eng.sparse_apply_strided(opt.table(lf.embeddings), sp, k, dZ, o, **kw)
    return ms_g, nbytes, valid, timed(applies, window)


def state_bytes(model, opt):
    n = 0
    for lf in model._latent_factors:
        v = lf.embeddings
        n += v.t.numel() * v.t.element_size()
        n += sum(s.numel() * s.element_size() for s in opt.slots(v) if s is not None)
    return n


def speed(args, tf):
    from openrec_b200.tf2.recommenders import DLRM
    from openrec_b200.tfshim.keras.optimizers import RowwiseAdagrad
    mk_opt = {"adagrad": lambda: tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR),
              "rowwise": lambda: RowwiseAdagrad(learning_rate=DLRM_LR)}
    result = {"metric": "dlrm_bf16_tables_samples_per_sec", "unit": "samples/s", "gpus": 1, "batch": DLRM_B,
              "tables": f"{DLRM_T} x {DLRM_VOCAB} x {D}", "bag_sizes": BAGS, "hbm_peak_gbs_datasheet": HBM_GBS,
              "configs": {}, "checks": {}}
    rng = np.random.default_rng(7)
    for ids in ("onehot", "multihot"):
        multihot = ids == "multihot"
        data = batches(rng, multihot)
        for opt_name in ("adagrad", "rowwise"):
            kw = dict(m_spa=D, ln_emb=[DLRM_VOCAB] * DLRM_T, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, interaction_mode="dlrm",
                      bag_sizes=BAGS if multihot else None, pooling="sum")
            bf = DLRM(embedding_dtype="bfloat16", **kw)
            bf._graph(DLRM_DENSE)
            fp = DLRM(**kw)
            fp._graph(DLRM_DENSE)
            for a, b in zip(fp.trainable_variables, bf.trainable_variables):
                a.t.copy_(b.t)
            models = {"fp32": (fp, mk_opt[opt_name]()), "bf16": (bf, mk_opt[opt_name]())}
            chk = check_step(tf, bf, fp, models["bf16"][1], models["fp32"][1], data[0], multihot)
            result["checks"][f"{ids}/{opt_name}"] = chk
            if not chk["passed"]:
                print(json.dumps({"error": "the bf16 step does not round the fp32 step", "check": chk}))
                sys.exit(1)
            steps, cnt = {}, {"k": 0}
            for dt, (m, o) in models.items():
                st = make_step(tf, m, o)

                def go(st=st):
                    st(*data[cnt["k"] % len(data)])
                    cnt["k"] += 1
                steps[dt] = go
                for _ in range(2):
                    go()
            ms = {dt: [] for dt in models}
            for _ in range(3):               # alternate fp32 and bf16 windows
                for dt in models:
                    ms[dt].append(timed(steps[dt], args.window))
            for dt, (m, o) in models.items():
                ms_g, nbytes, valid, ms_a = parts(m, o, data[0], multihot, args.window, dt == "bf16")
                med = float(np.median(ms[dt]))
                result["configs"][f"{ids}/{opt_name}/{dt}"] = {
                    "ms_per_step": med, "ms_per_step_windows": ms[dt], "samples_per_sec": DLRM_B / (med * 1e-3),
                    "gather_ms": ms_g, "gather_bytes": nbytes, "valid_lookups": valid,
                    "gather_gbs": nbytes / (ms_g * 1e-3) / 1e9,
                    "gather_share_of_hbm_peak": nbytes / (ms_g * 1e-3) / 1e9 / HBM_GBS,
                    "applies_26_tables_ms": ms_a, "table_and_slot_bytes": state_bytes(m, o)}
            del models, steps, bf, fp
            torch.cuda.empty_cache()
    result["value"] = result["configs"]["multihot/adagrad/bf16"]["samples_per_sec"]
    result["card"], result["power_limit_w"] = card()
    return result


def quality(tf):
    """Synthetic clicks from a planted logistic teacher; fp32 and bf16 DLRM from the same start on the same batches."""
    from openrec_b200.tf2.recommenders import DLRM
    rng = np.random.default_rng(2024)
    vocab, m, B, steps = [5000, 2000, 500, 50], 16, 1024, 600
    teach = [rng.standard_normal((V, 4)) * 0.7 for V in vocab]
    w_teach, u_teach = rng.standard_normal((len(vocab), 4)), rng.standard_normal(DLRM_DENSE) * 0.3

    def draw(n):
        dense = rng.standard_normal((n, DLRM_DENSE)).astype(np.float32)
        sp = np.stack([np.minimum(rng.zipf(1.2, n) - 1, V - 1) for V in vocab], 1).astype(np.int32)
        logit = dense @ u_teach + sum((teach[k][sp[:, k]] * w_teach[k]).sum(1) for k in range(len(vocab))) - 0.5
        y = (rng.random(n) < 1 / (1 + np.exp(-logit))).astype(np.float32)
        return dense, sp, y
    train = [draw(B) for _ in range(steps)]
    held = [draw(B) for _ in range(20)]
    out = {"task": f"planted logistic teacher, tables {vocab}, m_spa {m}, B {B}, {steps} steps", "runs": {}}
    for opt_name in ("adagrad", "adam"):
        models = {}
        for dt in ("float32", "bfloat16"):
            models[dt] = DLRM(m_spa=m, ln_emb=vocab, ln_bot=[32, m], ln_top=[64, 32, 1], interaction_mode="dlrm",
                              loss_func="bce", embedding_dtype=dt, rounding_seed=1)
            models[dt]._graph(DLRM_DENSE)
        for a, b in zip(models["float32"].trainable_variables, models["bfloat16"].trainable_variables):
            a.t.copy_(b.t)
        for dt, model in models.items():
            opt = tf.keras.optimizers.Adagrad(learning_rate=0.05) if opt_name == "adagrad" else tf.keras.optimizers.Adam()
            step = make_step(tf, model, opt)
            losses = [float(step(*(torch.from_numpy(a).cuda() for a in b)).numpy()) for b in train]
            auc = tf.keras.metrics.AUC()
            for d, s, y in held:
                auc.update_state(y_true=y, y_pred=model.inference(d, s))
            out["runs"][f"{opt_name}/{dt}"] = {"held_out_auc": float(auc.result().numpy()),
                                               "final_loss_mean_last_50": float(np.mean(losses[-50:]))}
    out["card"], out["power_limit_w"] = card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    ap.add_argument("--quality", action="store_true", help="train the synthetic click task instead of timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dlrm_bf16.py needs a CUDA device")
    import tensorflow as tf
    print(json.dumps(quality(tf) if args.quality else speed(args, tf)))


if __name__ == "__main__":
    main()
