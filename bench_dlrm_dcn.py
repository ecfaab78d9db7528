"""DLRM-DCNv2 benchmark: bench.py's DLRM workload (26 tables x 1M rows x 128, B = 32 768, bottom 512-256-128, top
1024-1024-512-256-1, Adagrad) with the MLPerf DLRM-DCNv2 multi-hot bag sizes of bench_dlrm_multihot.py and the DCN-v2
cross network in place of the dot interaction: 3 cross layers of rank 512 over W = 27 x 128 = 3456 columns.  Prints
one JSON line.

    python bench_dlrm_dcn.py [--window 1.0]

A step is DLRM(arch_interaction_op="cross") + tf.GradientTape + Adagrad.apply_gradients.  Before timing, one step is
checked against a float64 restatement run on the device (tests/dcn_np.py): the loss, every Dense and cross variable and
the touched rows of three tables (a mismatch exits non-zero).  Then, with CUDA events over windows of at least --window
seconds, alternated with the 'dot' multi-hot step on the same bags:
  - step time and samples/s of both models.  The two models share one set of embedding tables and Adagrad slots
    (26.6 GB), so that both fit beside their activations; the output says so;
  - the cross GEMMs (the six projections' forward, dgrad and wgrad calls of orx_mlp_layer_fwd/bwd): time and TFLOP/s,
    against the 3xTF32 ceiling (the H100 SXM data sheet's 495 dense TF32 TFLOP/s / 3);
  - the cross kernels (3 orx_cross_fwd + 3 orx_cross_bwd + the final pass): time and GB/s from the operands they must
    move (B x W x 4 bytes each), against the data sheet's 3.35 TB/s;
  - device memory in use after a step, and its peak.
The card name and power limit are read in the same run.  Nothing is written to disk."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat"), os.path.join(ROOT, "tests")]
from bench import D, DLRM_B, DLRM_BOT, DLRM_DENSE, DLRM_LR, DLRM_T, DLRM_TOP, DLRM_VOCAB  # noqa: E402
from bench_dlrm_multihot import BAGS, HBM_GBS, draw, make_step, timed  # noqa: E402
from bench_eval import card  # noqa: E402

LAYERS, RANK = 3, 512
W = (DLRM_T + 1) * D
TF32_TFLOPS = 495.0
CHECKED = (0, 9, 20)
# operands (B x W floats) each cross pass reads + writes: forward x0, x_l, y -> x_{l+1}; TOP G, x0, y -> dy, A;
# MID G, P, x0, y, A -> G, dy, A; FINAL G, P, A -> dL/dx0
OPERANDS = LAYERS * 4 + 5 + (LAYERS - 1) * 8 + 4


def check_step(tf, model, opt, batch, col_off):
    """One step against the float64 restatement on the device: the loss, every Dense / cross variable, and the touched
    rows of CHECKED (Adagrad, initial accumulator 0.1)."""
    import dcn_np as X
    dense, sp, label = batch
    tv = model.trainable_variables
    d64 = lambda t: t.detach().to(torch.float64)
    embs, touched = [], {}
    for k in range(DLRM_T):
        cols = sp[:, col_off[k]:col_off[k + 1]].long()
        embs.append(d64(model._latent_factors[k].embeddings.t[cols]).sum(1))
        if k in CHECKED:
            touched[k] = (cols, d64(model._latent_factors[k].embeddings.t))
    dvars = [d64(v.t) for v in tv[DLRM_T:]]
    bw, bb, tw, tb, layers = X.split_dense(dvars, len(DLRM_BOT), len(DLRM_TOP), RANK)
    rl, dx0, grads = X.loss_and_grads_t(embs, bw, bb, tw, tb, layers, d64(dense), d64(label))
    del embs
    loss = float(make_step(tf, model, opt)(dense, sp, label).numpy())
    ada = lambda v, g: v - DLRM_LR * g / (torch.sqrt(0.1 + g * g) + 1e-7)
    err_d = max(float((v.t.to(torch.float64) - ada(r, g)).abs().max()) for v, r, g in zip(tv[DLRM_T:], dvars, grads))
    err_t = 0.0
    for k, (cols, tab) in touched.items():
        g = torch.zeros_like(tab)
        g.index_add_(0, cols.reshape(-1), dx0[:, D * (k + 1):D * (k + 2)].repeat_interleave(cols.shape[1], 0))
        rows = torch.unique(cols)
        err_t = max(err_t, float((model._latent_factors[k].embeddings.t[rows].to(torch.float64)
                                  - ada(tab[rows], g[rows])).abs().max()))
    return {"loss": loss, "loss_float64": rl, "max_abs_err_dense_and_cross": err_d, "max_abs_err_tables": err_t,
            "passed": abs(loss - rl) <= 2e-6 + 1e-5 * abs(rl) and err_d <= 2e-5 and err_t <= 2e-5}


def cross_parts(model, batch, window):
    """The cross network's GEMM calls and element-wise passes of one step, timed apart on the step's own activations:
    -> (GEMM ms, GEMM FLOP, kernels ms)."""
    from openrec_b200 import native as N
    from openrec_b200.tf2 import mlp_ops
    eng = N.engine()
    dense, sp, label = batch
    g = model._graph(DLRM_DENSE)
    c = g.forward(dense, sp, label, want_grad=True)
    B = dense.shape[0]
    x0, xs, acts = c["x0"], c["xs"], c["cross_acts"]
    G = torch.randn(B, W, device="cuda") * 1e-4
    dy, P, A = (torch.zeros(B, W, device="cuda") for _ in range(3))
    dh = torch.empty(B, RANK, device="cuda")
    dw = [[torch.empty_like(w) for w, _ in p] for p in g.cross]
    db = [torch.empty_like(p[1][1]) for p in g.cross]

    def gemms():                 # activation 0: orx_mlp_layer_bwd leaves its dy (here G) unchanged
        for l, p in enumerate(g.cross):
            (v, _), (u, b) = p
            eng.mlp_fwd(xs[l], v, None, 0, acts[l][0])
            eng.mlp_fwd(acts[l][0], u, b, 0, acts[l][1])
        for l in range(len(g.cross) - 1, -1, -1):
            (v, _), (u, b) = g.cross[l]
            eng.mlp_bwd(acts[l][0], acts[l][1], u, 0, G, dh, dw[l][1], db[l])
            eng.mlp_bwd(xs[l], acts[l][0], v, 0, dh, P, dw[l][0], None)
    flops = LAYERS * (2 * 2 * B * W * RANK + 4 * 2 * B * W * RANK)
    ms_gemm = timed(gemms, window)      # includes the bias column sums of the three U layers

    out = torch.empty(B, W, device="cuda")
    d_lo, dZ = mlp_ops._rows(B, D, x0.device), torch.empty(B, W - D, device="cuda")

    def kernels():
        for l in range(LAYERS):
            eng.cross_fwd(x0, xs[l], acts[l][1], out)
        for l in range(LAYERS - 1, -1, -1):
            eng.cross_bwd(N.ORX_CROSS_TOP if l == LAYERS - 1 else N.ORX_CROSS_MID, G, A, P=P, x0=x0, y=acts[l][1],
                          dy=dy)
        eng.cross_bwd(N.ORX_CROSS_FINAL, G, A, P=P, dx_lo=d_lo, dx_hi=dZ)
    ms_k = timed(kernels, window)
    return ms_gemm, flops, ms_k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of steps per timed window")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dlrm_dcn.py needs a CUDA device")
    import tensorflow as tf
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(11)
    kw = dict(m_spa=D, ln_bot=DLRM_BOT, ln_top=DLRM_TOP, bag_sizes=BAGS, pooling="sum")
    dcn = DLRM(ln_emb=[DLRM_VOCAB] * DLRM_T, arch_interaction_op="cross", cross_layers=LAYERS,
               cross_projection_dim=RANK, **kw)
    dot = DLRM(ln_emb=[1] * DLRM_T, interaction_mode="dlrm", **kw)
    dot._latent_factors = dcn._latent_factors           # one set of tables (and, through the optimizer, of slots)
    dcn._graph(DLRM_DENSE), dot._graph(DLRM_DENSE)
    opt = tf.keras.optimizers.Adagrad(learning_rate=DLRM_LR)
    data, col_off = draw(rng, False)
    check = check_step(tf, dcn, opt, data[0], col_off)
    if not check["passed"]:
        print(json.dumps({"error": "the DLRM-DCN step does not match float64", "check": check}))
        sys.exit(1)
    steps = {"dcn": make_step(tf, dcn, opt), "dot": make_step(tf, dot, opt)}
    cnt = {"k": 0}

    def run(name):
        def go():
            steps[name](*data[cnt["k"] % len(data)])
            cnt["k"] += 1
        return go
    for _ in range(3):
        run("dcn")(), run("dot")()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    run("dcn")()
    torch.cuda.synchronize()
    mem = {"allocated_gb_after_step": torch.cuda.memory_allocated() / 1e9,
           "peak_allocated_gb_in_step": torch.cuda.max_memory_allocated() / 1e9,
           "reserved_gb": torch.cuda.memory_reserved() / 1e9}
    ms = {"dcn": [], "dot": []}
    for _ in range(3):                                   # alternate the two steps
        for name in ("dcn", "dot"):
            ms[name].append(timed(run(name), args.window))
    ms_gemm, flops, ms_k = cross_parts(dcn, data[0], args.window)
    nbytes = OPERANDS * DLRM_B * W * 4
    best = min(ms["dcn"])
    result = {"metric": "dlrm_dcn_samples_per_sec", "unit": "samples/s", "value": DLRM_B / (best * 1e-3), "gpus": 1,
              "batch": DLRM_B, "tables": f"{DLRM_T} x {DLRM_VOCAB} x {D}", "bag_sizes": BAGS,
              "cross": f"{LAYERS} layers, rank {RANK}, W = {W}", "optimizer": f"Adagrad lr {DLRM_LR}",
              "shared_tables": "the dcn and dot models share one set of embedding tables and Adagrad slots",
              "ms_per_step": best, "ms_per_step_windows": ms["dcn"],
              "dot_multihot_ms_per_step_windows": ms["dot"],
              "dot_multihot_samples_per_sec": DLRM_B / (min(ms["dot"]) * 1e-3),
              "cross_gemm_ms": ms_gemm, "cross_gemm_tflop": flops / 1e12,
              "cross_gemm_tflops": flops / (ms_gemm * 1e-3) / 1e12,
              "cross_gemm_share_of_3xtf32_ceiling": flops / (ms_gemm * 1e-3) / 1e12 / (TF32_TFLOPS / 3),
              "cross_kernels_ms": ms_k, "cross_kernels_bytes": nbytes,
              "cross_kernels_gbs": nbytes / (ms_k * 1e-3) / 1e9,
              "cross_kernels_share_of_hbm_peak": nbytes / (ms_k * 1e-3) / 1e9 / HBM_GBS,
              "peaks_datasheet": {"tf32_dense_tflops": TF32_TFLOPS, "hbm_gbs": HBM_GBS},
              "memory": mem, "check": check}
    result["card"], result["power_limit_w"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
