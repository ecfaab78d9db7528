"""GPU: DLRM kernels and model vs the oracle / the golden vectors recorded from the reference's dlrm.py."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import openrec_oracle as O
from openrec_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def tf():
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def close(t, ref, atol=1e-5, rtol=1e-5):
    got = t.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(t) else np.asarray(t, dtype=np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol)


# ---- Dense-layer GEMMs ------------------------------------------------------------------------------------------
# Every GEMM launch is checked twice: the handle's dispatch record must name the kernel, operand layout and split-K count
# that the dispatch rule below gives, and the result must be within the error model of that kernel.  The error is
# normalised per output, e = max |C - C64| / (|A| |B|), so that a small output of a row of tiny values is held to the
# same relative bar as a large one:
#  - k_gemm_tma (3xTF32, accumulator folded every 64 K-elements): e <= 2^-18;
#  - k_gemm (fp32 SIMT, one sequential sum per output and split): e <= C_SIMT 2^-24 sqrt(K).
E_TC = 2.0 ** -18
C_SIMT = 8.0
TMA, SIMT = L.ORX_VARIANT_GEMM_TMA, L.ORX_VARIANT_GEMM_SIMT


def _cdiv(a, b):
    return -(-a // b)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gemm_rule(TA, TB, M, N, K, lda, ldb, aligned, sms):
    """(variant, S) of C[M,N] = op(A)[M,K] op(B)[K,N]: orx_launch_gemm_tc takes what the TMA can describe and fills a
    tile, launch_gemm (SIMT) the rest; both split K when the tiles do not fill the machine and K is long."""
    if not (TA and TB) and N >= 16 and K >= 8 and M >= 64 and lda % 4 == 0 and ldb % 4 == 0 and aligned:
        tiles, nkb, S = _cdiv(N, 128) * _cdiv(M, 128), _cdiv(K, 16), 1
        if tiles < sms and nkb >= 32:
            S = max(1, min(_cdiv(2 * sms, tiles), nkb // 8))
        return TMA, S
    tiles, S = _cdiv(N, 64) * _cdiv(M, 64), 1
    if tiles < sms and K >= 1024:
        S = min(_cdiv(2 * sms, tiles), K // 256, 65535)
    return SIMT, S


def _layer_gemms(B, inn, out, ldx, ldw, lddy, x_ptr, w_ptr, dy_ptr, sms, want_dx=True):
    """The GEMMs of one orx_mlp_layer_fwd + orx_mlp_layer_bwd call, in launch order: (TA, TB, M, N, K, variant, S)."""
    al = lambda *p: all(q % 16 == 0 for q in p)
    calls = [(0, 0, B, out, inn, ldx, ldw, al(x_ptr, w_ptr)),          # y = x w
             (1, 0, inn, out, B, ldx, lddy, al(x_ptr, dy_ptr))]        # dw = x^T dz
    if want_dx:
        calls.append((0, 1, B, inn, out, lddy, ldw, al(dy_ptr, w_ptr)))   # dx = dz w^T
    return [(TA, TB, M, N, K) + _gemm_rule(TA, TB, M, N, K, lda, ldb, a, sms) for TA, TB, M, N, K, lda, ldb, a in calls]


def _f64(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _check_dispatch(eng, expect):
    from openrec_b200.native import Dispatch
    got = eng.debug_dispatch_log()
    want = [Dispatch(L.ORX_OP_GEMM, v, TA, TB, M, N, K, S) for TA, TB, M, N, K, v, S in expect]
    assert got == want


def _gemm_err(case, what, t, ref, scale, variant, K):
    got = _f64(t)
    assert np.isfinite(got).all(), f"{case} {what}: non-finite output"
    e = float(np.max(np.abs(got - ref) / np.maximum(scale, 1e-30)))
    bar = E_TC if variant == TMA else C_SIMT * 2.0 ** -24 * np.sqrt(K)
    print(f"gemm-error {case} {what} {'k_gemm_tma' if variant == TMA else 'k_gemm'} K={K} e={e:.3e} bar={bar:.3e}")
    assert e <= bar, (case, what, e, bar)
    return e


def _run_layer(eng, case, tx, tw, tb, act, ty, tdy, tdx, bwd=True, atol=False):
    """orx_mlp_layer_fwd, then orx_mlp_layer_bwd, on the given views (any leading dimension); checks the dispatch record
    of every GEMM and y, dw, dx, db against the float64 oracle on the float32 inputs."""
    B, inn = tx.shape
    out = tw.shape[1]
    x, w = _f64(tx), _f64(tw)
    b = _f64(tb) if tb is not None else None
    name = {0: None, 1: "relu", 2: "sigmoid"}[act]
    gemms = _layer_gemms(B, inn, out, tx.stride(0), tw.stride(0), tdy.stride(0), tx.data_ptr(), tw.data_ptr(),
                         tdy.data_ptr(), _sms(), tdx is not None)
    eng.debug_dispatch_log()
    eng.mlp_fwd(tx, tw, tb, act, ty)
    _check_dispatch(eng, gemms[:1])
    y_ref = O.mlp_forward(x, [w], [b], "relu", name)[0]
    if act == 2:                                   # sigmoid: an absolute bar on the activation output
        close(ty, y_ref, atol=2e-5)
    else:                                          # relu is 1-Lipschitz: the normalised bar holds through it
        _gemm_err(case, "y", ty, y_ref, np.abs(x) @ np.abs(w) + (np.abs(b) if b is not None else 0), gemms[0][5], inn)
    if atol:
        close(ty, y_ref, atol=2e-5)
    if not bwd:
        return
    # backward from the oracle's y: a relu mask taken from the kernel's own y flips on |y| ~ 1e-7 ties (seen at B = 8192)
    ty.copy_(torch.as_tensor(y_ref, dtype=torch.float32))
    y, dy = _f64(ty), _f64(tdy)
    tdw, tdb = torch.empty_like(tw), (torch.empty(out, device="cuda") if tb is not None else None)
    eng.mlp_bwd(tx, ty, tw, act, tdy, tdx, tdw, tdb)
    _check_dispatch(eng, gemms[1:])
    dx_ref, (dw_ref,), (db_ref,) = O.mlp_backward(x, [w], [y], dy, "relu", name)
    dz = np.abs(O._act_bwd(y, dy, name))
    _gemm_err(case, "dw", tdw, dw_ref, np.abs(x).T @ dz, gemms[1][5], B)
    if tdx is not None:
        _gemm_err(case, "dx", tdx, dx_ref, dz @ np.abs(w).T, gemms[2][5], out)
    if tdb is not None:
        close(tdb, db_ref, atol=1e-4)
    if atol:
        if tdx is not None:
            close(tdx, dx_ref, atol=5e-5)
        close(tdw, dw_ref, atol=2e-4, rtol=1e-4)


LAYER_CASES = [(37, 13, 8, 1), (300, 479, 96, 2), (1000, 64, 1, 0), (129, 5, 130, 1), (512, 256, 128, 1),
               (1111, 479, 1024, 1), (4096, 512, 256, 0), (200, 13, 512, 1), (777, 1024, 64, 2),
               (8192, 13, 512, 1), (8192, 256, 1, 2), (6000, 300, 200, 1),   # split-K / split col-sum
               # tensor-core tile and K tails: M 64/65/127/128/129, N 16/20/132, K 8/16/20/64/68/1028, nkb = 1, nkb % 4 != 0
               (64, 64, 128, 0), (65, 20, 132, 1), (127, 16, 20, 0), (128, 8, 16, 1), (200, 68, 20, 0),
               (129, 68, 17, 0),                                 # N = 17: ld % 4 != 0 -> SIMT for all three
               (300, 65, 128, 1),                                # K = 65: ldx % 4 != 0 -> SIMT forward and dw
               (256, 1028, 128, 1), (129, 1024, 64, 2),          # forward split-K, bias + relu / sigmoid in the reduce
               (256, 128, 1028, 0),                              # dx split-K
               (37, 1024, 8, 1), (200, 13, 1024, 0)]             # SIMT split-K of the forward / of dx


@pytest.mark.parametrize("B,inn,out,act", LAYER_CASES)
def test_mlp_layer_fwd_bwd(B, inn, out, act):
    from openrec_b200 import native as N
    eng = N.engine()
    rng = np.random.default_rng(B * 7 + inn)
    x, w, b = rng.standard_normal((B, inn)), rng.standard_normal((inn, out)) * 0.3, rng.standard_normal(out) * 0.1
    dy = rng.standard_normal((B, out))
    _run_layer(eng, f"{B}x{inn}x{out}", dev(x), dev(w), dev(b), act, torch.empty(B, out, device="cuda"), dev(dy),
               torch.empty(B, inn, device="cuda"), atol=True)


def test_gemm_dispatch_coverage():
    """The cases above reach every kernel / operand layout / split-K combination the dispatch can choose."""
    sms, seen = _sms(), set()
    for B, inn, out, _ in LAYER_CASES:
        for TA, TB, _, _, _, v, S in _layer_gemms(B, inn, out, inn, out, out, 0, 0, 0, sms):
            seen.add((v, TA, TB, S > 1))
    want = {(v, TA, TB, split) for v in (TMA, SIMT) for TA, TB in ((0, 0), (1, 0), (0, 1)) for split in (False, True)}
    assert seen == want, sorted(want - seen)


def test_gemm_splitk_empty_last_split():
    """A split-K forward whose last split has no k-block (it must contribute zeros, not stale workspace)."""
    from openrec_b200 import native as N
    eng = N.engine()
    B, out, sms = 128, 128, _sms()                  # one tile
    for nkb in range(32, 1 << 16):                  # the first K (with a K tail, ld % 4 == 0) whose last split is empty
        S = max(1, min(_cdiv(2 * sms, 1), nkb // 8))
        if S > 1 and (S - 1) * _cdiv(nkb, S) >= nkb:
            break
    inn = 16 * nkb - 8
    assert _gemm_rule(0, 0, B, out, inn, inn, out, True, sms) == (TMA, S)
    rng = np.random.default_rng(81)
    # a first, larger split-K GEMM leaves non-zero partials in the workspace the empty split would otherwise expose
    big = dev(rng.standard_normal((B, inn + 512)))
    eng.mlp_fwd(big, dev(rng.standard_normal((inn + 512, out))), None, 0, torch.empty(B, out, device="cuda"))
    _run_layer(eng, f"empty-split nkb={nkb} S={S}", dev(rng.standard_normal((B, inn))),
               dev(rng.standard_normal((inn, out)) * 0.3), dev(rng.standard_normal(out) * 0.1), 1,
               torch.empty(B, out, device="cuda"), dev(rng.standard_normal((B, out))), torch.empty(B, inn, device="cuda"))


def _nan_rows(B, n, ld):
    """[B, n] view of a NaN-filled [B, ld] buffer, and the buffer."""
    buf = torch.full((B, ld), float("nan"), device="cuda")
    return buf[:, :n], buf


def _assert_nan_padding(buf, n):
    pad = buf[:, n:]
    assert torch.equal(pad.view(torch.int32), torch.full_like(pad, float("nan")).view(torch.int32))


def test_mlp_layer_dlrm_layout():
    """DLRMGraph's operands: x = top_in (479 columns, ld = 480), y into a column slice of a wider buffer, dx into
    d_top_in-shaped storage; NaN in every padding column must neither reach a result nor be overwritten."""
    from openrec_b200 import native as N
    from openrec_b200.tf2.mlp_ops import _rows
    eng = N.engine()
    B, inn, out = 1000, 479, 128
    ld = _rows(1, inn, "cuda").stride(0)
    assert ld == 480
    rng = np.random.default_rng(479)
    tx, xbuf = _nan_rows(B, inn, ld)
    tx.copy_(dev(rng.standard_normal((B, inn))))
    ty, ybuf = _nan_rows(B, out, ld)
    tdx, dxbuf = _nan_rows(B, inn, ld)
    _run_layer(eng, "dlrm-layout", tx, dev(rng.standard_normal((inn, out)) * 0.1), dev(rng.standard_normal(out) * 0.1),
               1, ty, dev(rng.standard_normal((B, out))), tdx)
    for buf, n in ((xbuf, inn), (ybuf, out), (dxbuf, inn)):
        _assert_nan_padding(buf, n)


def test_mlp_layer_misaligned_base():
    """x starts one float into its buffer (ld % 4 == 0): the TMA cannot take it, the SIMT kernel must."""
    from openrec_b200 import native as N
    eng = N.engine()
    B, inn, out = 300, 128, 64
    rng = np.random.default_rng(5)
    buf = torch.empty(B * inn + 4, device="cuda")
    tx = buf[1:1 + B * inn].view(B, inn)
    tx.copy_(dev(rng.standard_normal((B, inn))))
    assert tx.data_ptr() % 16 == 4
    gemms = _layer_gemms(B, inn, out, inn, out, out, tx.data_ptr(), 0, 0, _sms())
    assert [g[5] for g in gemms] == [SIMT, SIMT, TMA]
    _run_layer(eng, "misaligned", tx, dev(rng.standard_normal((inn, out)) * 0.3), dev(rng.standard_normal(out) * 0.1),
               0, torch.empty(B, out, device="cuda"), dev(rng.standard_normal((B, out))), torch.empty(B, inn, device="cuda"))


@pytest.mark.parametrize("which", ["fwd", "dw"])
def test_gemm_long_k_positive_operands(which):
    """A, B ~ U(0, 1), K = 8192: every product has the same sign, so a truncating accumulator that is never folded
    into round-to-nearest fp32 shows up as an error growing with K.  'fwd': enough tiles for the machine, so there is
    no split and one CTA sums all 512 k-blocks; 'dw': the same through the split-K weight gradient."""
    from openrec_b200 import native as N
    eng = N.engine()
    sms, K = _sms(), 8192
    rng = np.random.default_rng(8192)
    if which == "fwd":
        side = 128 * int(np.ceil(np.sqrt(sms)))
        B, inn, out = side, K, side
        assert _gemm_rule(0, 0, B, out, inn, inn, out, True, sms) == (TMA, 1)
    else:
        B, inn, out = K, 256, 128
        assert _gemm_rule(1, 0, inn, out, B, inn, out, True, sms)[1] > 1
    u = lambda *s: dev(rng.random(s))
    _run_layer(eng, f"positive-{which}", u(B, inn), u(inn, out), u(out), 0, torch.empty(B, out, device="cuda"),
               u(B, out), torch.empty(B, inn, device="cuda") if which == "dw" else None, bwd=which == "dw")


def test_gemm_row_dynamic_range():
    """Rows of x (and of dy) scaled by 2^20 and 2^-20 in turn: the error must be small relative to each output's own
    magnitude, which an absolute tolerance set by the large rows would not see."""
    from openrec_b200 import native as N
    eng = N.engine()
    B, inn, out = 1000, 256, 128
    rng = np.random.default_rng(20)
    scale = np.where(np.arange(B) % 2 == 0, 2.0 ** 20, 2.0 ** -20)[:, None]
    _run_layer(eng, "row-range", dev(rng.standard_normal((B, inn)) * scale), dev(rng.standard_normal((inn, out)) * 0.3),
               None, 0, torch.empty(B, out, device="cuda"), dev(rng.standard_normal((B, out)) * scale),
               torch.empty(B, inn, device="cuda"))


@pytest.mark.parametrize("self_int", [False, True])
@pytest.mark.parametrize("mode", ["reference", "dlrm"])
def test_interaction_fwd_bwd(golden_dir, self_int, mode):
    from openrec_b200 import native as N
    from openrec_b200.tf2.mlp_ops import interaction_width
    eng = N.engine()
    rng = np.random.default_rng(3)
    B, F, D = 50, 27, 16
    feats = [rng.standard_normal((B, D)).astype(np.float32).astype(np.float64) for _ in range(F)]
    ref = O.second_order_interaction(feats, self_int, mode)
    P = interaction_width(F, self_int)
    emb = dev(np.stack(feats[:-1], 1))
    dense = dev(feats[-1])
    out = torch.empty(B, P, device="cuda")
    eng.interact_fwd(emb, dense, self_int, 0 if mode == "reference" else 1, out)
    close(out, ref, atol=2e-5)
    dout = rng.standard_normal((B, P)).astype(np.float32).astype(np.float64)
    dZ = O.second_order_interaction_bwd(feats, dout, self_int, mode)
    demb, ddense = torch.empty_like(emb), torch.full_like(dense, 0.5)     # ddense is accumulated into
    eng.interact_bwd(emb, dense, dev(dout), self_int, 0 if mode == "reference" else 1, demb, ddense)
    close(demb, dZ[:, :F - 1, :], atol=5e-5), close(ddense, dZ[:, F - 1, :] + 0.5, atol=5e-5)
    if mode == "reference":   # the golden recorded from the reference's own layer (F=5, D=7)
        g = dict(np.load(os.path.join(golden_dir, "interaction.npz")))
        f = [g[f"in{k}"] for k in range(5)]
        o = torch.empty(6, interaction_width(5, self_int), device="cuda")
        eng.interact_fwd(dev(np.stack(f[:-1], 1)), dev(f[-1]), self_int, 0, o)
        close(o, g[f"out_self{int(self_int)}"], atol=2e-5)


# ---- interaction: the warp fast path at its limits and the generic path, against the float64 oracle -----------------
# e = max |out - ref| / (|Z| |Z|^T) (bwd: / ((|dP| + |dP|^T) |Z|)), an fp32 dot product of length D (F) per output.
C_INTER = 8.0


def _inter_err(what, got, ref, scale, n):
    got = _f64(got)
    assert np.isfinite(got).all(), what
    e = float(np.max(np.abs(got - ref.reshape(got.shape)) / np.maximum(scale.reshape(got.shape), 1e-30)))
    assert e <= C_INTER * 2.0 ** -24 * np.sqrt(n), (what, e)


def _interaction_check(eng, Z, emb, dense, out, dout, demb, ddense, self_int, mode, variant):
    """fwd + bwd on the given views (Z [B, F, D] float32 holds the same features, the dense vector last); ddense must
    already hold the values the gradient is added to."""
    from openrec_b200.native import Dispatch
    B, F, D = Z.shape
    m = 0 if mode == "reference" else 1
    feats = [Z[:, f].astype(np.float64) for f in range(F)]
    afeats = [np.abs(f) for f in feats]
    eng.debug_dispatch_log()
    eng.interact_fwd(emb, dense, self_int, m, out)
    assert eng.debug_dispatch_log() == [Dispatch(L.ORX_OP_INTERACT_FWD, variant, 0, 0, B, F, D, 1)]
    _inter_err("fwd", out, O.second_order_interaction(feats, self_int, mode),
               O.second_order_interaction(afeats, self_int, mode), D)
    g = _f64(dout)
    pre = _f64(ddense)
    eng.interact_bwd(emb, dense, dout, self_int, m, demb, ddense)
    assert eng.debug_dispatch_log() == [Dispatch(L.ORX_OP_INTERACT_BWD, variant, 0, 0, B, F, D, 1)]
    dZ = O.second_order_interaction_bwd(feats, g, self_int, mode)
    scale = O.second_order_interaction_bwd(afeats, np.abs(g), self_int, mode)
    _inter_err("bwd emb", demb, dZ[:, :F - 1], scale[:, :F - 1], F)
    _inter_err("bwd dense (accumulated)", ddense, pre + dZ[:, F - 1], np.abs(pre) + scale[:, F - 1], F)


def _interaction_case(B, F, D, self_int, mode, variant, seed):
    from openrec_b200 import native as N
    from openrec_b200.tf2.mlp_ops import interaction_width
    eng = N.engine()
    rng = np.random.default_rng(seed)
    Z = rng.standard_normal((B, F, D)).astype(np.float32)
    emb, dense = dev(Z[:, :F - 1]), dev(Z[:, F - 1])
    P = interaction_width(F, self_int)
    _interaction_check(eng, Z, emb, dense, torch.full((B, P), float("nan"), device="cuda"),
                       dev(rng.standard_normal((B, P))), torch.full_like(emb, float("nan")),
                       dev(rng.standard_normal((B, D))), self_int, mode, variant)


@pytest.mark.parametrize("self_int", [False, True])
@pytest.mark.parametrize("F", [2, 9, 10, 27, 28, 32])
@pytest.mark.parametrize("D", [4, 124, 128])
def test_interaction_warp_path(D, F, self_int):
    """k_interact_{fwd,bwd}_warp: D = 4 (one active lane) to 128 (all 32), F = 2 .. 32 (nine-row blocks that do and do
    not divide F); B is not a multiple of the 4 samples of a CTA and exceeds one grid, so the grid-stride loop runs."""
    B = 5003
    assert B > 4 * 4 * _sms()
    _interaction_case(B, F, D, self_int, "dlrm", L.ORX_VARIANT_INTERACT_WARP, 100 * F + D)


@pytest.mark.parametrize("D,F,mode", [(13, 27, "dlrm"), (256, 27, "dlrm"), (128, 33, "dlrm"), (128, 27, "reference")])
@pytest.mark.parametrize("self_int", [False, True])
def test_interaction_generic_path(D, F, mode, self_int):
    _interaction_case(777, F, D, self_int, mode, L.ORX_VARIANT_INTERACT, 7 * F + D)


@pytest.mark.parametrize("self_int", [False, True])
def test_interaction_dlrm_graph_layout(self_int):
    """DLRMGraph's views: dense = top_in[:, :D], out = top_in[:, D:] (top_in from _rows, padded to a multiple of 4
    floats), ddense = d_top_in[:, :D] holding the bottom MLP's gradient, which the interaction adds to."""
    from openrec_b200 import native as N
    from openrec_b200.tf2.mlp_ops import _rows, interaction_width
    eng = N.engine()
    B, T, D = 4099, 26, 128
    W = D + interaction_width(T + 1, self_int)
    ld = _rows(1, W, "cuda").stride(0)
    assert ld > W                                   # 479 -> 480, 506 -> 508: there is a padding column
    rng = np.random.default_rng(T)
    Z = rng.standard_normal((B, T + 1, D)).astype(np.float32)
    top_in, tbuf = _nan_rows(B, W, ld)
    d_top_in, dbuf = _nan_rows(B, W, ld)
    top_in[:, :D] = dev(Z[:, T])
    d_top_in[:, D:] = dev(rng.standard_normal((B, W - D)))
    d_top_in[:, :D] = dev(rng.standard_normal((B, D)))
    emb = dev(Z[:, :T])
    _interaction_check(eng, Z, emb, top_in[:, :D], top_in[:, D:], d_top_in[:, D:], torch.empty_like(emb),
                       d_top_in[:, :D], self_int, "dlrm", L.ORX_VARIANT_INTERACT_WARP)
    _assert_nan_padding(tbuf, W)
    _assert_nan_padding(dbuf, W)


# ---- prediction loss (orx_pred_loss): clip, MSE / BCE, the masked gradients, the grid-stride loop ---------------------
@pytest.mark.parametrize("clip", [0.0, 0.3])
@pytest.mark.parametrize("kind", ["mse", "bce"])
@pytest.mark.parametrize("B", [1, 255, 257, 70_000])
def test_pred_loss(B, kind, clip):
    from openrec_b200 import native as N
    eng = N.engine()
    rng = np.random.default_rng(B)
    f32 = np.float32
    p = rng.uniform(-0.05, 1.05, B).astype(f32)
    lo, hi = f32(clip), f32(1) - f32(clip)          # the clip bounds as the kernel computes them (float32)
    # on the clip bounds (kept) and one float32 step outside them (masked); BCE: outside [1e-7, 1 - 1e-7] (masked) and
    # just inside it
    special = [lo, hi, np.nextafter(lo, f32(0)), np.nextafter(hi, f32(1)), f32(0), f32(3e-8), f32(2e-7),
               f32(0.9999998), f32(0.99999994), f32(1)]
    n = min(B, len(special))
    p[:n] = np.array(special[:n], dtype=f32)
    label = rng.random(B).astype(f32)               # fractional labels
    keep = np.ones(B, dtype=bool)
    pc = p
    if 0.0 < clip < 1.0:
        keep = (p >= lo) & (p <= hi)
        pc = np.clip(p, lo, hi)
        assert keep[:2].all() and (B < 4 or not keep[2:4].any())
    loss_ref, d_ref = O.dlrm_loss(pc.astype(np.float64), label.astype(np.float64), kind)
    d_ref = d_ref * keep
    if kind == "bce":
        # BCE evaluates the log at p clipped to [1e-7, 1 - 1e-7] in float32, as Keras does; 1 - 1e-7 is not a float32
        # (it rounds to 1 - 2^-23), and log(1 - p + 1e-7) there differs by 0.1 from its float64 value: the loss is
        # taken at the float32 bounds
        ph = np.clip(pc, f32(1e-7), f32(1) - f32(1e-7)).astype(np.float64)
        loss_ref = O.dlrm_loss(ph, label.astype(np.float64), kind)[0]
        # the oracle's float64 test of [1e-7, 1 - 1e-7] agrees with the kernel's float32 one on these inputs
        inside = (pc >= f32(1e-7)) & (pc <= f32(1) - f32(1e-7))
        pc64 = pc.astype(np.float64)
        assert np.array_equal(inside, (pc64 >= 1e-7) & (pc64 <= 1 - 1e-7))
    pred_out, dpred = torch.empty(B, device="cuda"), torch.full((B,), float("nan"), device="cuda")
    out4 = torch.zeros(4, device="cuda")
    eng.pred_loss(dev(p), dev(label), 0 if kind == "mse" else 1, clip, pred_out, dpred, out4)
    assert np.array_equal(pred_out.cpu().numpy(), pc)
    got = dpred.cpu().numpy()
    assert np.isfinite(got).all()
    assert (got[d_ref == 0] == 0).all()             # masked gradients are exactly zero
    close(got, d_ref, atol=1e-6 * np.abs(d_ref).max(), rtol=1e-5)
    close(float(out4[0]), loss_ref, atol=1e-7, rtol=1e-5)


def _load_golden_into(model, g):
    """Copy the golden's variables (creation order) into the model."""
    dense = g["dense"]
    model._graph(dense.shape[1])
    tv = model.trainable_variables
    assert len(tv) == int(g["n_vars"])
    for k, v in enumerate(tv):
        assert tuple(v.shape) == g[f"var{k}"].shape, (k, v.shape, g[f"var{k}"].shape)
        v.assign(g[f"var{k}"].astype(np.float32))
    return tv


@pytest.mark.parametrize("tag,kw", [("mse", {}), ("bce_self", dict(loss_func="bce", arch_interaction_itself=True)),
                                    ("clip", dict(loss_threshold=0.45)), ("bce", dict(loss_func="bce"))])
def test_dlrm_model_matches_reference_golden(tf, golden_dir, tag, kw):
    from openrec.tf2.recommenders import DLRM
    g = dict(np.load(os.path.join(golden_dir, f"dlrm_{tag}.npz")))
    model = DLRM(m_spa=4, ln_emb=[11, 7, 13], ln_bot=[8, 4], ln_top=[16, 8, 1], **kw)
    tv = _load_golden_into(model, g)
    close(model.inference(g["dense"].astype(np.float32), g["sparse"]).numpy(), g["pred"], atol=2e-6)
    with tf.GradientTape() as tape:
        loss = model(g["dense"].astype(np.float32), g["sparse"], g["label"])
    # 'bce_self': the self-interaction saturates the top sigmoid, and log(1 - p + 1e-7) at p -> 1 is only good to
    # ~1e-3 in float32 (the reference computes in float32 too; the golden is float64)
    saturated = tag == "bce_self"
    close(float(loss), g["loss"], atol=2e-6, rtol=2e-3 if saturated else 1e-5)
    grads = tape.gradient(loss, tv)
    for k, (gr, v) in enumerate(zip(grads, tv)):
        ref = g[f"grad{k}"]
        if gr.indices is not None:
            got = torch.zeros(v.shape, device="cuda").index_add_(0, gr.indices.t.long(), gr.values.t).cpu().numpy()
        else:
            got = gr.values.numpy()
        if saturated:   # 1 - p is not representable near p = 1 in float32 (the reference computes in float32 too):
            continue    # the gradient is ill-conditioned there; dlrm_bce.npz is the BCE parity case
        close(got, ref, atol=2e-6)


@pytest.mark.parametrize("optname,mode", [("adam", "reference"), ("sgd", "dlrm"), ("adagrad", "dlrm")])
def test_dlrm_training_step(tf, optname, mode):
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(21)
    B, m_spa, ln_emb = 256, 16, [50, 31, 77, 20]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=[32, m_spa], ln_top=[64, 32, 1], interaction_mode=mode)
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sparse = np.stack([rng.integers(0, n, B) for n in ln_emb], 1).astype(np.int64)     # un-cast ids (dataloader.py:75)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    var = [v.numpy().astype(np.float64) for v in tv]
    T = len(ln_emb)
    tabs, rest = var[:T], var[T:]
    bot_w, bot_b, top_w, top_b = [rest[0], rest[2]], [rest[1], rest[3]], rest[4::2], rest[5::2]
    opt = {"adam": tf.keras.optimizers.Adam(), "sgd": tf.keras.optimizers.SGD(learning_rate=0.1),
           "adagrad": tf.keras.optimizers.Adagrad(learning_rate=0.05)}[optname]
    kind = {"adam": O.OPT_ADAM_DENSE, "sgd": O.OPT_SGD, "adagrad": O.OPT_ADAGRAD}[optname]
    if kind == O.OPT_ADAGRAD:
        st = [(np.full_like(v, 0.1), None) for v in var]
    else:
        st = [(np.zeros_like(v), np.zeros_like(v)) for v in var]
    for step in (1, 2):
        with tf.GradientTape() as tape:
            loss = model(dense, sparse, label)
        grads = tape.gradient(loss, tv)
        opt.apply_gradients(zip(grads, tv))
        cache = O.dlrm_forward(tabs, bot_w, bot_b, list(top_w), list(top_b), dense.astype(np.float64), sparse,
                               interaction_mode=mode)
        rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
        gr = O.dlrm_backward(cache, tabs, bot_w, list(top_w), dense.astype(np.float64), sparse, dpred,
                             interaction_mode=mode)
        close(float(loss), rl, atol=2e-6)
        dense_grads = [gr["bot_w"][0], gr["bot_b"][0], gr["bot_w"][1], gr["bot_b"][1]]
        for l in range(len(top_w)):
            dense_grads += [gr["top_w"][l], gr["top_b"][l]]
        for k in range(T):
            O.apply_sparse(kind, var[k], st[k][0], st[k][1], sparse[:, k], gr["emb"][k], step, opt.learning_rate)
        for j, gd in enumerate(dense_grads):
            O.apply_dense(kind, var[T + j], st[T + j][0], st[T + j][1], gd, step, opt.learning_rate)
        for v, ref in zip(tv, var):
            close(v.numpy(), ref, atol=2e-5)
    if mode == "dlrm":
        assert np.abs(gr["emb"][0]).max() > 0      # the fixed interaction does train the tables


def test_dlrm_full_shape_training_step(tf):
    """BASELINE.json configs[3]: the Criteo shape (26 tables x 1M x 128, B = 32768, MLPs 13-512-256-128 and
    479-1024-1024-512-256-1, Adagrad): one training step through the class surface (TMA-fed wgmma Dense layers, warp
    interaction kernels, strided gathers / sparse applies) against the float64 oracle on the touched rows."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(33)
    B, m_spa, T = 32768, 128, 26
    ln_emb, ln_bot, ln_top = [1_000_000] * T, [512, 256, 128], [1024, 1024, 512, 256, 1]
    model = DLRM(m_spa=m_spa, ln_emb=ln_emb, ln_bot=ln_bot, ln_top=ln_top, interaction_mode="dlrm")
    dense = np.log1p(rng.integers(0, 100, (B, 13))).astype(np.float32)
    sparse = np.stack([rng.integers(0, n, B) for n in ln_emb], 1).astype(np.int64)
    label = (rng.random(B) < 0.3).astype(np.float32)
    model._graph(13)
    tv = model.trainable_variables
    assert len(tv) == T + 2 * (len(ln_bot) + len(ln_top))
    rows, csparse, tabs = [], np.zeros_like(sparse), []
    for k in range(T):                              # compact oracle problem: the touched rows of every table
        r = np.unique(sparse[:, k])
        rows.append(r)
        csparse[:, k] = np.searchsorted(r, sparse[:, k])
        tabs.append(tv[k].t[torch.from_numpy(r).cuda()].cpu().numpy().astype(np.float64))
    untouched = [int(np.setdiff1d(np.arange(2000), rows[k])[0]) for k in (0, T - 1)]
    before = [tv[k].t[u].clone() for k, u in zip((0, T - 1), untouched)]
    rest = [v.numpy().astype(np.float64) for v in tv[T:]]
    nb = len(ln_bot)
    bot_w, bot_b, top_w, top_b = rest[0:2 * nb:2], rest[1:2 * nb:2], rest[2 * nb::2], rest[2 * nb + 1::2]
    opt = tf.keras.optimizers.Adagrad(learning_rate=0.05)
    with tf.GradientTape() as tape:
        loss = model(dense, sparse, label)
    opt.apply_gradients(zip(tape.gradient(loss, tv), tv))
    cache = O.dlrm_forward(tabs, bot_w, bot_b, list(top_w), list(top_b), dense.astype(np.float64), csparse,
                           interaction_mode="dlrm")
    rl, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = O.dlrm_backward(cache, tabs, bot_w, list(top_w), dense.astype(np.float64), csparse, dpred, interaction_mode="dlrm")
    close(float(loss), rl, atol=2e-6)
    dense_grads = []
    for l in range(nb):
        dense_grads += [gr["bot_w"][l], gr["bot_b"][l]]
    for l in range(len(top_w)):
        dense_grads += [gr["top_w"][l], gr["top_b"][l]]
    for j, gd in enumerate(dense_grads):
        ref = rest[j]
        O.apply_dense(O.OPT_ADAGRAD, ref, np.full_like(ref, 0.1), None, gd, 1, 0.05)
        close(tv[T + j].numpy(), ref, atol=2e-5)
    assert np.abs(gr["emb"][0]).max() > 0
    for k in (0, 7, T - 1):
        O.apply_sparse(O.OPT_ADAGRAD, tabs[k], np.full_like(tabs[k], 0.1), None, csparse[:, k], gr["emb"][k], 1, 0.05)
        close(tv[k].t[torch.from_numpy(rows[k]).cuda()], tabs[k], atol=2e-5)
    for k, u, b in zip((0, T - 1), untouched, before):
        assert torch.equal(tv[k].t[u], b)          # rows outside the batch are bit-identical
