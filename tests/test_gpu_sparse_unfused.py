"""GPU parity of the un-fused sparse entry points (orx_pairwise_fwd / _grad, orx_pointwise_fwd / _grad) against the
float64 oracle, at dims below, at and above a warp's width, with batch tails (B not a multiple of the 8 samples per
warp) and bad ids (-1, the row count, 2^31 - 1).  A sample with a bad id is skipped: it adds nothing to the loss or the
l2 term and gets zero gradient rows and g_out = 0.  Also: a pointwise step with profiling on records its phases."""
import numpy as np
import pytest
import torch

from oracle import openrec_oracle as O
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

DIMS = (1, 12, 50, 128, 260)
U, I, B = 40, 60, 77
BAD = (-1, None, 2**31 - 1)   # None: the table's row count


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def close(t, ref, atol=1e-5, what=""):
    got = t.detach().cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=1e-5,
                               err_msg=what)


def _spoil(ids, rows, at):
    """ids with the three bad ids written at positions `at` (one per bad kind)."""
    ids = ids.copy()
    for pos, bad in zip(at, BAD):
        ids[pos] = rows if bad is None else bad
    return ids


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


# ---- pairwise ---------------------------------------------------------------------------------------------------------
def _pair_problem(kind, D):
    rng = np.random.default_rng([D, 0 if kind == "bpr" else 1])
    user, item, bias = (rng.uniform(-0.05, 0.05, s) for s in ((U, D), (I, D), (I, 1)))
    uid = _spoil(rng.integers(0, U, B).astype(np.int32), U, (0, 30, 76))
    pid = _spoil(rng.integers(0, I, B).astype(np.int32), I, (9, 41, 64))
    nid = _spoil(rng.integers(0, I, B).astype(np.int32), I, (17, 50, 71))
    return user, item, bias, uid, pid, nid


def _pair_grad(eng, kind, D, outs):
    """orx_pairwise_grad (c_loss 0.7, c_l2 0.3) writing only the outputs named in `outs` (the others NULL)."""
    user, item, bias, uid, pid, nid = _pair_problem(kind, D)
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    shapes = {"d_user": (B, D), "d_pos": (B, D), "d_neg": (B, D), "d_bp": (B,), "d_bn": (B,), "g_out": (B,)}
    got = {o: _nan(*shapes[o]) for o in outs}
    tabs = [dev(x) for x in (user, item, bias)]   # an orx_table_t holds no reference: keep the tensors alive
    eng.pairwise_grad(k, *(N.table(t) for t in tabs), *(dev(x, torch.int32) for x in (uid, pid, nid)), 0.5, 0.7, 0.3,
                      **got)
    torch.cuda.synchronize()
    return got


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_pairwise_unfused_vs_oracle(eng, kind, D):
    user, item, bias, uid, pid, nid = _pair_problem(kind, D)
    ok = (uid >= 0) & (uid < U) & (pid >= 0) & (pid < I) & (nid >= 0) & (nid < I)
    assert (~ok).sum() == 9
    v = np.flatnonzero(ok)
    nv = len(v)
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    out4 = _nan(4)
    tabs = [dev(x) for x in (user, item, bias)]
    eng.pairwise_fwd(k, *(N.table(t) for t in tabs), *(dev(x, torch.int32) for x in (uid, pid, nid)), out4, margin=0.5)
    # the oracle over the valid triplets; BPR's mean and gradient scale stay 1 / B of the whole batch
    ids = (uid[v], pid[v], nid[v])
    if kind == "bpr":
        loss, l2 = O.bpr_forward(user, item, bias, *ids)
        loss *= nv / B
        g = O.bpr_grads(user, item, bias, *ids, c_loss=0.7 * nv / B, c_l2=0.3)
    else:
        loss, l2 = O.ucml_forward(user, item, bias, *ids, margin=0.5)
        g = O.ucml_grads(user, item, bias, *ids, margin=0.5, c_loss=0.7, c_l2=0.3)
    close(out4[:2], [loss, l2], what="loss, l2")
    assert out4[2:].tolist() == [0.0, 0.0]

    got = _pair_grad(eng, kind, D, ("d_user", "d_pos", "d_neg", "d_bp", "d_bn", "g_out"))
    want = {"d_user": np.zeros((B, D)), "d_pos": np.zeros((B, D)), "d_neg": np.zeros((B, D)),
            "d_bp": np.zeros(B), "d_bn": np.zeros(B), "g_out": np.zeros(B)}
    want["d_user"][v] = g["user"][1]
    want["d_pos"][v], want["d_neg"][v] = g["item"][1][:nv], g["item"][1][nv:]
    gb = g["bias"][1].reshape(-1)
    want["d_bp"][v], want["d_bn"][v] = gb[:nv], gb[nv:]
    want["g_out"][v] = g["g"]
    for name, w in want.items():
        close(got[name], w, what=name)
        assert (got[name][torch.from_numpy(~ok).cuda()] == 0).all(), name   # skipped triplets: exact zeros


@pytest.mark.parametrize("out", ["d_user", "d_pos", "d_neg", "d_bp", "d_bn", "g_out"])
@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_pairwise_grad_one_output(eng, kind, out):
    full = _pair_grad(eng, kind, 50, ("d_user", "d_pos", "d_neg", "d_bp", "d_bn", "g_out"))
    alone = _pair_grad(eng, kind, 50, (out,))
    assert torch.equal(alone[out], full[out])


# ---- pointwise --------------------------------------------------------------------------------------------------------
def _point_problem(kind, D):
    rng = np.random.default_rng([D, 2 if kind == "gmf" else 3])
    user, item, bias, w = (rng.uniform(-0.3, 0.3, s) for s in ((U, D), (I, D), (I, 1), (1, D)))
    uid = _spoil(rng.integers(0, U, B).astype(np.int32), U, (0, 30, 76))
    iid = _spoil(rng.integers(0, I, B).astype(np.int32), I, (9, 41, 64))
    label = (rng.random(B) < 0.3).astype(np.float64)
    ab = (1.0, 1.0) if kind == "gmf" else (3.0, 0.5)
    return user, item, bias, w, uid, iid, label, ab


def _point_call(eng, kind, D, fn, *args, **kw):
    """eng.<fn> (pointwise_fwd / pointwise_grad) on the problem of (kind, D), then a device synchronise."""
    user, item, bias, w, uid, iid, label, (a, b) = _point_problem(kind, D)
    k = N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF
    tabs = [dev(x) for x in (user, item, bias, w)]   # an orx_table_t holds no reference: keep the tensors alive
    wt = N.table(tabs[3]) if kind == "gmf" else None
    getattr(eng, fn)(k, *(N.table(t) for t in tabs[:3]), wt, dev(uid, torch.int32), dev(iid, torch.int32), dev(label),
                     *args, a=a, b=b, **kw)
    torch.cuda.synchronize()


def _point_grad(eng, kind, D, outs):
    shapes = {"d_user": (B, D), "d_item": (B, D), "d_bias": (B,), "d_w": (D,), "g_out": (B,)}
    got = {o: _nan(*shapes[o]) for o in outs}
    _point_call(eng, kind, D, "pointwise_grad", use_sigmoid=False, c_loss=0.7, c_l2=0.3, **got)
    return got


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
def test_pointwise_unfused_vs_oracle(eng, kind, D):
    user, item, bias, w, uid, iid, label, (a, b) = _point_problem(kind, D)
    ok = (uid >= 0) & (uid < U) & (iid >= 0) & (iid < I)
    assert (~ok).sum() == 6
    v = np.flatnonzero(ok)
    out4 = _nan(4)
    _point_call(eng, kind, D, "pointwise_fwd", out4)
    ids = (uid[v], iid[v], label[v])
    if kind == "gmf":
        loss, l2 = O.gmf_forward(user, item, bias, w, *ids)
        loss *= len(v) / B
        g = O.gmf_grads(user, item, bias, w.reshape(-1, 1), *ids, c_loss=0.7 * len(v) / B, c_l2=0.3)
    else:
        loss, l2 = O.wrmf_forward(user, item, bias, *ids, a, b)
        g = O.wrmf_grads(user, item, bias, *ids, a, b, c_loss=0.7, c_l2=0.3)
    close(out4[:2], [loss, l2], atol=3e-5, what="loss, l2")
    assert out4[2:].tolist() == [0.0, 0.0]

    outs = ("d_user", "d_item", "d_bias", "g_out") + (("d_w",) if kind == "gmf" else ())
    got = _point_grad(eng, kind, D, outs)
    want = {"d_user": np.zeros((B, D)), "d_item": np.zeros((B, D)), "d_bias": np.zeros(B), "g_out": np.zeros(B)}
    want["d_user"][v], want["d_item"][v] = g["user"][1], g["item"][1]
    want["d_bias"][v], want["g_out"][v] = g["bias"][1].reshape(-1), g["g"]
    for name, wv in want.items():
        close(got[name], wv, atol=3e-5, what=name)
        assert (got[name][torch.from_numpy(~ok).cuda()] == 0).all(), name
    if kind == "gmf":
        close(got["d_w"], g["w"], atol=3e-5, what="d_w")


@pytest.mark.parametrize("kind,out", [(k, o) for k in ("gmf", "wrmf") for o in ("d_user", "d_item", "d_bias", "g_out")]
                         + [("gmf", "d_w")])
def test_pointwise_grad_one_output(eng, kind, out):
    full = _point_grad(eng, kind, 50, ("d_user", "d_item", "d_bias", "g_out") + (("d_w",) if kind == "gmf" else ()))
    alone = _point_grad(eng, kind, 50, (out,))
    if out == "d_w":   # summed with float atomics: the order of the additions varies from call to call
        close(alone[out], full[out].cpu().numpy(), atol=1e-6)
    else:
        assert torch.equal(alone[out], full[out])


# ---- profiling --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
def test_pointwise_step_profile(kind):
    """Every 8th pointwise step records the three phases of orx_profile_enable: index, step kernel, tail."""
    e = N.Engine(0)
    try:
        D = 64
        rng = np.random.default_rng(7)
        tabs = [dev(rng.uniform(-0.3, 0.3, s)) for s in ((U, D), (I, D), (I, 1), (1, D))]
        uid, iid = dev(rng.integers(0, U, B), torch.int32), dev(rng.integers(0, I, B), torch.int32)
        label = dev((rng.random(B) < 0.3).astype(np.float64))
        k = N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF
        wt = N.table(tabs[3]) if kind == "gmf" else None
        out4 = torch.zeros(4, device="cuda")
        e.profile_enable(True)
        for _ in range(17):
            e.pointwise_step(k, *(N.table(t) for t in tabs[:3]), wt, uid, iid, label, N.opt(N.ORX_OPT_SGD, 0.05), out4)
        ms, n = e.profile_read()
        e.profile_enable(False)
        assert n == 3, n   # steps 0, 8 and 16
        assert len(ms) == 3 and all(t > 0 for t in ms), ms
    finally:
        e.close()
