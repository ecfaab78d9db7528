"""SGD with momentum (ORX_OPT_MOMENTUM) and Nesterov momentum (ORX_OPT_NESTEROV) on the GPU: every fused step, un-fused
apply, the home-routed sharded step and the Keras models that take them, judged against the float64 update under
tests/momentum_bar.py's bar, plus the cases that must be exact.

Fused steps run step_bar's arms at every specialised D and one generic D (50), on mixed, all-owned and all-staged
batches and batch tails, through orx_pairwise_step, _step_host, prefetched steps and orx_pointwise_step; each asserts the
kernel variant its dispatch record shows.  Exact: rows a run of steps never touches keep value and slot bit for bit;
with dyadic rows, slots, gradients, lr and momentum every path gives the float64 result bit for bit, and NESTEROV differs
from MOMENTUM by exactly m * a - lr * G - a."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import momentum_bar as MB
import step_bar as S
from _ranks import run_ranks
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N
from test_gpu_kernels import PAIR_OP, POINT_OP, SPECIAL_D, _point_rule, dev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOM, NEST = N.ORX_OPT_MOMENTUM, N.ORX_OPT_NESTEROV
ORX_ERR_INVALID = -1          # orx.h, orx_status
KINDS = {"bpr": N.ORX_PAIR_BPR, "ucml": N.ORX_PAIR_UCML, "gmf": N.ORX_POINT_GMF, "wrmf": N.ORX_POINT_WRMF}


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def _pair_rule(D):
    """(variant, CTAs/SM bound) of the momentum k_pair_step (orx_pairwise.cu launch_pair_step_kind_opt): the register
    double-buffer at D = 32 and 64, one buffer at 3 CTAs/SM at D = 128 and at 2 CTAs/SM at D = 256."""
    if D in (32, 64):
        return L.ORX_VARIANT_STEP_PIPE, 2
    if D == 128:
        return L.ORX_VARIANT_STEP, 3
    if D == 256:
        return L.ORX_VARIANT_STEP, 2
    return L.ORX_VARIANT_STEP_GENERIC, 0


def _check_dispatch(eng, op, kind, opt, B, D, index_set=0):
    """The one record of the step just launched: the variant of the rule, TB = the optimizer kind passed in."""
    v, minb = _pair_rule(D) if op == PAIR_OP else _point_rule(D)
    got = eng.debug_dispatch_log()
    assert len(got) == 1, got
    want = N.Dispatch(op, v, kind, opt, B, D, minb, got[0].s if index_set == "prefetch" else index_set)
    assert got[0] == want, (got[0], want)
    if index_set == "prefetch":
        assert got[0].s in (1, 2), got[0]
    return got[0].s


def _opt(c):
    return N.opt(c.opt, c.lr, eps=c.P["eps"], beta1=MB.momentum_of(c), beta2=c.P["beta2"], step=c.step)


class Dev:
    """A case's tables and momentum slots on the device."""

    def __init__(self, c):
        self.t = {n: [None if x is None else dev(x) for x in (c.tabs[n], *c.slots[n])] for n in c.names}
        self.tt = {n: N.table(*v) for n, v in self.t.items()}

    def got(self):
        torch.cuda.synchronize()
        return {n: tuple(None if x is None else x.cpu().numpy().astype(np.float64) for x in v)
                for n, v in self.t.items()}


def _pair_launch(eng, c, d, entry, dids=None):
    P = dict(margin=c.P["margin"], c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    out = torch.zeros(4, device="cuda")
    if entry == "host":
        ids = [torch.from_numpy(x).pin_memory() for x in c.ids]
        out = torch.zeros(4).pin_memory()
        eng.pairwise_step_host(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c), out, **P)
        torch.cuda.synchronize()
    else:
        eng.pairwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"],
                          *(dids or [dev(x, torch.int32) for x in c.ids]), _opt(c), out, **P)
    return out


def _point_launch(eng, c, d):
    out = torch.zeros(4, device="cuda")
    eng.pointwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], d.tt.get("w"),
                       *(dev(x, torch.int32) for x in c.ids), dev(c.label), _opt(c), out,
                       c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False),
                       c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    return out


def _sid(s):
    return "-".join(map(str, s))


# ---- fused steps ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", MB.pair_specs(), ids=_sid)
def test_momentum_pairwise_step(eng, spec):
    entry = spec[6]
    eng.debug_dispatch_log()
    if entry == "prefetch":
        sets = []
        for k in (0, 1):
            c = MB.build(spec, k)
            d = Dev(c)
            dids = [dev(x, torch.int32) for x in c.ids]
            torch.cuda.synchronize()
            eng.pairwise_prefetch(d.tt["user"], d.tt["item"], *dids, c.opt, ids_ready=True)
            _pair_launch(eng, c, d, "step", dids)
            sets.append(_check_dispatch(eng, PAIR_OP, KINDS[c.kind], c.opt, c.B, c.D, "prefetch"))
            MB.MomBar(c).check(d.got(), f"prefetched step {k}")
        assert sorted(sets) == [1, 2], sets
        return
    c = MB.build(spec)
    d = Dev(c)
    _pair_launch(eng, c, d, entry)
    _check_dispatch(eng, PAIR_OP, KINDS[c.kind], c.opt, c.B, c.D, "prefetch" if entry == "host" else 0)
    MB.MomBar(c).check(d.got(), entry)


@pytest.mark.parametrize("spec", MB.point_specs(), ids=_sid)
def test_momentum_pointwise_step(eng, spec):
    c = MB.build(spec)
    d = Dev(c)
    eng.debug_dispatch_log()
    _point_launch(eng, c, d)
    _check_dispatch(eng, POINT_OP, KINDS[c.kind], c.opt, c.B, c.D)
    MB.MomBar(c).check(d.got(), "pointwise step")


def test_momentum_dispatch_coverage():
    """The specs above reach every (op, variant, kind, optimizer, specialised D or generic, index set) combination,
    and batch tails at every specialised D and the generic one."""
    dcls = lambda D: D if D in SPECIAL_D else "generic"
    kinds = dict(KINDS, wrmf_sig=N.ORX_POINT_WRMF)
    seen = set()
    for arm, kind, o, D, B, ids, entry in MB.pair_specs():
        for s in ((0,) if entry == "step" else (1, 2) if entry == "prefetch" else ()):
            seen.add((PAIR_OP, _pair_rule(D)[0], kinds[kind], o, dcls(D), s))
    for arm, kind, o, D, B, ids, entry in MB.point_specs():
        seen.add((POINT_OP, _point_rule(D)[0], kinds[kind], o, dcls(D), 0))
    want = {(PAIR_OP, _pair_rule(D)[0], k, o, dcls(D), s) for D in SPECIAL_D + (50,) for o in MB.KINDS
            for k in (N.ORX_PAIR_BPR, N.ORX_PAIR_UCML) for s in (0, 1, 2)}
    want |= {(POINT_OP, _point_rule(D)[0], k, o, dcls(D), 0) for D in SPECIAL_D + (50,) for o in MB.KINDS
             for k in (N.ORX_POINT_GMF, N.ORX_POINT_WRMF)}
    assert seen == want, (sorted(want - seen), sorted(seen - want))
    assert {D for _, _, _, D, B, _, _ in MB.pair_specs() if B % 8} >= set(SPECIAL_D + (50,)), "batch tails"
    assert {s[5] for s in MB.pair_specs()} == {"mixed", "owned", "staged"}


@pytest.mark.parametrize("opt", MB.KINDS)
@pytest.mark.parametrize("kind,D", [("bpr", 128), ("ucml", 50), ("gmf", 64), ("wrmf", 256)])
def test_momentum_untouched_rows_over_five_steps(eng, kind, D, opt):
    """Five steps whose ids stay below row 40: rows 40.. keep value and slot bit for bit, while the slots of the rows
    the steps touch have moved."""
    rng = np.random.default_rng(S.spec_seed("mom_untouched", kind, D, opt))
    pair = kind in S.PAIR_KINDS
    U, I = 60, 70
    sc = 0.05 if kind == "bpr" else 0.3
    tabs = [S.f32(rng.uniform(-sc, sc, s)) for s in ((U, D), (I, D), (I, 1), (1, D))][:4 if kind == "gmf" else 3]
    slots = [S.f32(rng.uniform(-0.02, 0.02, t.shape)) for t in tabs]
    t = [dev(x) for x in tabs]
    s = [dev(x) for x in slots]
    tt = [N.table(a, b) for a, b in zip(t, s)]
    o = N.opt(opt, 0.05, beta1=0.9)
    for _ in range(5):
        out = torch.zeros(4, device="cuda")
        if pair:
            ids = [dev(rng.integers(0, 40, 128), torch.int32) for _ in range(3)]
            eng.pairwise_step(KINDS[kind], *tt, *ids, o, out)
        else:
            ids = [dev(rng.integers(0, 40, 128), torch.int32) for _ in range(2)]
            eng.pointwise_step(KINDS[kind], *tt[:3], tt[3] if kind == "gmf" else None, *ids,
                               dev((rng.random(128) < 0.4).astype(np.float32)), o, out)
    torch.cuda.synchronize()
    for j in range(3):
        got_v, got_s = t[j].cpu().numpy(), s[j].cpu().numpy()
        assert np.array_equal(got_v[40:], tabs[j][40:]) and np.array_equal(got_s[40:], slots[j][40:]), j
        assert (got_s[:40] != slots[j][:40]).any(), j


# ---- exact cases ------------------------------------------------------------------------------------------------------
def _dyadic(rng, shape, q, lim):
    return np.round(rng.uniform(-lim, lim, shape) / q) * q


@pytest.mark.parametrize("entry", ("sparse", "strided", "bag_sum", "bag_mean", "dense"))
@pytest.mark.parametrize("D", (128, 50))
def test_momentum_exact_dyadic(eng, entry, D):
    """Rows on the 2^-4 grid, slots on 2^-8, gradients on 2^-4 (at most four per row, bags of 1, 2 or 4), lr 2^-3,
    m 2^-1: every product, sum and difference is exact in float32, so each path equals the float64 update bit for bit,
    and NESTEROV's value minus MOMENTUM's is exactly m * a_new - lr * G - a_new."""
    rng = np.random.default_rng(S.spec_seed("mom_exact", entry, D))
    R, lr, m = 64, 0.125, 0.5
    var, a = _dyadic(rng, (R, D), 2.0 ** -4, 2.0), _dyadic(rng, (R, D), 2.0 ** -8, 0.5)
    res = {}
    for opt in MB.KINDS:
        tv, ta = dev(var), dev(a)
        o = N.opt(opt, lr, beta1=m)
        if entry == "dense":
            g = _dyadic(np.random.default_rng(7), (R, D), 2.0 ** -4, 2.0)
            eng.dense_apply(tv, ta, None, dev(g), o)
            idx, G = np.arange(R), g
        else:
            ids = np.repeat(np.arange(0, R - 8), 1 + np.arange(R - 8) % 4)      # 1..4 lookups per row, rows R-8.. untouched
            ids = np.random.default_rng(8).permutation(ids).astype(np.int32)
            vals = _dyadic(np.random.default_rng(9), (len(ids), D), 2.0 ** -4, 2.0)
            tab = N.table(tv, ta)
            if entry == "sparse":
                eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
                lk_ids, lk_vals = ids, vals
            elif entry == "strided":
                eng.sparse_apply_strided(tab, dev(np.stack([ids[::-1], ids], 1), torch.int32), 1,
                                         dev(np.stack([np.zeros_like(vals), vals], 1)), o)
                lk_ids, lk_vals = ids, vals
            else:
                sizes = np.random.default_rng(10).choice([1, 2, 4], 60)
                Lmax = 4
                sp = np.full((60, Lmax), -1, np.int32)
                pool = np.random.default_rng(11).integers(0, R - 8, sizes.sum())
                k = 0
                for b, n in enumerate(sizes):
                    sp[b, :n] = pool[k:k + n]
                    k += n
                dz = _dyadic(np.random.default_rng(12), (60, D), 2.0 ** -4, 2.0)
                mean = entry == "bag_mean"
                eng.bag_sparse_apply(tab, dev(sp, torch.int32), 0, Lmax, dev(dz), 1 if mean else 0, o)
                b_of, l_of = np.nonzero(sp >= 0)
                lk_ids = sp[b_of, l_of]
                lk_vals = dz[b_of] / sizes[b_of, None] if mean else dz[b_of]
            idx, G = O.dedup(lk_ids, lk_vals)
        torch.cuda.synchronize()
        want_v, want_a = var.copy(), a.copy()
        a1 = m * a[idx] - lr * G
        want_a[idx] = a1
        want_v[idx] += m * a1 - lr * G if opt == NEST else a1
        got_v, got_a = tv.cpu().numpy().astype(np.float64), ta.cpu().numpy().astype(np.float64)
        assert np.array_equal(got_a, want_a), (entry, opt)
        assert np.array_equal(got_v, want_v), (entry, opt)
        res[opt] = (got_v, a1, idx, G)
    v_mom, a1, idx, G = res[MOM]
    v_nest = res[NEST][0]
    assert np.array_equal((v_nest - v_mom)[idx], m * a1 - lr * G - a1)


@pytest.mark.parametrize("kind", S.PAIR_KINDS)
@pytest.mark.parametrize("opt", MB.KINDS)
def test_momentum_fused_exact_zero_rows(eng, kind, opt):
    """Arm (c): users 0 and 1 meet only clamped / inactive triplets at c_l2 = 0, so G = 0 exactly: value and slot equal
    the float32 rounding of each operation (a = m a, var += a, or var += m a) bit for bit."""
    c = MB.build(("c", kind, opt, 64, 203, "mixed", "step"))
    d = Dev(c)
    _pair_launch(eng, c, d, "step")
    got = d.got()
    ref = MB.f32_step(c)
    for j in (0, 1):
        assert np.array_equal(got["user"][j][:2], ref["user"][j][:2]), j
    assert not np.array_equal(got["user"][1][:2], c.slots["user"][0][:2])
    MB.MomBar(c).check(got, "exact zero rows")


# ---- un-fused applies -------------------------------------------------------------------------------------------------
def _bags(rng, B, Lmax, R):
    sp = np.full((B, Lmax), -1, np.int32)
    for b in range(B):
        n = rng.integers(0, Lmax + 1)
        sp[b, :n] = rng.integers(0, R - 7, n)
    return sp


@pytest.mark.parametrize("opt", MB.KINDS)
@pytest.mark.parametrize("D", (128, 256, 50))
@pytest.mark.parametrize("entry", ("sparse", "strided", "bag_sum", "bag_mean", "dense"))
@pytest.mark.parametrize("offset", (0, 1, 4), ids=("aligned", "table_off16", "slot_off16"))
def test_momentum_unfused_apply(eng, opt, D, entry, offset):
    """orx_sparse_apply / _strided / orx_bag_sparse_apply (sum and mean over ragged bags) on duplicated ids, rows R-7..
    untouched, and orx_dense_apply; offset 1 / 4: the table / the slot starts 4 bytes off a 16-byte boundary (the scalar
    paths)."""
    rng = np.random.default_rng(S.spec_seed("mom_apply", opt, D, entry, offset))
    R, n = 97, 300
    lr, m = float(np.float32(0.05)), float(np.float32(0.9))
    var = S.f32(rng.uniform(-0.3, 0.3, (R, D)))
    a = S.f32(rng.uniform(-0.02, 0.02, (R, D)))
    vt = torch.zeros(R * D + 4, device="cuda")
    at = torch.zeros(R * D + 4, device="cuda")
    tv = vt[(1 if offset == 1 else 0):][:R * D].view(R, D)
    ta = at[(1 if offset == 4 else 0):][:R * D].view(R, D)
    tv.copy_(dev(var))
    ta.copy_(dev(a))
    tab = N.OrxTable(tv.data_ptr(), ta.data_ptr(), None, R, D)
    o = N.opt(opt, lr, beta1=m)
    if entry == "dense":
        g = S.f32(rng.standard_normal((R, D)) * 0.1)
        eng.dense_apply(tv, ta, None, dev(g), o)
        lk_ids, lk_vals = np.arange(R), g
    elif entry in ("sparse", "strided"):
        ids = rng.integers(0, R - 7, n).astype(np.int32)
        vals = S.f32(rng.standard_normal((n, D)) * 0.1)
        if entry == "sparse":
            eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
        else:
            eng.sparse_apply_strided(tab, dev(np.stack([ids[::-1], ids], 1), torch.int32), 1,
                                     dev(np.stack([np.zeros_like(vals), vals], 1)), o)
        lk_ids, lk_vals = ids, vals
    else:
        B, Lmax = 120, 5
        sp = _bags(rng, B, Lmax, R)
        dz = S.f32(rng.standard_normal((B, D)) * 0.1)
        mean = entry == "bag_mean"
        eng.bag_sparse_apply(tab, dev(sp, torch.int32), 0, Lmax, dev(dz), 1 if mean else 0, o)
        b_of, l_of = np.nonzero(sp >= 0)
        lk_ids = sp[b_of, l_of]
        cnt = (sp >= 0).sum(1).astype(np.float32)
        lk_vals = (dz[b_of] / cnt[b_of, None]).astype(np.float32).astype(np.float64) if mean else dz[b_of]
    idx, G, E = S.dedup(lk_ids, lk_vals, np.zeros_like(lk_vals), np.abs(lk_vals))
    ref, tol = MB.update_bar(opt, lr, m, (var, a, None), idx, G, E)
    torch.cuda.synchronize()
    q = S.ratios(ref, tol, [tv.cpu().numpy(), ta.cpu().numpy(), None])
    assert max(x for x in q if x is not None) <= 1.0, (entry, D, offset, q)


def test_momentum_step_off16_takes_generic(eng):
    """A table or slot off a 16-byte boundary takes k_pair_generic / k_point_generic, and updates correctly."""
    for spec, op in (((("a", "bpr", MOM, 128, 203, "mixed", "step")), PAIR_OP),
                     ((("d", "gmf", NEST, 64, 237, "mixed", "step")), POINT_OP)):
        for which in (0, 1):
            c = MB.build(spec)
            d = Dev(c)
            for n in ("user", "item"):
                buf = torch.zeros(d.t[n][which].numel() + 4, device="cuda")
                d.t[n][which] = buf[1:1 + d.t[n][which].numel()].view_as(d.t[n][which]).copy_(d.t[n][which])
                d.tt[n] = N.OrxTable(d.t[n][0].data_ptr(), d.t[n][1].data_ptr(), None, *d.t[n][0].shape)
            eng.debug_dispatch_log()
            _pair_launch(eng, c, d, "step") if op == PAIR_OP else _point_launch(eng, c, d)
            rec = eng.debug_dispatch_log()[0]
            assert rec.variant == L.ORX_VARIANT_STEP_GENERIC and rec.tb == c.opt, (spec, which, rec)
            MB.MomBar(c).check(d.got(), f"off16 {which}")


def test_momentum_far_table(eng):
    """orx_sparse_apply under NESTEROV on a [rows, 128] table past 2^32 elements (tests/far_tables.py): far rows update
    against the bar, their 32-bit alias rows and the untouched rows around them stay bit-identical."""
    import far_tables as F
    D = 128
    rows = F.far_rows(D)
    need = 2 * rows * D * 4 + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB free for a far table and its slot")
    rng = np.random.default_rng(17)
    far = np.unique(rng.integers(F.MID_END // D + 1, rows, 24))
    low = np.arange(5, 12)
    alias = np.unique(np.concatenate([F.alias_rows(r, D) for r in far]))
    touched = np.concatenate([far, low])
    watch = np.unique(np.concatenate([touched, alias, [rows - 1]]))
    var = S.f32(rng.uniform(-0.3, 0.3, (len(watch), D)))
    a = S.f32(rng.uniform(-0.02, 0.02, (len(watch), D)))
    tv = torch.empty(rows, D, device="cuda")
    ta = torch.empty(rows, D, device="cuda")
    try:
        wt = dev(watch, torch.int64)
        tv[wt] = dev(var)
        ta[wt] = dev(a)
        ids = rng.permutation(np.repeat(touched, 2)[: 2 * len(touched) - 3]).astype(np.int32)
        vals = S.f32(rng.standard_normal((len(ids), D)) * 0.1)
        lr, m = float(np.float32(0.05)), float(np.float32(0.9))
        eng.sparse_apply(N.table(tv, ta), dev(ids, torch.int32), dev(vals), N.opt(NEST, lr, beta1=m))
        got_v, got_a = tv[wt].cpu().numpy(), ta[wt].cpu().numpy()
    finally:
        del tv, ta
        torch.cuda.empty_cache()
    pos = {int(r): k for k, r in enumerate(watch)}
    cidx = np.array([pos[int(r)] for r in ids])
    idx, G, E = S.dedup(cidx, vals, np.zeros_like(vals), np.abs(vals))
    ref, tol = MB.update_bar(NEST, lr, m, (var, a, None), idx, G, E)
    q = S.ratios(ref, tol, [got_v, got_a, None])
    assert max(q[:2]) <= 1.0, q
    rest = np.array([pos[int(r)] for r in watch if r not in set(touched.tolist())])
    assert len(rest) and np.array_equal(got_v[rest], var[rest]) and np.array_equal(got_a[rest], a[rest])


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_momentum_refusals(eng):
    """A missing slot is ORX_ERR_INVALID before any device work, under both kinds, for every entry point that takes a
    table; kinds 4 and 7 stay unknown to every entry point."""
    lib = L.lib()
    var = torch.zeros(10, 8, device="cuda")
    s0 = torch.zeros(10, 8, device="cuda")
    b = torch.zeros(10, 1, device="cuda")
    bs = torch.zeros(10, 1, device="cuda")
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    vals = torch.zeros(4, 8, device="cuda")
    out4 = torch.zeros(4, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    before = var.clone()

    def calls(tab, btab, o):
        yield lib.orx_sparse_apply(eng.h, C.byref(tab), p(ids), p(vals), 4, C.byref(o), None)
        yield lib.orx_bag_sparse_apply(eng.h, C.byref(tab), p(ids), 1, 0, 1, 4, p(vals), 8, 0, C.byref(o), None)
        yield lib.orx_pairwise_step(eng.h, 0, C.byref(tab), C.byref(tab), C.byref(btab), p(ids), p(ids), p(ids), 4,
                                    C.c_float(0.5), C.c_float(1.0), C.c_float(1.0), C.byref(o), p(out4), None)
        yield lib.orx_pointwise_step(eng.h, 1, C.byref(tab), C.byref(tab), C.byref(btab), None, p(ids), p(ids),
                                     p(out4), 4, C.c_float(1.0), C.c_float(1.0), 0, C.c_float(1.0), C.c_float(1.0),
                                     C.byref(o), p(out4), None)
        yield lib.orx_dense_apply(eng.h, p(var), p(s0) if tab.s0 else None, None, p(vals), 32, C.byref(o), None)

    bare, bbare = N.OrxTable(var.data_ptr(), None, None, 10, 8), N.OrxTable(b.data_ptr(), None, None, 10, 1)
    for k in MB.KINDS:
        assert all(rc == ORX_ERR_INVALID for rc in calls(bare, bbare, N.opt(k, 0.05))), k
    full, bfull = N.table(var, s0), N.table(b, bs)
    for k in (4, 7):
        assert all(rc == ORX_ERR_INVALID for rc in calls(full, bfull, N.opt(k, 0.05))), k
        rc = lib.orx_pairwise_prefetch(eng.h, C.byref(full), C.byref(full), p(ids), p(ids), p(ids), 4, k, 1, None)
        assert rc == ORX_ERR_INVALID, k
    torch.cuda.synchronize()
    assert torch.equal(var, before) and not s0.any()


# ---- the home-routed sharded step (LoopbackGroup: R virtual ranks on one GPU) -----------------------------------------
def _ref_pair_step(kind, tabs, st, ids, lr, m, nest, margin, c_loss, c_l2):
    """The float64 step: the oracle's loss and gradients, then momentum on each table's deduplicated rows."""
    user, item, bias = tabs
    if kind == 0:
        out = O.bpr_forward(user, item, bias, *ids)
        gr = O.bpr_grads(user, item, bias, *ids, c_loss, c_l2)
    else:
        out = O.ucml_forward(user, item, bias, *ids, margin)
        gr = O.ucml_grads(user, item, bias, *ids, margin, c_loss, c_l2)
    for name, var in zip(("user", "item", "bias"), tabs):
        idx, val = gr[name]
        MB.momentum_sparse(var, st[name], idx, val.reshape(len(idx), -1), lr, m, nest)
    return out


LOOPBACK = [(1, 0, MOM, 64, "plain"), (2, 1, NEST, 64, "announce"), (3, 0, NEST, 192, "bad"),
            (4, 1, MOM, 256, "dups"), (8, 0, MOM, 8, "announce"), (2, 0, NEST, 512, "plain"),
            (4, 0, NEST, 128, "dups"), (3, 1, MOM, 8, "bad")]


@pytest.mark.parametrize("world,kind,opt,D,mode", LOOPBACK, ids=[_sid(x) for x in LOOPBACK])
def test_momentum_loopback(eng, world, kind, opt, D, mode):
    """orx_shard_step with R virtual ranks: three steps against the float64 step on the global batch and against the
    single-GPU orx_pairwise_step run from the same tables (announced batches, bad ids, heavy duplicates)."""
    from openrec_b200.sharded import LoopbackGroup
    rng = np.random.default_rng(S.spec_seed("mom_loop", world, kind, opt, D, mode))
    U, I, B = (37, 41, 96) if mode == "dups" else (501, 703, 96)
    lr, m, margin = float(np.float32(0.05)), float(np.float32(0.9)), 0.5
    sc = 0.05 if kind == 0 else 0.4
    tabs = [S.f32(rng.uniform(-sc, sc, s)) for s in ((U, D), (I, D), (I, 1))]
    g = LoopbackGroup(world, U, I, D, B, kind=kind, opt_kind=opt, lr=lr, beta1=m, margin=margin, init=False)
    single = [dev(t) for t in tabs]
    single_s = [torch.zeros_like(t) for t in single]
    stt = [N.table(a, b) for a, b in zip(single, single_s)]
    try:
        g.load_global(*tabs)
        ref = [t.copy() for t in tabs]
        st = {n: np.zeros_like(t) for n, t in zip(("user", "item", "bias"), tabs)}
        steps = 3
        all_ids = [[rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)] for _ in range(steps)]
        if mode == "bad":
            for ids in all_ids:
                ids[0][3], ids[1][B // 2], ids[2][-1] = -1, I, -7
        batches = [[tuple(dev(a[r * B:(r + 1) * B], torch.int32) for a in ids) for r in range(world)] for ids in all_ids]
        for k, ids in enumerate(all_ids):
            nxt = batches[k + 1] if mode == "announce" and k + 1 < steps else None
            outs = [o.cpu().numpy() for o in g.step(batches[k], next_batches=nxt)]
            g.check()
            ok = (ids[0] >= 0) & (ids[0] < U) & (ids[1] >= 0) & (ids[1] < I) & (ids[2] >= 0) & (ids[2] < I)
            frac = ok.sum() / (B * world) if kind == 0 else 1.0
            loss, l2 = _ref_pair_step(kind, ref, st, [x[ok] for x in ids], lr, m, opt == NEST, margin, frac, 1.0)
            for o in outs:
                np.testing.assert_allclose(o, [loss * frac, l2], rtol=3e-5, atol=1e-6)
                assert np.array_equal(o, outs[0])
            out4 = torch.zeros(4, device="cuda")
            eng.pairwise_step(kind, *stt, *(dev(x, torch.int32) for x in ids), N.opt(opt, lr, beta1=m), out4,
                              margin, 1.0, 1.0)
        got = [t.cpu().numpy() for t in g.gather_global()]
        tol = 1e-5 if kind == 0 else 2e-4
        for a, r, s in zip(got, ref, single):
            np.testing.assert_allclose(a, r, atol=tol)
            np.testing.assert_allclose(a, s.cpu().numpy(), atol=tol)
    finally:
        g.close()


# ---- whole models ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


@pytest.mark.parametrize("nesterov", (False, True))
@pytest.mark.parametrize("kind", ("bpr", "ucml"))
def test_momentum_pairwise_models(tf, kind, nesterov):
    """BPR / UCML (with censor_vec after each step) through tape + SGD(momentum=0.9[, nesterov]): three steps against
    the oracle's gradients and the float64 momentum update."""
    from openrec.tf2.recommenders import BPR, UCML
    rng = np.random.default_rng(1)
    U, I, D, B = 60, 90, 32, 128
    model = BPR(D, D, U, I) if kind == "bpr" else UCML(D, D, U, I)
    opt = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nesterov)
    ref = [v.numpy().astype(np.float64) for v in model.trainable_variables]
    st = {n: np.zeros_like(t) for n, t in zip(("user", "item", "bias"), ref)}
    m = float(np.float32(0.9))
    for _ in range(3):
        ids = tuple(rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
        with tf.GradientTape() as tape:
            loss, l2 = model(*ids)
        opt.apply_gradients(zip(tape.gradient((loss, l2), model.trainable_variables), model.trainable_variables))
        want = _ref_pair_step(0 if kind == "bpr" else 1, ref, st, ids, float(np.float32(0.05)), m, nesterov, 0.5,
                              1.0, 1.0)
        np.testing.assert_allclose([float(loss.numpy()), float(l2.numpy())], want, rtol=1e-5, atol=1e-6)
        if kind == "ucml":
            model.censor_vec(*ids)
            O.ucml_censor_vec(ref[0], ref[1], *ids)
        for v, r, n in zip(model.trainable_variables, ref, ("user", "item", "bias")):
            np.testing.assert_allclose(v.numpy(), r, atol=2e-6, rtol=1e-5)
            np.testing.assert_allclose(opt.slots(v)[0].cpu().numpy(), st[n], atol=1e-7, rtol=1e-5)


def _grads_by_sgd_twin(tf, models, inputs, opt):
    """Step models[0] with SGD at lr 1 and models[1] with opt from the same weights: -> (old weights, the gradients
    models[0]'s step applied)."""
    for a, b in zip(models[0].trainable_variables, models[1].trainable_variables):
        b.t.copy_(a.t)
    old = [v.numpy().astype(np.float64) for v in models[0].trainable_variables]
    for m, o in zip(models, (tf.keras.optimizers.SGD(learning_rate=1.0), opt)):
        with tf.GradientTape() as tape:
            out = m(*inputs)
        o.apply_gradients(zip(tape.gradient(out, m.trainable_variables), m.trainable_variables))
    return old, [o - v.numpy().astype(np.float64) for o, v in zip(old, models[0].trainable_variables)]


def _check_momentum_apply(opt, old, grads, variables, m, nesterov, lr=0.05):
    """A first step from zero slots: a = -lr G, var += a (or m a - lr G), for every element (untouched rows: G = 0)."""
    for o, G, v in zip(old, grads, variables):
        a = -lr * G
        want = o + (m * a - lr * G if nesterov else a)
        np.testing.assert_allclose(opt.slots(v)[0].cpu().numpy(), a, rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(v.numpy(), want, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("nesterov", (False, True))
@pytest.mark.parametrize("kind", ("gmf", "wrmf"))
def test_momentum_pointwise_models(tf, kind, nesterov):
    """GMF (its w a dense variable) / WRMF through tape + SGD(momentum=0.9[, nesterov]) against the update of the
    gradients an SGD twin applies."""
    from openrec.tf2.recommenders import GMF, WRMF
    rng = np.random.default_rng(2)
    U, I, D, B = 50, 80, 32, 128
    models = [GMF(D, D, U, I), GMF(D, D, U, I)] if kind == "gmf" else [WRMF(D, D, U, I), WRMF(D, D, U, I)]
    opt = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nesterov)
    inputs = (rng.integers(0, U, B).astype(np.int32), rng.integers(0, I, B).astype(np.int32),
              (rng.random(B) < 0.4).astype(np.float32))
    old, grads = _grads_by_sgd_twin(tf, models, inputs, opt)
    _check_momentum_apply(opt, old, grads, models[1].trainable_variables, float(np.float32(0.9)), nesterov)


@pytest.mark.parametrize("nesterov", (False, True))
@pytest.mark.parametrize("bags", (False, True))
def test_momentum_dlrm_model(tf, bags, nesterov):
    """DLRM (one-hot and bag_sizes) through tape + SGD(momentum=0.9[, nesterov]): embedding tables and Dense layers
    against the update of the gradients an SGD twin applies."""
    from openrec.tf2.recommenders import DLRM
    rng = np.random.default_rng(3)
    vocab, D, B = [30, 1, 200, 2], 16, 128
    sizes = [2, 1, 3, 1] if bags else None
    kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[16, D], ln_top=[32, 1], interaction_mode="dlrm")
    if bags:
        kw.update(bag_sizes=sizes, pooling="sum")
    models = [DLRM(**kw), DLRM(**kw)]
    for mo in models:
        mo._graph(13)
    cols = sizes or [1] * len(vocab)
    inputs = (rng.random((B, 13)).astype(np.float32),
              np.concatenate([rng.integers(0, v, (B, c)) for v, c in zip(vocab, cols)], 1).astype(np.int32),
              (rng.random(B) < 0.3).astype(np.float32))
    opt = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nesterov)
    old, grads = _grads_by_sgd_twin(tf, models, inputs, opt)
    _check_momentum_apply(opt, old, grads, models[1].trainable_variables, float(np.float32(0.9)), nesterov)


# ---- checkpoints ------------------------------------------------------------------------------------------------------
def test_momentum_checkpoint_continue(tf, tmp_path):
    """BPR under SGD(momentum=0.9, nesterov=True): two steps, save, load into a fresh model and optimizer, two more
    steps, equal to four uninterrupted steps; HomeRoutedPairwise.save_shard / load_shard likewise.  (Not bit for bit:
    a staged row's gradient is a sum of float atomics, in no fixed order.)"""
    from openrec.tf2.recommenders import BPR
    from openrec_b200.tf2 import checkpoint
    rng = np.random.default_rng(4)
    U, I, D, B = 60, 90, 32, 128
    batches = [tuple(rng.integers(0, n, B).astype(np.int32) for n in (U, I, I)) for _ in range(4)]

    def run(model, opt, bs):
        for ids in bs:
            with tf.GradientTape() as tape:
                out = model(*ids)
            opt.apply_gradients(zip(tape.gradient(out, model.trainable_variables), model.trainable_variables))

    mk = lambda: tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=True)
    m1, o1 = BPR(D, D, U, I), mk()
    m2, o2 = BPR(D, D, U, I), mk()
    for a, b in zip(m1.trainable_variables, m2.trainable_variables):
        b.t.copy_(a.t)
    run(m1, o1, batches)
    run(m2, o2, batches[:2])
    checkpoint.save(str(tmp_path / "ck.npz"), m2, o2)
    m3, o3 = BPR(D, D, U, I), mk()
    checkpoint.load(str(tmp_path / "ck.npz"), m3, o3)
    run(m3, o3, batches[2:])
    assert o3.iterations == 4
    for a, b in zip(m1.trainable_variables, m3.trainable_variables):
        np.testing.assert_allclose(b.numpy(), a.numpy(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(o3.slots(b)[0].cpu().numpy(), o1.slots(a)[0].cpu().numpy(), rtol=1e-5, atol=1e-8)
        assert not np.array_equal(o1.slots(a)[0].cpu().numpy(), 0)

    from openrec_b200.sharded import LoopbackGroup
    tabs = [S.f32(rng.uniform(-0.05, 0.05, s)) for s in ((U, D), (I, D), (I, 1))]
    ids = [[dev(rng.integers(0, n, B), torch.int32) for n in (U, I, I)] for _ in range(4)]
    kw = dict(kind=0, opt_kind=MOM, lr=0.05, beta1=0.9, init=False)
    res = []
    for split in (False, True):
        g = LoopbackGroup(1, U, I, D, B, **kw)
        try:
            g.load_global(*tabs)
            for k in range(4):
                if split and k == 2:
                    g.ranks[0].save_shard(str(tmp_path / "shard.npz"))
                    g.close()
                    g = LoopbackGroup(1, U, I, D, B, **kw)
                    g.ranks[0].load_shard(str(tmp_path / "shard.npz"))
                g.step([tuple(ids[k])])
            g.check()
            r = g.ranks[0]
            res.append([t.cpu().numpy() for t in (r.user, r.item, r.bias, *r.user_slots[:1], *r.item_slots[:1])])
        finally:
            g.close()
    for a, b in zip(*res):
        np.testing.assert_allclose(b, a, rtol=1e-5, atol=1e-8)


# ---- sharded models in an NCCL group ----------------------------------------------------------------------------------
_SHARD = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
import tensorflow as tf
from openrec.tf2.recommenders import (BPR, DLRM, GMF, UCML, WRMF, ShardedBPR, ShardedDLRM, ShardedGMF, ShardedUCML,
                                      ShardedWRMF)

def shard_of(full, r, R):
    return full[r::R]

def run(models, data, nest):
    losses, opts = [], []
    for model in models:
        optimizer = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nest)
        losses.append([])
        for b in data:
            with tf.GradientTape() as tape:
                out = model(*b)
            optimizer.apply_gradients(zip(tape.gradient(out, model.trainable_variables), model.trainable_variables))
            out = out if isinstance(out, tuple) else (out,)
            losses[-1].append([float(x.numpy()) for x in out])
        opts.append(optimizer)
    np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5, atol=1e-6)
    return opts

rng = np.random.default_rng(0)
which, nest = {which!r}, {nest!r}
# one home-routed model per process: ShardedBPR / ShardedUCML models stepped one after another in a process do not match
# their single-GPU models past the first (under every optimizer), which is not what this checks
for _ in (0,):
    # factor models: the rank's shard rows r, r + R, ... of the single-GPU tables (every rank holds the whole model)
    U, I, D, B = 300, 2000, 64, 256
    for S_cls, F_cls, pair in [x for x in ((ShardedBPR, BPR, True), (ShardedUCML, UCML, True),
                                           (ShardedGMF, GMF, False), (ShardedWRMF, WRMF, False))
                               if x[1].__name__.lower() == which]:
        models = [S_cls(D, D, U, I, seed=3), F_cls(D, D, U, I)]
        for a_, b_ in zip(models[1].trainable_variables, models[0].trainable_variables):
            if a_.t.shape == b_.t.shape and world == 1:
                a_.t.copy_(b_.t)
        if world > 1:          # the single-GPU model starts from the shards' union
            for a_, b_ in zip(models[1].trainable_variables, models[0].trainable_variables):
                if a_.t.dim() == 2 and a_.t.shape[0] in (U, I):
                    full = torch.zeros_like(a_.t)
                    parts = [torch.zeros_like(b_.t) for _ in range(world)]
                    dist.all_gather(parts, b_.t.contiguous())
                    for r in range(world):
                        n = len(range(r, a_.t.shape[0], world))
                        full[r::world] = parts[r][:n]
                    a_.t.copy_(full)
                else:
                    a_.t.copy_(b_.t)
        g = np.random.default_rng(1)     # the same global batch on every rank; each rank passes its slice
        data = []
        for _ in range(3):
            if pair:
                ids = [g.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
                data.append(tuple(x[rank * B:(rank + 1) * B] for x in ids))
            else:
                ids = [g.integers(0, U, B * world).astype(np.int32), g.integers(0, I, B * world).astype(np.int32),
                       (g.random(B * world) < 0.3).astype(np.float32)]
                data.append(tuple(x[rank * B:(rank + 1) * B] for x in ids))
        if world == 1:
            opts = run(models, data, nest)
            for a_, b_ in zip(models[0].trainable_variables, models[1].trainable_variables):
                torch.testing.assert_close(a_.t[:b_.t.shape[0]], b_.t, atol=1e-5, rtol=1e-5)
                torch.testing.assert_close(opts[0].slots(a_)[0][:b_.t.shape[0]], opts[1].slots(b_)[0],
                                           atol=1e-5, rtol=1e-5)
        else:                    # every rank: its shard after the global steps against the full model's rows
            sopt = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nest)
            for b in data:
                with tf.GradientTape() as tape:
                    out = models[0](*b)
                sopt.apply_gradients(zip(tape.gradient(out, models[0].trainable_variables),
                                         models[0].trainable_variables))
            gdata = []
            for b in data:
                parts = [[torch.zeros_like(torch.as_tensor(x)).cuda() for _ in range(world)] for x in b]
                for p, x in zip(parts, b):
                    dist.all_gather(p, torch.as_tensor(x).cuda())
                gdata.append(tuple(torch.cat(p).cpu().numpy() for p in parts))
            fopt = tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nest)
            for b in gdata:
                with tf.GradientTape() as tape:
                    out = models[1](*b)
                fopt.apply_gradients(zip(tape.gradient(out, models[1].trainable_variables),
                                         models[1].trainable_variables))
            for a_, b_ in zip(models[0].trainable_variables, models[1].trainable_variables):
                if b_.t.dim() == 2 and b_.t.shape[0] in (U, I):
                    n = len(range(rank, b_.t.shape[0], world))
                    torch.testing.assert_close(a_.t[:n], b_.t[rank::world], atol=2e-5, rtol=1e-4)
                    torch.testing.assert_close(sopt.slots(a_)[0][:n], fopt.slots(b_)[0][rank::world],
                                               atol=2e-5, rtol=1e-4)
    if world == 1 and which == "dlrm":      # ShardedDLRM against DLRM, one-hot and multi-hot
        vocab, D = [3, 1, 500, 2, 90], 16
        for bags in (None, [2, 1, 3, 1, 2]):
            kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[32, D], ln_top=[64, 1], interaction_mode="dlrm")
            if bags:
                kw.update(bag_sizes=bags, pooling="mean")
            models = [ShardedDLRM(**kw), DLRM(**kw)]
            models[0]._build(13); models[1]._graph(13)
            for lf, k in zip(models[1]._latent_factors, np.cumsum([0] + vocab[:-1])):
                lf.embeddings.t.copy_(models[0].embedding_shard.t[k:k + lf.embeddings.t.shape[0]])
            for a, b in zip(models[0].trainable_variables[1:], models[1].trainable_variables[len(vocab):]):
                b.t.copy_(a.t)
            cols = bags or [1] * len(vocab)
            data = [(rng.random((64, 13)).astype(np.float32),
                     np.concatenate([rng.integers(0, v, (64, c)) for v, c in zip(vocab, cols)], 1).astype(np.int32),
                     (rng.random(64) < 0.3).astype(np.float32)) for _ in range(3)]
            opts = run(models, data, nest)
            table = torch.cat([lf.embeddings.t for lf in models[1]._latent_factors])
            torch.testing.assert_close(models[0].embedding_shard.t[:table.shape[0]], table, atol=1e-5, rtol=1e-5)
            a = torch.cat([opts[1].slots(lf.embeddings)[0] for lf in models[1]._latent_factors])
            torch.testing.assert_close(opts[0].slots(models[0].embedding_shard)[0][:a.shape[0]], a, atol=1e-5,
                                       rtol=1e-5)
dist.destroy_process_group()
print("sharded ok")
"""


@pytest.mark.parametrize("nest", (False, True))
@pytest.mark.parametrize("which", ("bpr", "ucml", "gmf", "wrmf", "dlrm"))
def test_momentum_sharded_models_one_rank(which, nest):
    """ShardedBPR / UCML / GMF / WRMF and ShardedDLRM (one-hot and bag_sizes) in a one-rank NCCL group under
    SGD(momentum=0.9[, nesterov]) match their single-GPU models, slots included."""
    [(rc, out)] = run_ranks(1, _SHARD.format(root=ROOT, which=which, nest=nest), f"gpu_momentum sharded {which} {nest}",
                            timeout=600)
    assert rc == 0 and "sharded ok" in out, out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("nest", (False, True))
@pytest.mark.parametrize("which", ("bpr", "ucml", "gmf", "wrmf"))
def test_momentum_sharded_models_two_ranks(which, nest):
    """ShardedBPR / UCML / GMF / WRMF over two real ranks under SGD(momentum=0.9[, nesterov]): each rank's shard and
    slot rows after three global steps equal those rows of the single-GPU model stepped on the global batches."""
    outs = run_ranks(2, _SHARD.format(root=ROOT, which=which, nest=nest), f"gpu_momentum sharded2 {which} {nest}",
                     timeout=600)
    for rc, out in outs:
        assert rc == 0 and "sharded ok" in out, out
