"""The sparse training steps judged by their per-element updates (tests/step_bar.py), not by their values.

Every table and optimizer slot's change new - old is compared with the float64 oracle's change, under the bar whose
terms step_bar.py writes down: a few float32 ulps, the MUFU divide, and the float32 error bound of each row's summed
gradient carried through the optimizer.  At that bar a 10 % error in BPR's or GMF's c_loss / B loss gradient, a
neighbour's g, a score without its bias or a lost duplicate fails by orders of magnitude; at the older atol / rtol 1e-5
on the values it passes.  Four arms (step_bar.arm_consts): (a) loss only, Keras slots; (b) c_loss = B, c_l2 = 1;
(c) tie / saturation tables on a dyadic grid, with rows whose every contribution is an exact zero (left bit-identical
by SGD / Adagrad, moved by lazy Adam's m decay); (d) beta1 0.5, beta2 0.75, eps 1e-2, margin 1.25 at step 3.
tests/test_step_bar_cpu.py shows on CPU that the float32 oracle passes every case here and the mutants fail."""
import numpy as np
import pytest
import torch

import step_bar as S
from oracle import openrec_oracle as O
from openrec_b200 import native as N
from test_gpu_kernels import PAIR_OP, POINT_OP, SPECIAL_D, _check_step_dispatch, _pair_rule, _point_rule, dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def _opt(c):
    return N.opt(c.opt, c.lr, eps=c.P["eps"], beta1=c.P["beta1"], beta2=c.P["beta2"], step=c.step)


class Dev:
    """A case's tables and slots on the device."""

    def __init__(self, c):
        self.c = c
        self.t = {n: [None if x is None else dev(x) for x in (c.tabs[n], *c.slots[n])] for n in c.names}
        self.tt = {n: N.table(*v) for n, v in self.t.items()}

    def got(self):
        torch.cuda.synchronize()
        return {n: tuple(None if x is None else x.cpu().numpy().astype(np.float64) for x in v)
                for n, v in self.t.items()}


def _record(eng, op, c, index_set=0):
    return _check_step_dispatch(eng, op, _kind(c), c.opt, c.B, c.D, index_set)


def _kind(c):
    return {"bpr": N.ORX_PAIR_BPR, "ucml": N.ORX_PAIR_UCML, "gmf": N.ORX_POINT_GMF, "wrmf": N.ORX_POINT_WRMF}[c.kind]


def _judge(c, d, what):
    S.Bar(c).check(d.got(), what)


def _pair_launch(eng, c, d, entry, dids=None):
    P = dict(margin=c.P["margin"], c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    out = torch.zeros(4, device="cuda")
    if entry == "host":
        ids = [torch.from_numpy(x).pin_memory() for x in c.ids]
        out = torch.zeros(4).pin_memory()
        eng.pairwise_step_host(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c), out, **P)
        torch.cuda.synchronize()     # the pinned ids must outlive the upload
    else:
        eng.pairwise_step(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"],
                          *(dids or [dev(x, torch.int32) for x in c.ids]), _opt(c), out, **P)
    return out


@pytest.mark.parametrize("spec", S.pair_specs(), ids=lambda s: "-".join(map(str, s)))
def test_pairwise_step_updates(eng, spec):
    entry = spec[5]
    eng.debug_dispatch_log()
    if entry == "prefetch":
        sets = []
        for k in (0, 1):
            c = S.build(spec, k)
            d = Dev(c)
            dids = [dev(x, torch.int32) for x in c.ids]
            torch.cuda.synchronize()
            eng.pairwise_prefetch(d.tt["user"], d.tt["item"], *dids, c.opt, ids_ready=True)
            _pair_launch(eng, c, d, "step", dids)
            sets.append(_record(eng, PAIR_OP, c, "prefetch"))
            _judge(c, d, f"prefetched step {k}")
        assert sorted(sets) == [1, 2], sets
        return
    c = S.build(spec)
    d = Dev(c)
    _pair_launch(eng, c, d, entry)
    _record(eng, PAIR_OP, c, "prefetch" if entry == "host" else 0)
    _judge(c, d, entry)


@pytest.mark.parametrize("spec", S.point_specs(), ids=lambda s: "-".join(map(str, s)))
def test_pointwise_step_updates(eng, spec):
    c = S.build(spec)
    d = Dev(c)
    eng.debug_dispatch_log()
    out = torch.zeros(4, device="cuda")
    wrmf = c.kind == "wrmf"
    eng.pointwise_step(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], None if wrmf else d.tt["w"],
                       *(dev(x, torch.int32) for x in c.ids), dev(c.label), _opt(c), out,
                       c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False),
                       c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    _record(eng, POINT_OP, c)
    _judge(c, d, "pointwise step")


@pytest.mark.parametrize("kind", S.PAIR_KINDS)
@pytest.mark.parametrize("opt", range(4))
def test_zero_contribution_rows(eng, kind, opt):
    """Arm (c): users 0 and 1 (and their tie triplets' items) meet only clamped / inactive triplets at c_l2 = 0, so every
    contribution to them is an exact zero.  SGD / Adagrad leave them bit-identical; lazy Adam moves them by m's decay,
    as the oracle does (the bar holds the values); dense Adam moves every row."""
    c = S.pair_case("c", kind, opt, 64, 203, S.spec_seed("zero", kind, opt))
    d = Dev(c)
    eng.debug_dispatch_log()
    _pair_launch(eng, c, d, "step")
    _record(eng, PAIR_OP, c)
    got = d.got()
    S.Bar(c).check(got, "zero-contribution rows")
    old, new = c.tabs["user"][:2], got["user"][0][:2]
    if opt in (O.OPT_SGD, O.OPT_ADAGRAD):
        assert np.array_equal(old, new)
    else:
        assert (old != new).mean() > 0.5, "Adam leaves a row with m != 0 unmoved"


# ---- the un-fused forms: per-lookup gradient rows ---------------------------------------------------------------------
def _lookup_check(got, ref, tol, what):
    got = np.asarray(got, np.float64).reshape(ref.shape)
    q = np.abs(got - ref) / np.maximum(tol, 1e-45)
    assert q.max() <= 1.0, f"{what}: err/tol {q.max():.3g} at {np.unravel_index(q.argmax(), q.shape)}"


@pytest.mark.parametrize("arm", "ac")
@pytest.mark.parametrize("kind", S.PAIR_KINDS)
@pytest.mark.parametrize("D", (12, 128))
def test_pairwise_grad_lookups(eng, arm, kind, D):
    """orx_pairwise_grad: every lookup's gradient row (with its L2 term) under the per-lookup bar."""
    c = S.pair_case(arm, kind, O.OPT_SGD, D, 203, S.spec_seed("grad", arm, kind, D))
    d = Dev(c)
    B = c.B
    out = {k: torch.full(s, float("nan"), device="cuda") for k, s in
           (("d_user", (B, D)), ("d_pos", (B, D)), ("d_neg", (B, D)), ("d_bp", (B,)), ("d_bn", (B,)))}
    eng.pairwise_grad(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], *(dev(x, torch.int32) for x in c.ids),
                      c.P["margin"], c.P["c_loss"], c.P["c_l2"], **out)
    torch.cuda.synchronize()
    bar = S.lookup_bar(c)
    g = {k: v.cpu().numpy() for k, v in out.items()}
    _lookup_check(g["d_user"], *bar["user"], "d_user")
    _lookup_check(np.concatenate([g["d_pos"], g["d_neg"]]), *bar["item"], "d_pos / d_neg")
    _lookup_check(np.concatenate([g["d_bp"], g["d_bn"]]), *bar["bias"], "d_bp / d_bn")


@pytest.mark.parametrize("arm", "ac")
@pytest.mark.parametrize("kind", ("gmf", "wrmf", "wrmf_sig"))
@pytest.mark.parametrize("D", (10, 128))
def test_pointwise_grad_lookups(eng, arm, kind, D):
    """orx_pointwise_grad: every lookup's gradient row, and GMF's summed d_w."""
    c = S.point_case(arm, kind[:4], O.OPT_SGD, D, 203, S.spec_seed("pgrad", arm, kind, D), sig=kind == "wrmf_sig")
    d = Dev(c)
    B = c.B
    out = {k: torch.full(s, float("nan"), device="cuda") for k, s in
           (("d_user", (B, D)), ("d_item", (B, D)), ("d_bias", (B,)))}
    if c.kind == "gmf":
        out["d_w"] = torch.full((D,), float("nan"), device="cuda")
    eng.pointwise_grad(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], d.tt.get("w"),
                       *(dev(x, torch.int32) for x in c.ids), dev(c.label), c.P.get("a", 1.0), c.P.get("b", 1.0),
                       c.P.get("sig", False), c.P["c_loss"], c.P["c_l2"], **out)
    torch.cuda.synchronize()
    bar = S.lookup_bar(c)
    g = {k: v.cpu().numpy() for k, v in out.items()}
    for k, name in (("d_user", "user"), ("d_item", "item"), ("d_bias", "bias")):
        _lookup_check(g[k], *bar[name], k)
    if c.kind == "gmf":
        _, rows = S.lookups(c, c.state())
        idx, G, E = S.dedup(*rows["w"])
        _lookup_check(g["d_w"], G[0], E[0] + 2 * S.ulp32(G[0]), "d_w")


def _fetched(rng, c, lookups):
    """Fetched rows of the row-form gradients: lookup k's row (width D + 4: embedding, then the item bias in column D,
    zero padding) at a random position slot[k] of a table with as many rows as lookups."""
    D = c.D
    slot = rng.permutation(len(lookups)).astype(np.int32)
    rows = np.zeros((len(lookups), D + 4))
    for k, (name, i) in enumerate(lookups):
        rows[slot[k], :D] = c.tabs[name][i]
        if name == "item":
            rows[slot[k], D] = c.tabs["bias"][i, 0]
    return rows, slot


@pytest.mark.parametrize("arm", "ac")
@pytest.mark.parametrize("kind", S.PAIR_KINDS)
@pytest.mark.parametrize("D", (12, 64, 128))
def test_pairwise_grad_rows_lookups(eng, arm, kind, D):
    """orx_pairwise_grad_rows (the row-form gradients of the NCCL sharded step) on an arm (a) / (c) case: every lookup's
    fetched row gets its gradient row (embedding, item bias in column D) under the per-lookup bar; padding is zero."""
    c = S.pair_case(arm, kind, O.OPT_SGD, D, 203, S.spec_seed("grad_rows", arm, kind, D))
    B = c.B
    uid, pid, nid = c.ids
    rows, slot = _fetched(np.random.default_rng(S.spec_seed("slots", arm, kind, D)), c,
                          [("user", i) for i in uid] + [("item", i) for i in pid] + [("item", i) for i in nid])
    us, ps, ns = slot[:B], slot[B:2 * B], slot[2 * B:]
    d_rows = torch.full((3 * B, D + 4), 7.0, device="cuda")
    out4 = torch.zeros(4, device="cuda")
    eng.pairwise_grad_rows(_kind(c), dev(rows), D, *(dev(x, torch.int32) for x in (us, ps, ns)), 1.0 / B, d_rows, out4,
                           c.P["margin"], c.P["c_loss"], c.P["c_l2"])
    g = d_rows.cpu().numpy()
    bar = S.lookup_bar(c)
    _lookup_check(g[us, :D], *bar["user"], "user rows")
    _lookup_check(g[np.r_[ps, ns], :D], *bar["item"], "item rows")
    _lookup_check(g[np.r_[ps, ns], D], *bar["bias"], "item bias column")
    assert not g[us, D:].any() and not g[:, D + 1:].any(), "padding / the user rows' bias column must be zero"


@pytest.mark.parametrize("arm", "ac")
@pytest.mark.parametrize("kind", ("gmf", "wrmf", "wrmf_sig"))
@pytest.mark.parametrize("D", (10, 64, 128))
def test_pointwise_grad_rows_lookups(eng, arm, kind, D):
    """orx_pointwise_grad_rows on an arm (a) / (c) case: d_rows[2b] / d_rows[2b + 1] (user / item row, item bias in
    column D) under the per-lookup bar, and GMF's gw with add_w_terms against the summed w gradient."""
    c = S.point_case(arm, kind[:4], O.OPT_SGD, D, 203, S.spec_seed("pgrad_rows", arm, kind, D), sig=kind == "wrmf_sig")
    B = c.B
    uid, iid = c.ids
    rows, slot = _fetched(np.random.default_rng(S.spec_seed("pslots", arm, kind, D)), c,
                          [x for b in range(B) for x in (("user", uid[b]), ("item", iid[b]))])
    w = dev(c.tabs["w"].reshape(-1)) if c.kind == "gmf" else None
    d_rows, gw, _ = eng.pointwise_grad_rows(_kind(c), dev(rows), D, dev(slot, torch.int32), dev(c.label), w, 1.0 / B,
                                            c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False),
                                            c.P["c_loss"], c.P["c_l2"], add_w_terms=True)
    g = d_rows.cpu().numpy()
    bar = S.lookup_bar(c)
    _lookup_check(g[0::2, :D], *bar["user"], "user rows")
    _lookup_check(g[1::2, :D], *bar["item"], "item rows")
    _lookup_check(g[1::2, D], *bar["bias"], "item bias column")
    assert not g[0::2, D:].any() and not g[:, D + 1:].any(), "padding / the user rows' bias column must be zero"
    if c.kind == "gmf":
        _, rws = S.lookups(c, c.state())
        _, G, E = S.dedup(*rws["w"])
        _lookup_check(gw.cpu().numpy(), G[0], E[0] + 2 * S.ulp32(G[0]), "gw")


# ---- the sparse / dense applies under arm (d)'s optimizer constants -------------------------------------------------
@pytest.mark.parametrize("opt", range(4))
@pytest.mark.parametrize("D", (12, 64, 128))
@pytest.mark.parametrize("entry", ("sparse", "strided", "bag", "dense"))
def test_apply_constants(eng, opt, D, entry):
    """orx_sparse_apply, orx_sparse_apply_strided, orx_bag_sparse_apply (one-row sum bags) and orx_dense_apply with
    beta1 0.5, beta2 0.75, eps 1e-2 at step 3, on duplicated ids; each row's gradient is summed in float32."""
    rng = np.random.default_rng(S.spec_seed("apply", opt, D, entry))
    R, n = 97, 300
    lr, stp = float(np.float32(S.OPT_LR[opt])), 3
    P = {k: float(np.float32(S.ARM_D[k])) for k in ("eps", "beta1", "beta2")}
    var = S.f32(rng.uniform(-0.3, 0.3, (R, D)))
    old = (var, *S.init_slots(opt, var))
    t = [None if x is None else dev(x) for x in old]
    o = N.opt(opt, lr, step=stp, **P)
    vals = S.f32(rng.standard_normal((n, D)) * 0.1)
    if entry == "dense":
        G = S.f32(rng.standard_normal((R, D)) * 0.1)
        eng.dense_apply(t[0], t[1], t[2], dev(G), o)
        idx, E = np.arange(R), np.zeros_like(G)     # dense Adam (lazy or not) is Adam on every row
        ref, tol = S.update_bar(opt if opt != O.OPT_ADAM_LAZY else O.OPT_ADAM_DENSE, lr, old, idx, G, E, P, stp)
    else:
        ids = rng.integers(0, R - 7, n).astype(np.int32)      # rows R-7.. untouched
        tab = N.table(*t)
        if entry == "sparse":
            eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
        elif entry == "strided":
            ids2 = np.stack([ids[::-1], ids], 1)
            v3 = np.stack([np.zeros_like(vals), vals], 1)
            eng.sparse_apply_strided(tab, dev(ids2, torch.int32), 1, dev(v3), o)
        else:
            sparse = dev(ids.reshape(n, 1), torch.int32)
            eng.bag_sparse_apply(tab, sparse, 0, 1, dev(vals), 0, o)
        idx, G, E = S.dedup(ids, vals, np.zeros_like(vals), np.abs(vals))
        ref, tol = S.update_bar(opt, lr, old, idx, G, E, P, stp)
    torch.cuda.synchronize()
    got = [None if x is None else x.cpu().numpy() for x in t]
    q = S.ratios(ref, tol, got)
    assert max(x for x in q if x is not None) <= 1.0, (entry, opt, D, q)


def test_step_updates_dispatch_coverage():
    """The specs above reach every (op, variant, kind, optimizer, specialised D or generic, index set) combination the
    dispatch can choose: pairwise steps on index sets 0 ("step"), 1 and 2 ("prefetch", "host": each asserts which set
    its record shows), pointwise steps on set 0."""
    dcls = lambda D: D if D in SPECIAL_D else "generic"
    kinds = {"bpr": N.ORX_PAIR_BPR, "ucml": N.ORX_PAIR_UCML, "gmf": N.ORX_POINT_GMF, "wrmf": N.ORX_POINT_WRMF,
             "wrmf_sig": N.ORX_POINT_WRMF}
    seen = set()
    for arm, kind, opt, D, B, entry in S.pair_specs():
        for s in ((0,) if entry == "step" else (1, 2) if entry == "prefetch" else ()):
            seen.add((PAIR_OP, _pair_rule(D, opt)[0], kinds[kind], opt, dcls(D), s))
    for arm, kind, opt, D, B, entry in S.point_specs():
        seen.add((POINT_OP, _point_rule(D)[0], kinds[kind], opt, dcls(D), 0))
    want = {(PAIR_OP, _pair_rule(D, opt)[0], k, opt, dcls(D), s)
            for D in SPECIAL_D + (12,) for opt in range(4) for k in (N.ORX_PAIR_BPR, N.ORX_PAIR_UCML) for s in (0, 1, 2)}
    want |= {(POINT_OP, _point_rule(D)[0], k, opt, dcls(D), 0)
             for D in SPECIAL_D + (10,) for opt in range(4) for k in (N.ORX_POINT_GMF, N.ORX_POINT_WRMF)}
    assert seen == want, (sorted(want - seen), sorted(seen - want))
    assert {D for *_, D, B, e in S.pair_specs() if B % 8} >= {12, 32, 64, 128, 256, 260}, "batch tails"
