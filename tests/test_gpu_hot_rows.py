"""The sparse steps and applies on hot rows, judged by tests/hot_rows.py's exact bar.

Every case's summed row gradients are exact in float32 whatever the order of the staging atomics
(tests/test_hot_rows_cpu.py proves it for each case here), so the bar has no gradient term: SGD, momentum and Nesterov
must give the float64 tables and slots bit for bit, Adagrad, row-wise Adagrad and both Adams must stay within a few
float32 ulps and the MUFU divide.  A hot row that loses one staged contribution, or gets one twice, fails by orders of
magnitude -- at Zipf(1.05) batches of 65 536 lookups, where step_bar's bar cannot see it.

Each fused step asserts the kernel its dispatch record names, its loss and l2, its bad-id count and its staged-row count;
rows a step does not touch are compared with their copy from before the step on the device."""
import numpy as np
import pytest
import torch

import hot_rows as H
import momentum_bar as MB
import rowwise_bar as RB
import step_bar as S
from oracle import openrec_oracle as O
from openrec_b200 import native as N
from test_gpu_kernels import PAIR_OP, POINT_OP, SPECIAL_D, _pair_rule, _point_rule, dev
from test_gpu_momentum import _pair_rule as _mom_pair_rule

pytestmark = pytest.mark.gpu
KINDS = {"bpr": N.ORX_PAIR_BPR, "ucml": N.ORX_PAIR_UCML, "gmf": N.ORX_POINT_GMF, "wrmf": N.ORX_POINT_WRMF}


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def _sid(s):
    return "-".join(map(str, s))


def _rule(op, D, opt):
    if op == POINT_OP:
        return _point_rule(D)
    return _mom_pair_rule(D) if opt in MB.KINDS else _pair_rule(D, opt)


def _check_dispatch(e, op, c, index_set=0):
    """The one record of the step just launched names the kernel of the rule; -> its index set."""
    v, minb = _rule(op, c.D, c.opt)
    got = e.debug_dispatch_log()
    assert len(got) == 1, got
    s = got[0].s if index_set == "prefetch" else index_set
    assert got[0] == N.Dispatch(op, v, KINDS[c.kind], c.opt, c.B, c.D, minb, s), got[0]
    if index_set == "prefetch":
        assert s in (1, 2), got[0]
    return s


def _opt(c):
    return N.opt(c.opt, c.lr, eps=c.P["eps"], beta1=c.P["beta1"], beta2=c.P["beta2"], step=c.step)


class Dev:
    """A case's tables and slots on the device, and their copies from before the step."""

    def __init__(self, c):
        self.c = c
        self.t = {n: [None if x is None else dev(x) for x in (c.tabs[n], *c.slots[n])] for n in c.names}
        kind = lambda n: RB.OPT_ROWWISE_ADAGRAD if c.opt == RB.OPT_ROWWISE_ADAGRAD and n in RB.TABLES else None
        self.tt = {n: N.table(*v, kind=kind(n)) for n, v in self.t.items()}
        self.before = {n: [None if x is None else x.clone() for x in v] for n, v in self.t.items()}

    def got(self):
        torch.cuda.synchronize()
        return {n: tuple(None if x is None else x.cpu().numpy().astype(np.float64) for x in v)
                for n, v in self.t.items()}

    def check_untouched(self, what=""):
        """Rows no lookup references keep value and slots bit for bit (dense Adam moves every row)."""
        c = self.c
        if c.opt == O.OPT_ADAM_DENSE:
            return
        refs = {"user": [c.ids[0]], "item": list(c.ids[1:]) if c.kind in S.PAIR_KINDS else [c.ids[1]]}
        refs["bias"] = refs["item"]
        for n in ("user", "item", "bias"):
            keep = torch.ones(len(c.tabs[n]), dtype=torch.bool, device="cuda")
            keep[dev(np.concatenate(refs[n]), torch.int64)] = False
            for j, (x, x0) in enumerate(zip(self.t[n], self.before[n])):
                if x is not None:
                    assert torch.equal(x[keep], x0[keep]), f"{what} {c}: an untouched {n} row moved ({j})"


def _launch(e, c, d, entry="step", dids=None):
    out = torch.zeros(4, device="cuda")
    if c.kind in S.PAIR_KINDS:
        P = dict(margin=c.P["margin"], c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
        if entry == "host":
            ids = [torch.from_numpy(x).pin_memory() for x in c.ids]
            out = torch.zeros(4).pin_memory()
            e.pairwise_step_host(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c), out, **P)
            torch.cuda.synchronize()       # the pinned ids must outlive the upload
        else:
            e.pairwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"],
                            *(dids or [dev(x, torch.int32) for x in c.ids]), _opt(c), out, **P)
    else:
        e.pointwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], d.tt.get("w"),
                         *(dev(x, torch.int32) for x in c.ids), dev(c.label), _opt(c), out,
                         c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False),
                         c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    return out


def _judge(c, d, out, what):
    got = out.cpu().numpy().astype(np.float64)
    loss, l2 = H.loss_l2(c)
    np.testing.assert_allclose(got[0], loss, rtol=2e-5, atol=1e-5, err_msg=f"loss {what} {c}")
    np.testing.assert_allclose(got[1], l2, rtol=2e-5, atol=1e-5, err_msg=f"l2 {what} {c}")
    assert got[2] == 0, (what, c, got)
    assert got[3] == H.staged_rows(c), (what, c, got[3], H.staged_rows(c))
    d.check_untouched(what)
    H.ExactBar(c).judge(d.got(), what)


class _Fresh:
    """The module's engine, or for a cluster case a handle of its own: its batch index is sized for this very batch
    (a handle keeps the index of the largest batch it has seen), so the cluster's ids home into its last slots."""

    def __init__(self, eng, spec):
        self.own = spec[4] == "cluster"
        self.e = N.Engine(torch.cuda.current_device()) if self.own else eng

    def __enter__(self):
        return self.e

    def __exit__(self, *a):
        if self.own:
            torch.cuda.synchronize()
            self.e.close()


@pytest.mark.parametrize("spec", H.pair_specs(), ids=_sid)
def test_hot_pairwise_step(eng, spec):
    entry = spec[5]
    with _Fresh(eng, spec) as e:
        e.debug_dispatch_log()
        if entry == "prefetch":
            # bench.py's loop: the next batch's index is built on the side stream right after this step is queued;
            # the two batches share their hot rows, each step has tables of its own
            cs = [H.build(spec, k) for k in (0, 1)]
            ds = [Dev(c) for c in cs]
            dids = [[dev(x, torch.int32) for x in c.ids] for c in cs]
            torch.cuda.synchronize()
            e.pairwise_prefetch(ds[0].tt["user"], ds[0].tt["item"], *dids[0], cs[0].opt, ids_ready=True)
            outs, sets = [], []
            for k in (0, 1):
                outs.append(_launch(e, cs[k], ds[k], "step", dids[k]))
                if k == 0:
                    e.pairwise_prefetch(ds[1].tt["user"], ds[1].tt["item"], *dids[1], cs[1].opt, ids_ready=True)
                recs = e.debug_dispatch_log()
                assert len(recs) == 1, recs
                v, minb = _rule(PAIR_OP, cs[k].D, cs[k].opt)
                assert recs[0] == N.Dispatch(PAIR_OP, v, KINDS[cs[k].kind], cs[k].opt, cs[k].B, cs[k].D, minb,
                                             recs[0].s), recs[0]
                sets.append(recs[0].s)
            assert sorted(sets) == [1, 2], sets
            for k in (0, 1):
                _judge(cs[k], ds[k], outs[k], f"prefetched step {k}")
            return
        c = H.build(spec)
        d = Dev(c)
        out = _launch(e, c, d, entry)
        _check_dispatch(e, PAIR_OP, c, "prefetch" if entry == "host" else 0)
        _judge(c, d, out, entry)


@pytest.mark.parametrize("spec", H.point_specs(), ids=_sid)
def test_hot_pointwise_step(eng, spec):
    with _Fresh(eng, spec) as e:
        c = H.build(spec)
        d = Dev(c)
        e.debug_dispatch_log()
        out = _launch(e, c, d)
        _check_dispatch(e, POINT_OP, c)
        _judge(c, d, out, "pointwise step")


def test_hot_rows_dispatch_coverage():
    """The specs above reach every specialised and generic kernel instance the dispatch rules list, for each op, kind and
    optimizer, the pairwise step on index sets 0, 1 and 2."""
    dcls = lambda D: D if D in SPECIAL_D else "generic"
    kinds = dict(KINDS, wrmf_sig=N.ORX_POINT_WRMF)
    seen = set()
    for kind, opt, D, B, p, entry in H.pair_specs():
        for s in ((0,) if entry == "step" else (1, 2) if entry == "prefetch" else ()):
            seen.add((PAIR_OP, _rule(PAIR_OP, D, opt), kinds[kind], opt, dcls(D), s))
    for kind, opt, D, B, p, entry in H.point_specs():
        seen.add((POINT_OP, _rule(POINT_OP, D, opt), kinds[kind], opt, dcls(D), 0))
    want = {(PAIR_OP, _rule(PAIR_OP, D, o), k, o, dcls(D), s) for D in H.DIMS for o in H.OPTS
            for k in (N.ORX_PAIR_BPR, N.ORX_PAIR_UCML) for s in (0, 1, 2)}
    want |= {(POINT_OP, _rule(POINT_OP, D, o), k, o, dcls(D), 0) for D in H.DIMS for o in H.OPTS
             for k in (N.ORX_POINT_GMF, N.ORX_POINT_WRMF)}
    assert seen == want, (sorted(want - seen), sorted(seen - want))
    specs = H.pair_specs() + H.point_specs()
    assert {s[4] for s in specs} == set(H.PATTERNS) and {1, H.tail_batch(), 4096, 65536} <= {s[3] for s in specs}
    for k in H.KINDS:
        assert {s[3] for s in specs if s[0] == k} >= {1, H.tail_batch(), 4096}, k


# ---- un-fused applies on hot ids -------------------------------------------------------------------------------------
def _apply_ref(opt, old, idx, G):
    """(ref, tol) of one table updated at rows idx by the exact summed gradients G (E = 0)."""
    E = np.zeros_like(G)
    if opt in MB.KINDS:
        return MB.update_bar(opt, H.LR, H.MOMENTUM, old, idx, G, E)
    P = {k: float(np.float32(v)) for k, v in (("eps", 1e-7), ("beta1", 0.9), ("beta2", 0.999))}
    if opt == RB.OPT_ROWWISE_ADAGRAD:
        return RB.row_update_bar(H.LR, P["eps"], old, idx, G, E)
    return S.update_bar(opt, H.LR, old, idx, G, E, P, 1)


def _apply_slots(opt, var, rng):
    c = S.Case("bpr", O.OPT_SGD, (var, var[:, :1], var[:, :1]), (np.zeros(1),) * 3, lr=H.LR)
    c.opt = opt
    c.names = ("user",)
    return H.set_slots(c, rng).slots["user"]


@pytest.mark.parametrize("opt", H.OPTS)
@pytest.mark.parametrize("D", (128, 12))
@pytest.mark.parametrize("entry", ("sparse", "strided", "bag_sum", "bag_mean"))
def test_hot_apply(eng, entry, D, opt):
    """orx_sparse_apply, orx_sparse_apply_strided (DLRM's [n, F] ids / [n, F, D] rows) and orx_bag_sparse_apply (sum bags,
    mean bags of 1, 2 or 4 valid ids, the division exact) on Zipf ids over 4096 rows: 16 384 lookups, hot rows with
    thousands, dyadic value rows on the 2^-4 grid.  Rows 4000.. are never referenced."""
    rng = np.random.default_rng(H.seed_of("apply", entry, D, opt))
    R, n = 4096, 16384
    var = H.grid(rng, (R, D))
    old = (var, *_apply_slots(opt, var, rng))
    t = [None if x is None else dev(x) for x in old]
    before = [None if x is None else x.clone() for x in t]
    tab = N.table(*t, kind=opt if opt == RB.OPT_ROWWISE_ADAGRAD else None)
    o = N.opt(opt, H.LR, beta1=H.MOMENTUM if opt in MB.KINDS else 0.9)
    ids = H.zipf_draw(4000, n, rng, rng.permutation(4000)).astype(np.int32)
    vals = H.grid(rng, (n, D), 1.0)
    if entry == "sparse":
        eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
        lk_ids, lk_vals = ids, vals
    elif entry == "strided":
        eng.sparse_apply_strided(tab, dev(np.stack([ids[::-1], ids], 1), torch.int32), 1,
                                 dev(np.stack([np.zeros_like(vals), vals], 1)), o)
        lk_ids, lk_vals = ids, vals
    else:
        Lmax, nb = 4, n // 2
        sizes = rng.choice([1, 2, 4], nb)
        sp = np.full((nb, Lmax), -1, np.int32)
        pool = np.resize(ids, sizes.sum())
        k = 0
        for b, m in enumerate(sizes):
            sp[b, :m] = pool[k:k + m]
            k += m
        dz = vals[:nb]
        mean = entry == "bag_mean"
        eng.bag_sparse_apply(tab, dev(sp, torch.int32), 0, Lmax, dev(dz), 1 if mean else 0, o)
        b_of, l_of = np.nonzero(sp >= 0)
        lk_ids = sp[b_of, l_of]
        lk_vals = dz[b_of] / sizes[b_of, None] if mean else dz[b_of]
    idx, G = O.dedup(lk_ids, lk_vals)
    ref, tol = _apply_ref(opt, old, idx, G)
    torch.cuda.synchronize()
    got = [None if x is None else x.cpu().numpy().astype(np.float64) for x in t]
    if opt in H.EXACT_OPTS:
        for j, (g, r) in enumerate(zip(got, ref)):
            if r is not None:
                assert np.array_equal(g.reshape(r.shape), r), (entry, opt, j)
    else:
        q = S.ratios(ref, tol, got)
        assert max(x for x in q if x is not None) <= 1.0, (entry, opt, D, q)
    if opt != O.OPT_ADAM_DENSE:
        for x, x0 in zip(t, before):
            if x is not None:
                assert torch.equal(x[4000:], x0[4000:]), (entry, opt)


# ---- the bench shape -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prefetch", (False, True))
def test_hot_bench_shape(eng, prefetch):
    """bench.py's bpr_zipf1.05 batch: BPR under Adagrad at U = I = 1M, D = 128, B = 65 536 Zipf(1.05) triplets, through
    the step bench.py times (unprefetched) and the prefetched one.  The touched rows against the float64 step (a case of
    those rows only: Adagrad updates rows independently), the untouched ones bit for bit on the device."""
    U = I = 1 << 20
    D, B = 128, 65536
    rng = np.random.default_rng(H.seed_of("bench", prefetch))
    ur, ir = rng.permutation(U), rng.permutation(I)
    ids = [H.zipf_draw(U, B, rng, ur), H.zipf_draw(I, B, rng, ir), H.zipf_draw(I, B, rng, ir)]
    ids = [x.astype(np.int32) for x in ids]
    h = D // 2
    gen = torch.Generator(device="cuda").manual_seed(7)
    g16 = lambda *s: torch.randint(-8, 9, s, generator=gen, device="cuda", dtype=torch.int32).float() / 16
    user = torch.zeros(U, D, device="cuda")
    user[:, :h] = g16(U, h)
    item = torch.empty(I, D, device="cuda")
    item[:, :h] = g16(1, h)
    item[:, h:] = g16(I, D - h)
    bias = torch.zeros(I, 1, device="cuda")
    t = {"user": [user, torch.full_like(user, 0.125)], "item": [item, torch.full_like(item, 0.125)],
         "bias": [bias, torch.full_like(bias, 0.125)]}
    before = {n: [x.clone() for x in v] for n, v in t.items()}
    tt = {n: N.table(*v) for n, v in t.items()}
    uu, ui = np.unique(ids[0]), np.unique(np.concatenate(ids[1:]))
    rows = {"user": uu, "item": ui, "bias": ui}
    # the case of the touched rows, ids renumbered into them
    sub = [before[n][0][dev(rows[n], torch.int64)].cpu().numpy().astype(np.float64) for n in ("user", "item", "bias")]
    cids = (np.searchsorted(uu, ids[0]), np.searchsorted(ui, ids[1]), np.searchsorted(ui, ids[2]))
    c = H.case_of("bpr", O.OPT_ADAGRAD, sub, cids, rng)       # Adagrad accumulators 1/8, as on the device
    H.assert_exact(c)
    dids = [dev(x, torch.int32) for x in ids]
    torch.cuda.synchronize()
    eng.debug_dispatch_log()
    if prefetch:
        eng.pairwise_prefetch(tt["user"], tt["item"], *dids, O.OPT_ADAGRAD, ids_ready=True)
    out = torch.zeros(4, device="cuda")
    eng.pairwise_step(N.ORX_PAIR_BPR, tt["user"], tt["item"], tt["bias"], *dids, _opt(c), out, c_loss=float(B),
                      c_l2=0.0)
    _check_dispatch(eng, PAIR_OP, c, "prefetch" if prefetch else 0)
    torch.cuda.synchronize()
    got = {n: tuple(x[dev(rows[n], torch.int64)].cpu().numpy().astype(np.float64) for x in t[n]) + (None,)
           for n in c.names}
    H.ExactBar(c).check(got, f"bench shape, prefetch {prefetch}")
    o = out.cpu().numpy()
    np.testing.assert_allclose(o[:2], H.loss_l2(c), rtol=2e-5)
    assert o[2] == 0 and o[3] == H.staged_rows(c), o
    for n in c.names:
        keep = torch.ones(len(t[n][0]), dtype=torch.bool, device="cuda")
        keep[dev(rows[n], torch.int64)] = False
        for x, x0 in zip(t[n], before[n]):
            assert torch.equal(x[keep], x0[keep]), n


# ---- the home-routed sharded step ------------------------------------------------------------------------------------
def _loopback_specs():
    return [(w, k, o, p) for w in (2, 4) for k in S.PAIR_KINDS for o in (O.OPT_SGD, O.OPT_ADAGRAD, O.OPT_ADAM_LAZY,
                                                                          MB.OPT_MOMENTUM)
            for p in ("zipf", "one_row")]


@pytest.mark.parametrize("world,kind,opt,pattern", _loopback_specs())
def test_hot_loopback(world, kind, opt, pattern):
    """orx_shard_step with `world` virtual ranks on one GPU, on the global batch (256 triplets a rank) of an exact case:
    hot rows shared by every rank, reduced across them at their home."""
    from openrec_b200.sharded import LoopbackGroup
    B, D = 256, 128
    c = H.make_case(kind, opt, D, B * world, pattern, H.seed_of("loopback", world, kind, opt, pattern))
    H.assert_exact(c)
    P = c.P
    g = LoopbackGroup(world, len(c.tabs["user"]), len(c.tabs["item"]), D, B, kind=S.PAIR_KINDS.index(kind),
                      opt_kind=opt, lr=c.lr, eps=P["eps"], beta1=P["beta1"], beta2=P["beta2"], margin=P["margin"],
                      init=False)
    try:
        g.load_global(*(c.tabs[n] for n in c.names))
        for m in g.ranks:
            m.iterations = c.step - 1
            for name, slots in zip(c.names, (m.user_slots, m.item_slots, m.bias_slots)):
                for k, s in enumerate(c.slots[name]):
                    if s is not None:
                        local = s[m.rank::world]
                        slots[k][:len(local)] = torch.as_tensor(local, dtype=torch.float32).reshape(-1, s.shape[1])
        batches = [tuple(torch.from_numpy(a[r * B:(r + 1) * B].copy()).cuda() for a in c.ids) for r in range(world)]
        g.step(batches, c_loss=P["c_loss"], c_l2=P["c_l2"])
        g.check()
        torch.cuda.synchronize()
        got = {}
        for j, name in enumerate(c.names):
            arrs = [c.tabs[name].copy()] + [None if s is None else s.copy() for s in c.slots[name]]
            for m in g.ranks:
                n_loc = len(arrs[0][m.rank::world])
                shard = (m.local_shards()[j], *((m.user_slots, m.item_slots, m.bias_slots)[j]))
                for a, x in zip(arrs, shard):
                    if a is not None:
                        a[m.rank::world] = x[:n_loc].cpu().numpy().reshape(n_loc, -1)
            got[name] = tuple(arrs)
        H.ExactBar(c).judge(got, f"loopback world {world}")
    finally:
        g.close()
