"""The update bar of tests/step_bar.py is right, on CPU: for every case tests/test_gpu_step_updates.py runs, the float32
oracle (the same formulas in float32, numpy's summation order) passes with headroom, max err / tol <= 1/4, and every
oracle mutant fails on the cases built for it by err / tol >= 4.

Where a mutant is invisible by nature its cases are the arm that exposes it:
  - beta / eps / margin mutants only differ from the oracle under arm (d)'s non-default constants, and beta only under
    Adam, eps under Adagrad and Adam (SGD has neither), margin only for UCML;
  - Adam at step 1 instead of step t differs only after step 1 (arm (d) runs at step 3);
  - the tie rule and the -30 clamp only matter where a score sits on them: arm (c)'s dyadic tie tables;
  - the use_sigmoid factor only exists for WRMF with use_sigmoid.
Under arm (a)'s Keras slots lazy Adam's first step is nearly sign(G): a scaled G there moves the update only where |G|
is near eps; the loss-gradient mutants are also run under arm (b) and arm (d), where every optimizer sees them."""
import numpy as np
import pytest

import step_bar as S
from oracle import openrec_oracle as O

HEADROOM, MARGIN = 0.25, 4.0
LOSS_MUTANTS = ("g_x0.9", "neighbour_g", "no_bias", "lost_dup")


def _cases():
    out = []
    for spec in S.pair_specs() + S.point_specs():
        out += [(spec, 0)] + ([(spec, 1)] if spec[5] == "prefetch" else [])
    return out


def _mutant_specs():
    """{mutant: [spec]} the cases built for each mutant, all of them among the GPU file's specs."""
    pair, point = S.pair_specs(), S.point_specs()
    m = {}
    for mut in LOSS_MUTANTS:
        m[mut] = [s for s in pair if s[3] == 128 and s[4] == 4096 and s[0] in "abd"]
        m[mut] += [s for s in point if s[3] == 128 and s[0] in "abd"]
    m["tie_flip"] = [s for s in pair if s[0] == "c" and s[5] == "step"]
    m["no_clamp"] = [s for s in pair if s[0] == "c" and s[1] == "bpr" and s[5] == "step"]
    m["margin_0.5"] = [s for s in pair if s[0] == "d" and s[1] == "ucml" and s[5] == "step"]
    adam = lambda s: s[0] == "d" and s[2] in (O.OPT_ADAM_LAZY, O.OPT_ADAM_DENSE) and s[5] == "step"
    for mut in ("beta_swap", "beta_default", "adam_step1"):
        m[mut] = [s for s in pair + point if adam(s)]
    m["eps_default"] = [s for s in pair + point if s[0] == "d" and s[2] != O.OPT_SGD and s[5] == "step"]
    m["neighbour_label"] = [s for s in point if s[1] != "wrmf_sig" and s[0] in "ab"]
    m["no_sig_factor"] = [s for s in point if s[1] == "wrmf_sig" and s[0] in "abd"]
    return m


def test_lookups_match_oracle():
    """The per-lookup gradients step_bar judges with are the oracle's *_grads, summed per row."""
    for spec in (("b", "bpr", 0, 12, 203, "step"), ("d", "ucml", 0, 32, 203, "step"), ("b", "gmf", 0, 10, 237, "step"),
                 ("d", "wrmf_sig", 0, 10, 237, "step")):
        c = S.build(spec)
        t = c.state()
        P = c.P
        if c.kind == "bpr":
            gr = O.bpr_grads(*(t[n][0] for n in c.names), *c.ids, P["c_loss"], P["c_l2"])
        elif c.kind == "ucml":
            gr = O.ucml_grads(*(t[n][0] for n in c.names), *c.ids, P["margin"], P["c_loss"], P["c_l2"])
        elif c.kind == "gmf":
            user, item, bias, w = (t[n][0] for n in c.names)
            gr = O.gmf_grads(user, item, bias, w.reshape(-1, 1), *c.ids, c.label, P["c_loss"], P["c_l2"])
        else:
            gr = O.wrmf_grads(*(t[n][0] for n in c.names), *c.ids, c.label, P["a"], P["b"], P["sig"], P["c_loss"],
                              P["c_l2"])
        _, rows = S.lookups(c, t)
        for name in ("user", "item", "bias"):
            idx, val = gr[name]
            np.testing.assert_allclose(rows[name][1], val.reshape(len(idx), -1), rtol=1e-12, atol=1e-15)
        if c.kind == "gmf":
            np.testing.assert_allclose(rows["w"][1].sum(0), gr["w"].reshape(-1), rtol=1e-12, atol=1e-15)


def test_dyadic_ties_are_exact():
    """The tie triplets of arm (c) sit exactly on their targets, in float32 as in float64."""
    for kind, ties in (("bpr", S.BPR_TIES), ("ucml", S.UCML_TIES)):
        for D in (12, 260):
            c = S.dyadic_pair(kind, 0, D, 203, 7, margin=1.25 if kind == "ucml" else 0.5)
            for dt in (np.float32, np.float64):
                tb = {n: c.tabs[n].astype(dt) for n in c.names}
                uid, pid, nid = c.ids
                u, p, n = tb["user"][uid], tb["item"][pid], tb["item"][nid]
                bp, bn = tb["bias"][pid, 0], tb["bias"][nid, 0]
                if kind == "bpr":
                    s = ((u * p).sum(1, dtype=dt) + bp) - ((u * n).sum(1, dtype=dt) + bn)
                else:
                    dp, dn = ((u - p) ** 2).sum(1, dtype=dt), ((u - n) ** 2).sum(1, dtype=dt)
                    s = dt(c.P["margin"]) - ((-dp + bp) - (-dn + bn))
                want = np.array([ties[4 if kind == "bpr" else 3]] * 3 + [t for t in ties for _ in range(4)])
                assert np.array_equal(s[:len(want)].astype(np.float64), want), (kind, D, dt)
    for kind in ("gmf", "wrmf"):
        c = S.dyadic_point(kind, 0, 260, 203, 7)
        uid, iid = c.ids
        u, i, b = c.tabs["user"][uid], c.tabs["item"][iid], c.tabs["bias"][iid, 0]
        z = ((u * i * c.tabs["w"][0]).sum(1) if kind == "gmf" else (u * i).sum(1)) + b
        t = S.POINT_TIES[kind]
        assert np.array_equal(z[:11], [t[0]] * 3 + [x for x in t for _ in range(4)])


@pytest.mark.parametrize("spec", S.loopback_specs())
def test_loopback_cases(spec):
    """The two-rank sharded step's cases: the float32 oracle within the headroom, and the loss-gradient mutants (the
    global 1 / B, a cross-rank duplicate's lost contribution) and, under arm (d), the constant mutants fail."""
    c = S.loopback_case(*spec)
    bar = S.Bar(c)
    assert bar.worst(S.step(c, np.float32))[0] <= HEADROOM
    muts = list(LOSS_MUTANTS) + (["eps_default"] if spec[1] == "d" and spec[3] else []) + \
        (["beta_swap", "adam_step1"] if spec[1] == "d" and spec[3] == O.OPT_ADAM_LAZY else []) + \
        (["margin_0.5"] if spec[1] == "d" and spec[2] == "ucml" else [])
    for mut in muts:
        q, where = bar.worst(S.step(c, np.float64, mut))
        assert q >= MARGIN, (spec, mut, where, q)


def test_float32_oracle_headroom(capsys):
    worst, by = 0.0, {}
    for spec, off in _cases():
        c = S.build(spec, off)
        q, where = S.Bar(c).worst(S.step(c, np.float32))
        assert q <= HEADROOM, (spec, off, where, q)
        key = (spec[0], spec[1])
        by[key] = max(by.get(key, 0.0), q)
        worst = max(worst, q)
    with capsys.disabled():
        print(f"\nfloat32 oracle, max err/tol over {len(_cases())} cases: {worst:.3f}")
        for k in sorted(by):
            print(f"  arm {k[0]} {k[1]:9s} {by[k]:.3f}")


@pytest.mark.parametrize("mutant", list(_mutant_specs()))
def test_mutant_fails(mutant, capsys):
    specs = _mutant_specs()[mutant]
    assert specs
    low = np.inf
    for spec in specs:
        c = S.build(spec)
        q, where = S.Bar(c).worst(S.step(c, np.float64, mutant))
        assert q >= MARGIN, (mutant, spec, where, q)
        low = min(low, q)
    with capsys.disabled():
        print(f"\nmutant {mutant:15s} fails all {len(specs):3d} of its cases, min max-err/tol {low:.3g}")
