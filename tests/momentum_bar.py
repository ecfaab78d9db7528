"""Keras SGD with momentum (ORX_OPT_MOMENTUM) and Nesterov momentum (ORX_OPT_NESTEROV) in float64, their float32
emulation, the update bar of their steps and the cases they run.  CPU only.

For a touched row r with summed gradient G (SparseApplyKerasMomentum on the deduplicated rows), momentum m:
    a[r] = m * a[r] - lr * G;   MOMENTUM: var[r] += a[r];   NESTEROV: var[r] += m * a[r] - lr * G   (a already updated)
Rows a step does not touch keep value and slot.  Dense variables take the same formula element-wise.

The bar follows tests/step_bar.py.  Each element's tolerance is
  ULP   K_ULP float32 ulps of the largest magnitude the element's arithmetic rounds: |m a_old|, |lr G| and |a_new| for the
        slot; for the value also |old|, |new| and, under NESTEROV, |m a_new|.  (The kernels round each product, sum and
        difference once, without FMA: orx_common.cuh.)
  GRAD  how far the float64 update moves when G moves by its float32 error bound E (step_bar's lookups / dedup):
        lr E for the slot and for a MOMENTUM value, (m + 1) lr E for a NESTEROV value, plus m times the slot's tolerance
        under NESTEROV (the value reads the rounded slot).
An element whose update is exactly the identity (a = 0, G = 0 with E = 0, or a row the batch does not touch) has
tolerance 0: it must be bit-identical.  The bar is tight enough that a slot one step stale (var += a_old) or the other
form (NESTEROV's value under MOMENTUM, or the reverse) falls outside it (tests/test_momentum_cpu.py)."""
import numpy as np

import step_bar as S
from oracle import openrec_oracle as O

OPT_MOMENTUM, OPT_NESTEROV = 6, 8   # include/orx.h
KINDS = (OPT_MOMENTUM, OPT_NESTEROV)
MUTANTS = ("stale_a", "other_form", "no_decay")


def momentum_sparse(var, a, indices, values, lr=0.01, momentum=0.9, nesterov=False):
    """Keras momentum on IndexedSlices: dedup (rows summed in batch order, as O.dedup), then the update of the rows
    touched, var and a in place."""
    idx, g = O.dedup(indices, values)
    _update(var, a, idx, g, lr, momentum, nesterov)


def momentum_dense(var, a, grad, lr=0.01, momentum=0.9, nesterov=False):
    """The same formula on every element of a dense variable."""
    new = momentum * a - lr * grad
    a[...] = new
    var += momentum * new - lr * grad if nesterov else new


def _update(var, a, idx, g, lr, m, nesterov, mutant=None):
    old = a[idx]
    new = m * old - lr * g if mutant != "no_decay" else old - lr * g
    a[idx] = new
    nest = nesterov != (mutant == "other_form")
    seen = old if mutant == "stale_a" else new     # the slot the value update reads
    var[idx] += m * seen - lr * g if nest else seen


def f32_update(var, a, idx, g, lr, m, nesterov):
    """The kernels' arithmetic in float32, each product, sum and difference rounded once (no FMA): -> (var, a) copies
    updated at rows idx by the float32 rounding of g."""
    f = np.float32
    v, s = var.astype(f), a.astype(f)
    g, lr, m = g.astype(f), f(lr), f(m)
    lg = lr * g
    new = m * s[idx] - lg
    s[idx] = new
    v[idx] = v[idx] + ((m * new - lg) if nesterov else new)
    return v.astype(np.float64), s.astype(np.float64)


def update_bar(kind, lr, m, old, idx, G, E):
    """-> (ref, tol) of one table (old = (var, a, None)) updated at rows idx by the summed gradients G with error bound E
    (module docstring)."""
    var, a = old[0], old[1]
    nest = kind == OPT_NESTEROV
    a0 = a[idx]
    a1 = m * a0 - lr * G
    d = m * a1 - lr * G if nest else a1
    ref_v, ref_a = var.copy(), a.copy()
    ref_v[idx] += d
    ref_a[idx] = a1
    ulp = lambda *x: S.K_ULP * S.ulp32(np.max(np.abs(np.stack(x)), 0))
    ta = ulp(m * a0, lr * G, a1) + lr * E
    if nest:
        td = ulp(m * a1, lr * G, d) + m * ta + (m + 1) * lr * E
    else:
        td = ta
    tv = ulp(var[idx], ref_v[idx], d) + td
    tol_v, tol_a = np.zeros_like(var), np.zeros_like(a)
    tol_a[idx] = np.where((a1 == a0) & (E == 0), 0.0, ta)
    tol_v[idx] = np.where((d == 0) & (E == 0), 0.0, tv)
    return (ref_v, ref_a, None), (tol_v, tol_a, None)


def momentum_of(case):
    return case.P["beta1"]


class MomBar(S.Bar):
    """The float64 momentum step of a case (to_momentum) and the tolerance of every element of every table and slot."""

    def __init__(self, case):
        self.case = case
        st = case.state()
        _, rows = S.lookups(case, st)
        self.ref, self.tol = {}, {}
        for name in case.names:
            idx, G, E = S.dedup(*rows[name])
            self.ref[name], self.tol[name] = update_bar(case.opt, case.lr, momentum_of(case), st[name], idx, G, E)


def step(case, mutant=None):
    """The float64 step of a case (or a mutant's) -> {name: (var, a, None)}."""
    st = case.state()
    _, rows = S.lookups(case, st)
    new = {}
    for name in case.names:
        idx, val = rows[name][:2]
        var, a = st[name][0].copy(), st[name][1].copy()
        uniq, g = O.dedup(idx, val.reshape(len(idx), -1))
        _update(var, a, uniq, g, case.lr, momentum_of(case), case.opt == OPT_NESTEROV, mutant)
        new[name] = (var, a, None)
    return new


def f32_step(case):
    """The float32 emulation of a case's step from float32 summed gradients -> {name: (var, a, None)}."""
    st = case.state()
    _, rows = S.lookups(case, st)
    new = {}
    for name in case.names:
        idx, G, _ = S.dedup(*rows[name])
        v, a = f32_update(st[name][0], st[name][1], idx, G, case.lr, momentum_of(case), case.opt == OPT_NESTEROV)
        new[name] = (v, a, None)
    return new


# ---- cases ---------------------------------------------------------------------------------------------------------
def to_momentum(case, kind, seed=0):
    """A step_bar Case built for SGD, turned into a momentum case: every table (and w) gets a slot a -- zero under the
    Keras initialisation, else uniform in [-0.02, 0.02] on the 2^-12 grid (dyadic, so arm (c)'s rows with exact-zero
    gradients decay exactly).  The momentum is the case's beta1 (0.9; 0.5 in arm (d))."""
    rng = np.random.default_rng(seed)
    assert case.opt == O.OPT_SGD and kind in KINDS
    case.opt = kind
    for n in case.names:
        t = case.tabs[n]
        a = np.zeros_like(t) if case.init == "keras" else np.round(rng.uniform(-0.02, 0.02, t.shape) * 4096) / 4096
        case.slots[n] = (S.f32(a), None)
    return case


SPECIAL_D, GENERIC_D = (32, 64, 128, 256), 50


def pair_specs():
    """(arm, kind, opt, D, B, ids, entry) of the fused pairwise steps; ids and entry as rowwise_bar's."""
    out = [(arm, k, o, D, 203, "mixed", "step") for arm in S.ARMS for k in S.PAIR_KINDS for o in KINDS
           for D in SPECIAL_D + (GENERIC_D,)]
    out += [(arm, k, o, 128, 4096, "mixed", "step") for arm in "ad" for k in S.PAIR_KINDS for o in KINDS]
    out += [("a", k, o, D, B, ids, "step") for k in S.PAIR_KINDS for o in KINDS for D in (64, 128, GENERIC_D)
            for ids, B in (("owned", 203), ("staged", 200))]
    out += [(arm, k, o, D, 237, "mixed", "prefetch") for arm in "ac" for k in S.PAIR_KINDS for o in KINDS
            for D in SPECIAL_D + (GENERIC_D,)]
    out += [(arm, k, o, D, 1000, "mixed", "host") for arm in "ad" for k in S.PAIR_KINDS for o in KINDS
            for D in (GENERIC_D, 128)]
    return out


def point_specs():
    out = [(arm, k, o, D, 237, "mixed", "step") for arm in S.ARMS for k in ("gmf", "wrmf", "wrmf_sig") for o in KINDS
           for D in SPECIAL_D + (GENERIC_D,)]
    out += [("b", k, o, D, B, ids, "step") for k in ("gmf", "wrmf") for o in KINDS for D in (128, GENERIC_D)
            for ids, B in (("owned", 237), ("staged", 236))]
    return out


def build(spec, seed_offset=0):
    """The momentum Case of one spec (pair_specs / point_specs)."""
    import rowwise_bar as RB
    arm, kind, opt, D, B, ids_mode, _ = spec
    seed = S.spec_seed("momentum", *spec) + seed_offset
    if kind in S.PAIR_KINDS:
        c = S.pair_case(arm, kind, O.OPT_SGD, D, B, seed)
    else:
        c = S.point_case(arm, kind[:4], O.OPT_SGD, D, B, seed, sig=kind == "wrmf_sig")
    if ids_mode != "mixed":
        c = RB._owned_or_staged(c, ids_mode, np.random.default_rng(seed))
    return to_momentum(c, opt, seed)
