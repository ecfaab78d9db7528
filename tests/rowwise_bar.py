"""Row-wise Adagrad (ORX_OPT_ROWWISE_ADAGRAD) in float64, the update bar of its steps and the cases they run.  CPU only.

One accumulator per table row: for a touched row r with summed gradient G (D elements),
    acc[r] += (1/D) * sum_j G[j]^2;   var[r][j] -= lr * G[j] / (sqrt(acc[r]) + eps).
A dim-1 table (the item bias) is element-wise Adagrad, which the same formula is at D = 1.

The bar follows tests/step_bar.py (K_ULP float32 ulps, the MUFU divide, each row's gradient error bound E carried through
the update), with one change: the update couples a row's elements through acc, so the +-E probe of step_bar.update_bar
is no bound (G + E raises sum G^2 only where G > 0).  The accumulator's increment is bounded by the sign-aligned
perturbations sum (|G| + E)^2 / D and sum max(|G| - E, 0)^2 / D, widened by the float32 rounding of a D-term sum, and
each element's update by the four corners (G_j +- E_j) x (that lowest / highest accumulator).  A row whose every
contribution is an exact zero has tolerance 0 in value and accumulator: it must be bit-identical, as untouched rows."""
import numpy as np

import step_bar as S
from oracle import openrec_oracle as O

OPT_ROWWISE_ADAGRAD = 5   # include/orx.h
TABLES = ("user", "item")   # the row tables of a step; the item bias and GMF's w keep element-wise Adagrad


def adagrad_rowwise_sparse(var, acc, indices, values, lr=0.001, eps=1e-7):
    """Row-wise Adagrad on the deduplicated rows (rows summed in batch order, as O.dedup): acc has one element per row
    of var ([rows] or [rows, 1]) and is updated in place, as var is."""
    idx, g = O.dedup(indices, values)
    a = acc.reshape(-1)
    new = a[idx] + (g * g).sum(1) / g.shape[1]
    a[idx] = new
    var[idx] -= var.dtype.type(lr) * g / (np.sqrt(new)[:, None] + var.dtype.type(eps))


def to_rowwise(case, seed=0):
    """A step_bar Case built for Adagrad, turned into its row-wise form: the user / item tables get one accumulator
    per row (Keras init 0.1, or uniform in [0.05, 0.3] for a "nontrivial" case), the item bias and w keep their
    element-wise ones."""
    rng = np.random.default_rng(seed)
    assert case.opt == O.OPT_ADAGRAD
    case.opt = OPT_ROWWISE_ADAGRAD
    for n in TABLES:
        rows = case.tabs[n].shape[0]
        acc = np.full(rows, 0.1) if case.init == "keras" else rng.uniform(0.05, 0.3, rows)
        case.slots[n] = (S.f32(acc), None)
    return case


def row_update_bar(lr, eps, old, idx, G, E):
    """-> (ref, tol) of one row table (old = (var, acc [rows], None)) updated at rows idx by summed gradients G with
    error bound E (module docstring)."""
    var, acc = old[0], old[1].reshape(-1)
    D = G.shape[1]
    a0 = acc[idx]
    rnd = (D + 2) * S.U24
    hi = ((np.abs(G) + E) ** 2).sum(1) / D
    lo = (np.maximum(np.abs(G) - E, 0.0) ** 2).sum(1) / D
    a_ref = a0 + (G * G).sum(1) / D
    a_hi, a_lo = a0 + hi * (1 + rnd), a0 + lo * (1 - rnd)
    upd = lambda g, a: var[idx] - lr * g / (np.sqrt(a)[:, None] + eps)
    r = upd(G, a_ref)
    grad = np.zeros_like(r)
    for s in (1.0, -1.0):
        for a in (a_hi, a_lo):
            grad = np.maximum(grad, np.abs(upd(G + s * E, a) - r))
    ref_v, tol_v = var.copy(), np.zeros_like(var)
    ref_v[idx] = r
    o = var[idx]
    delta = np.abs(r - o)
    t = S.K_ULP * S.ulp32(np.maximum(np.abs(o), np.abs(r))) + S.R_MUFU * delta + grad
    tol_v[idx] = np.where((delta == 0) & (grad == 0), 0.0, t)
    ref_a, tol_a = acc.copy(), np.zeros_like(acc)
    ref_a[idx] = a_ref
    ta = S.K_ULP * S.ulp32(a_ref) + np.maximum(a_hi - a_ref, a_ref - a_lo)
    tol_a[idx] = np.where(hi == 0, 0.0, ta)
    return (ref_v, ref_a, None), (tol_v, tol_a, None)


class RowBar(S.Bar):
    """The float64 row-wise step of a case (to_rowwise) and the tolerance of every element: user / item tables under
    row_update_bar, the item bias (and w) under step_bar's element-wise Adagrad bar."""

    def __init__(self, case):
        self.case = case
        st = case.state()
        _, rows = S.lookups(case, st)
        P, stp = S._opt_consts(case, None)
        self.ref, self.tol = {}, {}
        for name in case.names:
            idx, G, E = S.dedup(*rows[name])
            if name in TABLES and case.D > 1:
                self.ref[name], self.tol[name] = row_update_bar(case.lr, P["eps"], st[name], idx, G, E)
            else:
                self.ref[name], self.tol[name] = S.update_bar(O.OPT_ADAGRAD, case.lr, st[name], idx, G, E, P, stp)


def step(case):
    """The float64 row-wise step of a case -> {name: (var, s0, None)}."""
    st = case.state()
    _, rows = S.lookups(case, st)
    new = {}
    for name in case.names:
        idx, val = rows[name][:2]
        var, s0 = st[name][0].copy(), st[name][1].copy()
        if name in TABLES:
            adagrad_rowwise_sparse(var, s0, idx, val.reshape(len(idx), -1), case.lr, case.P["eps"])
        else:
            O.adagrad_sparse(var, s0, idx, val.reshape(len(idx), -1), case.lr, case.P["eps"])
        new[name] = (var, s0, None)
    return new


# ---- cases ---------------------------------------------------------------------------------------------------------
# (arm, kind, D, B, ids, entry).  ids: "mixed" (step_bar's cases: uniform ids, some rows seen once, some more often),
# "owned" (every row referenced once), "staged" (every row referenced at least twice).  entry as step_bar's.
SPECIAL_D, GENERIC_D = (32, 64, 128, 256), 50


def pair_specs():
    out = [(arm, k, D, 203, "mixed", "step") for arm in S.ARMS for k in S.PAIR_KINDS for D in SPECIAL_D + (GENERIC_D,)]
    out += [(arm, k, 128, 4096, "mixed", "step") for arm in "ad" for k in S.PAIR_KINDS]
    out += [("a", k, D, B, ids, "step") for k in S.PAIR_KINDS for D in (64, 128, GENERIC_D)
            for ids, B in (("owned", 203), ("staged", 200))]
    out += [(arm, k, D, 237, "mixed", "prefetch") for arm in "ac" for k in S.PAIR_KINDS
            for D in SPECIAL_D + (GENERIC_D,)]
    out += [(arm, k, D, 1000, "mixed", "host") for arm in "ad" for k in S.PAIR_KINDS for D in (GENERIC_D, 128)]
    return out


def point_specs():
    out = [(arm, k, D, 237, "mixed", "step") for arm in S.ARMS for k in ("gmf", "wrmf", "wrmf_sig")
           for D in SPECIAL_D + (GENERIC_D,)]
    out += [("b", k, D, B, ids, "step") for k in ("gmf", "wrmf") for D in (128, GENERIC_D)
            for ids, B in (("owned", 237), ("staged", 236))]
    return out


def _owned_or_staged(c, ids_mode, rng):
    """Replace a random case's ids: "owned" -- every user and item row once in the batch (tables grown to hold them);
    "staged" -- every user row twice, every item row twice over the batch's item lookups."""
    B = c.B
    pair = c.kind in S.PAIR_KINDS
    n_item = 2 * B if pair else B
    if ids_mode == "owned":
        U, I = B + 3, n_item + 5
        uid = rng.permutation(U)[:B]
        items = rng.permutation(I)[:n_item]
    else:
        U, I = B // 2, n_item // 2
        uid = rng.permutation(np.repeat(np.arange(U), 2))
        items = rng.permutation(np.repeat(np.arange(I), 2))
    sc = 0.05 if c.kind == "bpr" else 0.4 if c.kind == "ucml" else 0.3
    c.tabs["user"] = S.f32(rng.uniform(-sc, sc, (U, c.D)))
    c.tabs["item"] = S.f32(rng.uniform(-sc, sc, (I, c.D)))
    c.tabs["bias"] = S.f32(rng.uniform(-sc, sc, (I, 1)))
    c.slots["bias"] = S.init_slots(O.OPT_ADAGRAD, c.tabs["bias"], c.init)
    ids = (uid, items[:B], items[B:]) if pair else (uid, items)
    c.ids = tuple(np.asarray(x, np.int32) for x in ids)
    if c.kind == "ucml":     # keep every triplet off the hinge's kink (step_bar's module docstring): move its p's bias
        uid, pid, nid = c.ids
        for _ in range(20):
            user, item, bias = c.tabs["user"], c.tabs["item"], c.tabs["bias"][:, 0]
            dp, dn = ((user[uid] - item[pid]) ** 2).sum(1), ((user[uid] - item[nid]) ** 2).sum(1)
            bad = np.abs(c.P["margin"] - ((-dp + bias[pid]) - (-dn + bias[nid]))) < 1e-3
            if not bad.any():
                break
            c.tabs["bias"][pid[bad], 0] = S.f32(c.tabs["bias"][pid[bad], 0] + 0.01)
        assert not bad.any()
    return c


def build(spec, seed_offset=0):
    """The row-wise Case of one spec (pair_specs / point_specs)."""
    arm, kind, D, B, ids_mode, _ = spec
    seed = S.spec_seed("rowwise", *spec) + seed_offset
    if kind in S.PAIR_KINDS:
        c = S.pair_case(arm, kind, O.OPT_ADAGRAD, D, B, seed)
    else:
        c = S.point_case(arm, kind[:4], O.OPT_ADAGRAD, D, B, seed, sig=kind == "wrmf_sig")
    if ids_mode != "mixed":
        c = _owned_or_staged(c, ids_mode, np.random.default_rng(seed))
    return to_rowwise(c, seed)
