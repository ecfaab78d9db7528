"""The update bar of the sparse training steps, the cases it judges and the oracle mutants it must reject.  CPU only.

A step is judged by its per-element change Delta = new - old of every table and every optimizer slot, against the
float64 oracle's change from the same float32 start.  The older bar (atol 1e-5, rtol 1e-5 on the values) cannot see
the loss gradient of the mean-reduced models: BPR and GMF scale it by c_loss / B, and the L2 term and the absolute
tolerance hide a 10 % error in it.  The tolerance of one element is the sum of three terms:

  ULP   K_ULP float32 ulps of max(|old|, |new|).  The step rounds each updated value (and Adam's two-term m / v blends)
        to float32 once or twice; K_ULP leaves the float32 oracle at <= 1/4 of the bar for that rounding alone.
  MUFU  R_MUFU * |Delta|.  Adagrad and Adam divide by sqrt(s) + eps with sqrt.approx / rcp.approx (relative error
        ~2^-22 each, orx_common.cuh), and the host rounds Adam's lr_t to float32.
  GRAD  How far the oracle's own update moves when the row's summed gradient G moves by its float32 error bound E:
        max over +-E of |update(G +- E) - update(G)|, per element of the variable and of every slot.  E is the sum over
        the row's contributions of
          - the error of the per-sample loss gradient g: 2^-22 (|g| + g_abs), where g_abs is the size of g's absolute
            rounding floor (BPR / GMF: c_loss / B, a sigmoid minus a label; WRMF: 2 c_loss wgt (|label| + |pred|));
            plus |dg/dscore| times the float32 error bound of the score's dot product, (D + 4) 2^-24 times the sum of
            the magnitudes of its terms;
          - the rounding of the contribution itself, 2^-22 (|g| M + |c_l2 w|), M the magnitude of its multiplier
            before cancellation (BPR's user row: |p| + |n|, not |p - n|);
        plus n 2^-24 times the sum of the contribution magnitudes (the order of the red.add / staging sum of a row
        with n contributions).  A staged row whose contributions cancel so has a bar sized by its contributions, not
        by its near-zero Delta.  Through update() the term follows the optimizer: Adagrad's 1 / sqrt(acc), Adam's
        sign-like response near G = 0, the slots' G and G^2.

An element whose oracle update is exactly the identity with a zero GRAD term (a row whose every contribution is an
exact zero under SGD / Adagrad, an untouched row of dense Adam with m = 0) has tolerance 0: it must be bit-identical.

A UCML triplet's hinge flag and a BPR triplet's clamp flag are exact: the cases keep random triplets off the kinks and
place the tie triplets on a dyadic grid where every score is exact in float32 (dyadic_*).
"""
import numpy as np

from oracle import openrec_oracle as O

K_ULP = 8
R_MUFU = 2.0 ** -20
U22, U24 = 2.0 ** -22, 2.0 ** -24
PAIR_KINDS, POINT_KINDS = ("bpr", "ucml"), ("gmf", "wrmf")
OPT_LR = {0: 0.05, 1: 0.05, 2: 0.01, 3: 0.01}
DEFAULTS = dict(c_loss=1.0, c_l2=1.0, margin=0.5, eps=1e-7, beta1=0.9, beta2=0.999)
ARM_D = dict(c_loss=1.0, c_l2=1.0, margin=1.25, eps=1e-2, beta1=0.5, beta2=0.75)   # arm (d), run at step 3


def f32(a):
    """float64 copy of the float32 rounding of a."""
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def init_slots(opt, a, init="nontrivial"):
    """(s0, s1) of one table.  "nontrivial": Adagrad 0.1, Adam m = |a| / 100, v = a^2 / 50 + 1e-4 (the older suites');
    "keras": Keras's initial state, Adagrad 0.1, Adam m = v = 0."""
    if opt == O.OPT_SGD:
        return None, None
    if opt == O.OPT_ADAGRAD:
        return f32(np.full_like(a, 0.1)), None
    if init == "keras":
        return np.zeros_like(a), np.zeros_like(a)
    return f32(np.abs(a) * 0.01), f32(a * a * 0.02 + 1e-4)


class Case:
    """One step: float32-valued tables (float64 arrays), their slots, the batch and the step's constants.  names:
    user, item, bias (and w, [1, D], for GMF)."""

    def __init__(self, kind, opt, tabs, ids, label=None, *, step=1, init="nontrivial", lr=None, a=None, b=None,
                 sig=False, **consts):
        self.kind, self.opt, self.step, self.init = kind, opt, step, init
        # the C-ABI takes lr, eps, beta1 / beta2, margin, c_loss and c_l2 as float32: the oracle runs on those values
        # (0.999 is 1 - 9.9999e-4 in float32, which moves Adam's 1 - beta2^t by 1.3e-5 relative)
        self.lr = float(np.float32(OPT_LR[opt] if lr is None else lr))
        self.P = {k: float(np.float32(v)) for k, v in {**DEFAULTS, **consts}.items()}
        self.names = ("user", "item", "bias", "w")[:4 if kind == "gmf" else 3]
        self.tabs = {n: f32(t) for n, t in zip(self.names, tabs)}
        self.slots = {n: init_slots(opt, self.tabs[n], init) for n in self.names}
        self.ids = tuple(np.asarray(x, np.int32) for x in ids)
        self.label = None if label is None else np.asarray(label, np.float32)
        if kind == "wrmf":
            self.P.update(a=3.0 if a is None else a, b=0.5 if b is None else b, sig=sig)
        self.D = self.tabs["user"].shape[1]
        self.B = len(self.ids[0])

    def __repr__(self):
        return f"Case({self.kind} opt{self.opt} D={self.D} B={self.B} step {self.step} {self.init} {self.P})"

    def state(self, dt=np.float64):
        return {n: tuple(None if x is None else x.astype(dt) for x in (self.tabs[n], *self.slots[n]))
                for n in self.names}


# ---- per-lookup gradients with their float32 error bounds, and the mutants ------------------------------------------
MUTANTS = ("g_x0.9", "neighbour_g", "no_bias", "lost_dup", "tie_flip", "no_clamp", "margin_0.5", "beta_swap",
           "beta_default", "eps_default", "adam_step1", "neighbour_label", "no_sig_factor")


def _dup_last(ids):
    """Mask of each repeated id's last occurrence."""
    last = np.zeros(len(ids), bool)
    seen = {}
    for j, x in enumerate(ids):
        seen.setdefault(int(x), []).append(j)
    for js in seen.values():
        if len(js) > 1:
            last[js[-1]] = True
    return last


def lookups(case, st, dt=np.float64, mutant=None):
    """-> (g [B], {name: (idx, val [n, D'], err [n, D'], mag [n, D'])}): every lookup's gradient row of
    c_loss * loss + c_l2 * l2 (as TF's IndexedSlices, not deduplicated), its error bound and its magnitude, computed in
    dt from the state st (name -> (var, s0, s1)).  `mutant` is one of MUTANTS or None."""
    dt = np.dtype(dt)
    P, T = case.P, dt.type
    c, c2 = T(P["c_loss"]), T(P["c_l2"])
    B, D = case.B, case.D
    var = {n: st[n][0] for n in case.names}
    out = {}
    if case.kind in PAIR_KINDS:
        uid, pid, nid = case.ids
        u, p, n = var["user"][uid], var["item"][pid], var["item"][nid]
        bp, bn = var["bias"][pid, 0], var["bias"][nid, 0]
        if mutant == "no_bias":
            bp, bn = bp * 0, bn * 0
        if case.kind == "bpr":
            x = ((u * p).sum(1, dtype=dt) + bp) - ((u * n).sum(1, dtype=dt) + bn)
            on = (x > T(-30)) if mutant == "tie_flip" else (x >= T(-30))
            y = x if mutant == "no_clamp" else np.maximum(x, T(-30))
            if mutant == "no_clamp":
                on = np.ones(B, bool)
            s = O.sigmoid(-y)
            g = -(c / T(B)) * s * on
            gp = (c / T(B)) * s * (1 - s) * on
            gross = np.abs(u * p).sum(1) + np.abs(u * n).sum(1) + np.abs(bp) + np.abs(bn)
            g_abs = (c / T(B)) * on
        else:
            margin = T(0.5 if mutant == "margin_0.5" else P["margin"])
            dp, dn = ((u - p) ** 2).sum(1, dtype=dt), ((u - n) ** 2).sum(1, dtype=dt)
            h = margin - ((-dp + bp) - (-dn + bn))
            g = c * ((h > 0) if mutant == "tie_flip" else (h >= 0)).astype(dt)
            gp = gross = g_abs = np.zeros(B, dt)   # the hinge flag is exact off the kink (see the module docstring)
        g = _mutate_g(g, mutant)
        dg = U22 * (np.abs(g) + g_abs) + gp * gross * (D + 4) * U24
        g1 = g[:, None]
        if case.kind == "bpr":
            parts = {"user": [(uid, g1 * (p - n), np.abs(p) + np.abs(n), u)],
                     "item": [(pid, g1 * u, np.abs(u), p), (nid, -g1 * u, np.abs(u), n)],
                     "bias": [(pid, g1, 1, None), (nid, -g1, 1, None)]}
        else:
            parts = {"user": [(uid, 2 * g1 * (n - p), 2 * (np.abs(n) + np.abs(p)), u)],
                     "item": [(pid, -2 * g1 * (u - p), 2 * (np.abs(u) + np.abs(p)), p),
                              (nid, 2 * g1 * (u - n), 2 * (np.abs(u) + np.abs(n)), n)],
                     "bias": [(pid, -g1, 1, None), (nid, g1, 1, None)]}
    else:
        uid, iid = case.ids
        label = case.label.astype(dt)
        if mutant == "neighbour_label":
            label = np.roll(label, 1)
        u, i, bb = var["user"][uid], var["item"][iid], var["bias"][iid, 0]
        if mutant == "no_bias":
            bb = bb * 0
        if case.kind == "gmf":
            w = var["w"].reshape(1, -1)
            z = (u * i * w).sum(1, dtype=dt) + bb
            s = O.sigmoid(z)
            g = c * (s - label) / T(B)
            gp = c * s * (1 - s) / T(B)
            gross = np.abs(u * i * w).sum(1) + np.abs(bb)
            g_abs = np.full(B, c / T(B), dt)
        else:
            sig = P["sig"]
            pred = (u * i).sum(1, dtype=dt) + bb
            gross = np.abs(u * i).sum(1) + np.abs(bb)
            if sig:
                pred = O.sigmoid(pred)
            wgt = T(P["a"] - P["b"]) * label + T(P["b"])
            g = c * T(-2) * wgt * (label - pred)
            gp = 2 * c * wgt
            g_abs = 2 * c * wgt * (np.abs(label) + np.abs(pred))
            if sig:
                q = pred * (1 - pred)
                if mutant != "no_sig_factor":
                    g = g * q
                gp = gp * q * (q + np.abs(label - pred) * np.abs(1 - 2 * pred))
                g_abs = g_abs * pred
        g = _mutate_g(g.astype(dt), mutant)
        dg = U22 * (np.abs(g) + g_abs) + gp * gross * (D + 4) * U24
        g1 = g[:, None]
        parts = {"user": [(uid, g1 * (w * i) if case.kind == "gmf" else g1 * i,
                           np.abs(w * i) if case.kind == "gmf" else np.abs(i), u)],
                 "item": [(iid, g1 * (w * u) if case.kind == "gmf" else g1 * u,
                           np.abs(w * u) if case.kind == "gmf" else np.abs(u), i)],
                 "bias": [(iid, g1, 1, None)]}
        if case.kind == "gmf":
            parts["w"] = [(np.zeros(B, np.int32), g1 * (u * i), np.abs(u * i), None),
                          (np.zeros(1, np.int32), np.zeros((1, D), dt), 0, var["w"])]
    if mutant == "lost_dup":       # a duplicated user row loses its last contribution
        keep = ~_dup_last(case.ids[0])
        ((ids, val, M, own),) = parts["user"]
        parts["user"] = [(ids[keep], val[keep], M[keep], own[keep])]
    else:
        keep = slice(None)
    for name, lst in parts.items():
        idx, val, err, mag = [], [], [], []
        for ids, v, M, own in lst:
            d = np.zeros((1, 1)) if own is not None and len(ids) == 1 and name == "w" else \
                (dg[keep] if name == "user" else dg)[:, None]
            absg = np.abs(v)
            l2 = np.zeros_like(v) if own is None else c2 * own
            idx.append(ids)
            val.append(v + l2)
            mag.append(absg + np.abs(l2))
            err.append(d * M + U22 * (absg + np.abs(l2)))
        out[name] = tuple(np.concatenate(x) for x in (idx, val, err, mag))
    return g, out


def _mutate_g(g, mutant):
    if mutant == "g_x0.9":
        return g * g.dtype.type(0.9)
    if mutant == "neighbour_g":
        return np.roll(g, 1)
    return g


def _opt_consts(case, mutant):
    P = dict(eps=case.P["eps"], beta1=case.P["beta1"], beta2=case.P["beta2"])
    step = case.step
    if mutant == "beta_swap":
        P["beta1"], P["beta2"] = P["beta2"], P["beta1"]
    elif mutant == "beta_default":
        P["beta1"], P["beta2"] = 0.9, 0.999
    elif mutant == "eps_default":
        P["eps"] = 1e-7
    elif mutant == "adam_step1":
        step = 1
    return P, step


def _apply(opt, lr, old, idx, G, P, step):
    var, s0, s1 = (None if x is None else x.copy() for x in old)
    O.apply_sparse(opt, var, s0, s1, idx, G.reshape(len(idx), -1), step, lr, **P)
    return var, s0, s1


def dedup(idx, val, err, mag):
    """-> (unique rows, G, E): the summed gradient of each row and its error bound (module docstring)."""
    uniq, inv = O.unique_first_occurrence(idx)
    G, E, S = (np.zeros((len(uniq), val.shape[1])) for _ in range(3))
    np.add.at(G, inv, val)
    np.add.at(E, inv, err)
    np.add.at(S, inv, mag)
    cnt = np.bincount(inv, minlength=len(uniq))[:, None]
    return uniq, G, E + cnt * U24 * S


def step(case, dt=np.float64, mutant=None):
    """The oracle's step (or a mutant's) in dt.  -> {name: (var, s0, s1)} after the step (float64 arrays)."""
    st = case.state(dt)
    _, rows = lookups(case, st, dt, mutant)
    P, stp = _opt_consts(case, mutant)
    new = {}
    for name in case.names:
        idx, val = rows[name][:2]
        var, s0, s1 = (None if x is None else x.copy() for x in st[name])
        O.apply_sparse(case.opt, var, s0, s1, idx, val.reshape(len(idx), -1), stp, case.lr, **P)
        new[name] = tuple(None if x is None else x.astype(np.float64) for x in (var, s0, s1))
    return new


def ulp32(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def update_bar(opt, lr, old, idx, G, E, P, step):
    """-> (ref, tol): the oracle's update of the rows idx of one table (old = (var, s0, s1)) by the summed gradients G
    with error bound E, and the tolerance of every element (module docstring)."""
    ref, hi, lo = (_apply(opt, lr, old, idx, X, P, step) for X in (G, G + E, G - E))
    tol = []
    for o, r, h, l in zip(old, ref, hi, lo):
        if o is None:
            tol.append(None)
            continue
        grad = np.maximum(np.abs(h - r), np.abs(l - r))
        delta = np.abs(r - o)
        t = K_ULP * ulp32(np.maximum(np.abs(o), np.abs(r))) + R_MUFU * delta + grad
        tol.append(np.where((delta == 0) & (grad == 0), 0.0, t))
    return ref, tuple(tol)


def ratios(ref, tol, got):
    """-> [max err / tol] per array of (var, s0, s1) (inf where a bit-identical element moved; None: no such slot)."""
    out = []
    for g, r, t in zip(got, ref, tol):
        if t is None:
            out.append(None)
            continue
        err = np.abs(np.asarray(g, np.float64).reshape(r.shape) - r)
        q = np.where(t > 0, err / np.where(t > 0, t, 1), np.where(err > 0, np.inf, 0.0))
        out.append(float(q.max()) if q.size else 0.0)
    return out


class Bar:
    """The float64 oracle's step of a case and the tolerance of every element of every table and slot."""

    def __init__(self, case):
        self.case = case
        st = case.state()
        _, rows = lookups(case, st)
        P, stp = _opt_consts(case, None)
        self.ref, self.tol = {}, {}
        for name in case.names:
            idx, G, E = dedup(*rows[name])
            self.ref[name], self.tol[name] = update_bar(case.opt, case.lr, st[name], idx, G, E, P, stp)

    def ratios(self, got):
        """got: {name: (var, s0, s1)} after the step -> {"name/slot": max err / tol}."""
        out = {}
        for name in self.case.names:
            for j, q in enumerate(ratios(self.ref[name], self.tol[name], got[name])):
                if q is not None:
                    out[f"{name}/{('var', 's0', 's1')[j]}"] = q
        return out

    def worst(self, got):
        r = self.ratios(got)
        k = max(r, key=r.get)
        return r[k], k

    def check(self, got, what=""):
        q, k = self.worst(got)
        assert q <= 1.0, f"{what} {self.case}: {k} err/tol = {q:.3g} (all: {self.ratios(got)})"
        return q


def lookup_bar(case, dt=np.float64):
    """-> {name: (val, tol)} of every lookup's gradient row (the un-fused *_grad outputs, before the L2 term is
    summed into rows): tol is the row's error bound of the module docstring, with a float32 ulp of the value."""
    _, rows = lookups(case, case.state(dt), dt)
    return {n: (v[1], v[2] + 2 * ulp32(v[1])) for n, v in rows.items()}


# ---- case builders ----------------------------------------------------------------------------------------------------
def _pair_ids(rng, U, I, B):
    return (rng.integers(0, U, B), rng.integers(0, I, B), rng.integers(0, I, B))


def random_pair(kind, opt, D, U, I, B, seed, *, scale=None, init="nontrivial", step=1, **consts):
    """Uniform tables at the older suites' scale (BPR 0.05, UCML 0.4), uniform ids with one positive = negative and
    one duplicated user; the negatives of UCML triplets near the hinge's kink (|h| < 1e-3) are redrawn."""
    rng = np.random.default_rng(seed)
    sc = scale or (0.05 if kind == "bpr" else 0.4)
    tabs = [rng.uniform(-sc, sc, s) for s in ((U, D), (I, D), (I, 1))]
    uid, pid, nid = _pair_ids(rng, U, I, B)
    if B >= 4:
        nid[1], uid[2] = pid[1], uid[3]
    for _ in range(50):
        c = Case(kind, opt, tabs, (uid, pid, nid), step=step, init=init, **consts)
        bad = _near_kink(c) if kind == "ucml" else np.zeros(B, bool)
        if not bad.any():
            return c
        nid[bad] = rng.integers(0, I, bad.sum())
    raise AssertionError("could not avoid hinge ties")


def _near_kink(c, tol=1e-3):
    uid, pid, nid = c.ids
    t = c.tabs
    u, p, n = t["user"][uid], t["item"][pid], t["item"][nid]
    h = c.P["margin"] - ((-((u - p) ** 2).sum(1) + t["bias"][pid, 0]) - (-((u - n) ** 2).sum(1) + t["bias"][nid, 0]))
    return (np.abs(h) < tol) | (np.abs(h - c.P["margin"] + 0.5) < tol)   # nor the margin_0.5 mutant


def random_point(kind, opt, D, U, I, B, seed, *, sig=False, init="nontrivial", step=1, **consts):
    """Uniform tables at +-0.3 (and GMF's w), uniform ids, labels 1 with probability 0.4."""
    rng = np.random.default_rng(seed)
    tabs = [rng.uniform(-0.3, 0.3, s) for s in ((U, D), (I, D), (I, 1), (1, D))]
    ids = rng.integers(0, U, B), rng.integers(0, I, B)
    if B >= 4:
        ids[0][2] = ids[0][3]
    label = (rng.random(B) < 0.4).astype(np.float32)
    return Case(kind, opt, tabs[:4 if kind == "gmf" else 3], ids, label, step=step, init=init, sig=sig, **consts)


GRID = 2.0 ** -4     # table entries: multiples of 2^-4, |v| <= 1/2; biases: multiples of 2^-8
BPR_TIES = (-30.0, -30.0 - GRID, -30.0 + GRID, 40.0, -40.0)
UCML_TIES = (0.0, GRID, -GRID, -3.0)
POINT_TIES = {"gmf": (40.0, -40.0), "wrmf": (30.0, -30.0)}


def _grid(rng, shape, lim=0.5, q=GRID):
    return np.round(rng.uniform(-lim, lim, shape) / q) * q


def dyadic_pair(kind, opt, D, B, seed, *, init="nontrivial", **consts):
    """Tie / saturation table.  Every score is exact in float32 (terms are multiples of 2^-8, partial sums < 2^15, so
    under 2^23 units of 2^-8),
    whatever the order or FMA.  The first triplets sit exactly at the targets (BPR_TIES of x, UCML_TIES of h) through
    the bias of a negative item of their own; users are shared between tie triplets (staged rows) and alone (owned).
    Users 0 and 1 only meet clamped / inactive triplets (user 0 twice, user 1 once), as do their triplets' items: at
    c_l2 = 0 every contribution to those rows is an exact zero.  The remaining triplets are random on the grid."""
    rng = np.random.default_rng(seed)
    ties = BPR_TIES if kind == "bpr" else UCML_TIES
    dead = BPR_TIES[4] if kind == "bpr" else UCML_TIES[3]
    targets = [dead, dead, dead] + [t for t in ties for _ in range(4)]
    nt = len(targets)
    U, I = max(8, B // 3), 3 * B + 2 * nt
    user, item, bias = _grid(rng, (U, D)), _grid(rng, (I, D)), _grid(rng, (I, 1), 1.0, 2.0 ** -8)
    uid = rng.integers(2, U, B)
    pid = rng.integers(2 * nt, I, B)
    nid = rng.integers(2 * nt, I, B)
    uid[:3] = (0, 0, 1)
    uid[3:nt:3] = uid[3]                      # a staged user among the tie triplets
    pid[:nt] = np.arange(nt)                  # positives and negatives of the tie triplets: rows of their own
    nid[:nt] = nt + np.arange(nt)
    pid[3:nt:5] = pid[3]                      # ... except one positive shared by several tie triplets (staged)
    user[:2] = _grid(rng, (2, D))
    margin = consts.get("margin", DEFAULTS["margin"])
    for j, t in enumerate(targets):
        u, p, n = user[uid[j]], item[pid[j]], item[nid[j]]
        if kind == "bpr":     # x = (u.p + bp) - (u.n + bn) = t
            bias[nid[j], 0] = (u @ p + bias[pid[j], 0]) - u @ n - t
        else:                 # h = margin - ((-dp + bp) - (-dn + bn)) = t
            dp, dn = ((u - p) ** 2).sum(), ((u - n) ** 2).sum()
            bias[nid[j], 0] = t - margin + (-dp + bias[pid[j], 0]) + dn
    perm = np.r_[np.arange(nt), nt + rng.permutation(B - nt)] if B > nt else np.arange(B)
    c = Case(kind, opt, (user, item, bias), (uid[perm], pid[perm], nid[perm]), init=init, **consts)
    assert np.all(np.abs(c.tabs["bias"]) < 2 ** 14) and np.array_equal(c.tabs["bias"], bias)
    return c


def dyadic_point(kind, opt, D, B, seed, *, sig=None, init="nontrivial", **consts):
    """As dyadic_pair for GMF (z at +-40) and WRMF with use_sigmoid (pred's input at +-30), each target with both labels,
    through the bias of an item of its own; users 0 (twice) and 1 (once) meet only saturated samples.  WRMF's terms u i
    are multiples of 2^-8 as in dyadic_pair; GMF's u i w (w on the 2^-4 grid, |w| <= 1) and so its fitted biases are
    multiples of 2^-12 with partial sums below 2^7: under 2^19 units, still exact in float32."""
    rng = np.random.default_rng(seed)
    targets = [POINT_TIES[kind][0]] * 3 + [t for t in POINT_TIES[kind] for _ in range(4)]
    nt = len(targets)
    U, I = max(8, B // 3), 2 * B + nt
    user, item, bias = _grid(rng, (U, D)), _grid(rng, (I, D)), _grid(rng, (I, 1), 1.0, 2.0 ** -8)
    w = _grid(rng, (1, D), 1.0)
    uid, iid = rng.integers(2, U, B), rng.integers(nt, I, B)
    uid[:3] = (0, 0, 1)
    uid[3:nt:2] = uid[3]
    iid[:nt] = np.arange(nt)
    label = (rng.random(B) < 0.4).astype(np.float32)
    label[:nt] = np.arange(nt) % 2
    label[:3] = 1.0          # users 0 and 1: saturated towards the label (score +40 / +30), g ~ 0 but not exactly 0
    for j, t in enumerate(targets):
        u, i = user[uid[j]], item[iid[j]]
        s = (u * i * w[0]).sum() if kind == "gmf" else (u * i).sum()
        bias[iid[j], 0] = t - s
    perm = np.r_[np.arange(nt), nt + rng.permutation(B - nt)]
    tabs = (user, item, bias, w)[:4 if kind == "gmf" else 3]
    return Case(kind, opt, tabs, (uid[perm], iid[perm]), label[perm], init=init,
                sig=(kind == "wrmf") if sig is None else sig, **consts)


# ---- the arms ---------------------------------------------------------------------------------------------------------
def arm_consts(arm, B):
    """(step, init, consts) of an arm: (a) loss only, (b) amplified, (c) tie / saturation tables, (d) non-default
    optimizer constants and margin at step 3."""
    if arm == "a":
        return 1, "keras", dict(c_loss=1.0, c_l2=0.0)
    if arm == "b":
        return 1, "nontrivial", dict(c_loss=float(B), c_l2=1.0)
    if arm == "c":
        return 1, "nontrivial", dict(c_loss=1.0, c_l2=0.0)
    return 3, "nontrivial", dict(ARM_D)


def pair_case(arm, kind, opt, D, B, seed, U=None, I=None):
    step, init, consts = arm_consts(arm, B)
    if arm == "c":
        return dyadic_pair(kind, opt, D, B, seed, init=init, **consts)
    U, I = U or max(4, B // 2), I or max(6, B)
    return random_pair(kind, opt, D, U, I, B, seed, init=init, step=step, **consts)


def point_case(arm, kind, opt, D, B, seed, U=None, I=None, sig=False):
    step, init, consts = arm_consts(arm, B)
    if arm == "c":
        return dyadic_point(kind, opt, D, B, seed, sig=sig if kind == "wrmf" else None, init=init, **consts)
    U, I = U or max(4, B // 2), I or max(6, B)
    return random_point(kind, opt, D, U, I, B, seed, sig=sig, init=init, step=step, **consts)


# ---- the cases tests/test_gpu_step_updates.py runs ------------------------------------------------------------------
# (arm, kind, opt, D, B, entry).  entry: "step" (orx_pairwise_step / orx_pointwise_step), "prefetch" (two consecutive
# prefetched steps, index sets 1 and 2; the spec's case and the one of seed + 1), "host" (orx_pairwise_step_host).
ARMS = "abcd"
PAIR_TAIL_D, POINT_D = (12, 260, 32, 64, 256), (10, 32, 64, 128, 256)


def pair_specs():
    out = [(arm, k, opt, D, 203, "step") for arm in ARMS for k in PAIR_KINDS for opt in range(4) for D in PAIR_TAIL_D]
    out += [(arm, k, opt, 128, 4096, "step") for arm in ARMS for k in PAIR_KINDS for opt in range(4)]
    out += [(arm, k, opt, D, 237, "prefetch") for arm in "ac" for k in PAIR_KINDS for opt in range(4)
            for D in (12, 32, 64, 128, 256)]
    out += [(arm, k, opt, D, 1000, "host") for arm in "ad" for k in PAIR_KINDS for opt in range(4) for D in (12, 128)]
    return out


def point_specs():
    """kind "wrmf_sig": WRMF with use_sigmoid."""
    return [(arm, k, opt, D, 237, "step") for arm in ARMS for k in ("gmf", "wrmf", "wrmf_sig") for opt in range(4)
            for D in POINT_D]


def spec_seed(*spec):
    import zlib
    return zlib.crc32(repr(spec).encode())


def build(spec, seed_offset=0):
    """The Case of one spec."""
    arm, kind, opt, D, B, _ = spec
    seed = spec_seed(*spec) + seed_offset
    if kind in PAIR_KINDS:
        return pair_case(arm, kind, opt, D, B, seed)
    return point_case(arm, kind[:4], opt, D, B, seed, sig=kind == "wrmf_sig")


def loopback_specs():
    """(world, arm, kind, opt) of the two-rank home-routed sharded step (tests/test_gpu_shard_loopback.py): arms (a) and
    (d), SGD / Adagrad / lazy Adam (the optimizers orx_shard_step has)."""
    return [(2, arm, k, opt) for arm in "ad" for k in PAIR_KINDS for opt in range(3)]


def loopback_case(world, arm, kind, opt, D=128, B=256):
    """The global batch (world * B triplets, rank r's are [r B, (r + 1) B)) of one loopback spec."""
    return pair_case(arm, kind, opt, D, B * world, spec_seed("loopback", world, arm, kind, opt, D))
