"""Sparse-step cases on hot rows whose summed gradients are exact in float32, and the exact bar they are judged by.
CPU only.

Every sparse step sums a row's contributions with float32 red.add / atomicAdd in no fixed order, and step_bar.py's bar
allows for that with n 2^-24 sum |contribution| per element of a row with n contributions.  On a hot row (a Zipf(1.05)
batch of 65 536 triplets gives one user 7 000 lookups) that term is larger than any one contribution: a kernel that loses
one staged contribution, or applies one twice, passes it (test_hot_rows_cpu.py records the ratio).

The cases here make the order irrelevant.  Tables sit on a dyadic grid and every per-lookup contribution is an exact
dyadic number; as long as each element's sum of |contribution| stays below 2^24 units of the finest grid (exact_bound),
every partial sum of every order is exact, so each row's summed gradient G is exact in float32.  The exact bar is then
step_bar's (or momentum_bar's / rowwise_bar's) with the gradient error bound E set to 0: SGD, momentum and Nesterov
updates of such a G are exact too (exact_bound checks every product and sum of them), and must be bit-identical.

  BPR   user rows random on the 2^-4 grid in the first D/2 columns, zero in the rest; every item row shares one grid
        vector in its first D/2 columns and is random in the rest; biases 0.  Then u.p = u.n exactly, x = 0,
        sigmoid(-0) = 1/2 and with c_loss = B every triplet's g = -1/2 (batch sizes with B * float32(1/B) == 1 only).
  UCML  step_bar.dyadic_pair's grid: every score and hinge value is exact, so is the hinge flag; c_loss = 1.
  GMF   user rows zero in their second half, item rows zero in their first, biases 0: z = 0, g = +-1/2 at c_loss = B,
        and w's gradient is an exact zero.
  WRMF  plain (a = 3, b = 0.5): rows on the 2^-2 grid within +-1/4, biases on 2^-4 within +-1/2, so pred is a small
        multiple of 2^-4; with use_sigmoid: GMF's zero halves, pred = sigmoid(0) = 1/2.
Every case has c_l2 = 0, lr 2^-4, momentum 1/2 and dyadic initial slots.

Id patterns, each mixed with a uniform background so that rows seen once stay in the batch:
  zipf       Zipf(1.05) ranks relabelled by a permutation of the rows (bench.py's generator);
  one_row    the hot triplets share one user, their items come from a set of 1-3 rows, as positive and as negative;
  edge_rows  the hot ids are 0 and rows - 1;
  cluster    distinct ids whose home slot in the batch index fills the last slots of the table, so that linear probing
             runs past the last slot and wraps to slot 0; some of them repeat (staged rows), some appear once."""
import zlib

import numpy as np

import momentum_bar as MB
import rowwise_bar as RB
import step_bar as S
from oracle import openrec_oracle as O

LR, MOMENTUM = 2.0 ** -4, 0.5
ZIPF_A = 1.05
OPTS = (O.OPT_SGD, O.OPT_ADAGRAD, O.OPT_ADAM_LAZY, O.OPT_ADAM_DENSE, RB.OPT_ROWWISE_ADAGRAD, MB.OPT_MOMENTUM,
        MB.OPT_NESTEROV)
EXACT_OPTS = (O.OPT_SGD, MB.OPT_MOMENTUM, MB.OPT_NESTEROV)    # bit-identical updates
PATTERNS = ("zipf", "one_row", "edge_rows", "cluster")
KINDS = ("bpr", "ucml", "gmf", "wrmf", "wrmf_sig")
CLUSTER_SPAN = 256     # the cluster's ids home into the last CLUSTER_SPAN slots of the index table
LIMIT = 2 ** 24


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def batch_exact(B):
    """BPR's g = -(c_loss * float32(1 / B)) / 2 and GMF's c_loss (s - label) float32(1 / B) are exactly -1/2 and +-1/2 at
    c_loss = B only where float32 rounding gives B float32(1/B) == 1 and (B/2) float32(1/B) == 1/2."""
    f = np.float32
    inv = f(1.0) / f(B)
    return bool(f(B) * inv == f(1.0) and f(f(B) * f(0.5)) * inv == f(0.5))


def tail_batch():
    """The largest batch below 64 that is not a multiple of 8 (a partial CTA) and satisfies batch_exact."""
    return max(B for B in range(1, 64) if B % 8 and batch_exact(B))


# ---- the batch index's hash (orx_common.cuh orx_hash32, orx_ctx.cu orx_hash_shape) ------------------------------------
def hash_shape(lookups):
    """-> (capacity, lg): the least power of two >= 1024 that holds 4 lookups, and its log2.  An index is sized for the
    handle's batch capacity: `lookups` = B on the user side, 2 B on the item side of a step of B samples."""
    cap = 1024
    while cap < 4 * lookups:
        cap <<= 1
    return cap, cap.bit_length() - 1


def home_slot(ids, lg):
    return ((np.asarray(ids, np.uint64) * np.uint64(2654435769)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - lg)


def wrapped(ids, lookups):
    """True when linear probing of the distinct ids (the set of occupied slots does not depend on the order of the
    inserts) stores some id in a slot below its home: a probe chain ran past the last slot and wrapped to slot 0."""
    cap, lg = hash_shape(lookups)
    taken = np.zeros(cap, bool)
    wrap = False
    for x in np.unique(ids):
        h = int(home_slot(x, lg))
        s = h
        while taken[s]:
            s = (s + 1) % cap
        taken[s] = True
        wrap |= s < h
    return wrap


def cluster_ids(rows, lookups, rng, n=None):
    """Distinct ids < rows whose home slots lie in the last CLUSTER_SPAN slots of the index for `lookups`: more of them
    than the span holds, so their chains wrap."""
    cap, lg = hash_shape(lookups)
    cand = np.flatnonzero(home_slot(np.arange(rows), lg) >= cap - CLUSTER_SPAN)
    n = n or CLUSTER_SPAN + CLUSTER_SPAN // 2
    assert len(cand) >= n, f"{rows} rows hold only {len(cand)} ids homing into the last {CLUSTER_SPAN} slots"
    return rng.permutation(cand)[:n]


# ---- id patterns --------------------------------------------------------------------------------------------------------
def zipf_draw(rows, n, rng, relabel):
    """bench.py's Zipf(1.05) ids: p_k ~ k^-1.05 over the ranks, the ranks relabelled by a permutation of the rows."""
    pk = np.arange(1, rows + 1, dtype=np.float64) ** -ZIPF_A
    pk /= pk.sum()
    return relabel[rng.choice(rows, size=n, p=pk)]


def _hot_mask(rng, B, pattern):
    return rng.random(B) < (0.5 if pattern != "cluster" else 0.75)


def side_ids(pattern, rows, n, lookups, rng, hot_rng, hot=None):
    """n ids over [0, rows) of one lookup side: the pattern's hot ids where `hot` (a mask, default about half of them),
    uniform ids elsewhere.  hot_rng draws what is hot (the relabel, the hot rows), so that two batches built with the
    same hot_rng state share their hot rows."""
    ids = rng.integers(0, rows, n)
    hot = _hot_mask(rng, n, pattern) if hot is None else hot
    k = int(hot.sum())
    if pattern == "zipf":
        ids[hot] = zipf_draw(rows, k, rng, hot_rng.permutation(rows))
    elif pattern == "one_row":
        ids[hot] = rng.choice(hot_rng.permutation(rows)[:hot_rng.integers(1, 4)], k)
    elif pattern == "edge_rows":
        ids[hot] = rng.choice(np.array([0, rows - 1]), k)
    elif pattern == "cluster":
        cl = cluster_ids(rows, lookups, hot_rng)
        half = len(cl) // 2        # the first half once each (owned, unless the background repeats them), the rest staged
        pool = np.r_[cl[:half], rng.choice(cl[half:], max(k - half, 0))][:k]
        ids[hot] = rng.permutation(pool)
    else:
        raise ValueError(pattern)
    return ids.astype(np.int32)


def _rows_for(pattern, B, lookups):
    if pattern == "cluster":
        return 2 * hash_shape(lookups)[0]
    return 100_000 if B > 4096 else max(64, 4 * B)


def pair_ids(pattern, B, rng, hot_rng, cap_B=None):
    """(U, I, (uid, pid, nid)).  one_row: the hot triplets share one user row, and their positives and negatives come from
    the same 1-3 item rows.  cap_B: the batch capacity the index is sized for (default B)."""
    cap_B = cap_B or B
    U, I = _rows_for(pattern, B, cap_B), _rows_for(pattern, B, 2 * cap_B)
    hot = _hot_mask(rng, B, pattern)
    if pattern == "one_row":
        uid = np.where(hot, hot_rng.integers(0, U), rng.integers(0, U, B)).astype(np.int32)
        items = hot_rng.permutation(I)[:hot_rng.integers(1, 4)]
        pid, nid = (np.where(hot, rng.choice(items, B), rng.integers(0, I, B)).astype(np.int32) for _ in range(2))
        return U, I, (uid, pid, nid)
    uid = side_ids(pattern, U, B, cap_B, rng, hot_rng, hot)
    items = side_ids(pattern, I, 2 * B, 2 * cap_B, rng, hot_rng, np.r_[hot, hot])
    return U, I, (uid, items[:B], items[B:])


def point_ids(pattern, B, rng, hot_rng, cap_B=None):
    cap_B = cap_B or B
    U, I = _rows_for(pattern, B, cap_B), _rows_for(pattern, B, 2 * cap_B)
    hot = _hot_mask(rng, B, pattern)
    if pattern == "one_row":
        uid = np.where(hot, hot_rng.integers(0, U), rng.integers(0, U, B)).astype(np.int32)
        iid = np.where(hot, rng.choice(hot_rng.permutation(I)[:hot_rng.integers(1, 4)], B),
                       rng.integers(0, I, B)).astype(np.int32)
        return U, I, (uid, iid)
    return U, I, (side_ids(pattern, U, B, cap_B, rng, hot_rng, hot), side_ids(pattern, I, B, 2 * cap_B, rng, hot_rng, hot))


# ---- tables ---------------------------------------------------------------------------------------------------------------
def grid(rng, shape, lim=0.5, q=2.0 ** -4):
    return np.round(rng.uniform(-lim, lim, shape) / q) * q


def _tables(kind, D, U, I, rng):
    h = D // 2
    user, item, bias = np.zeros((U, D)), np.zeros((I, D)), np.zeros((I, 1))
    if kind == "bpr":
        user[:, :h] = grid(rng, (U, h))
        item[:, :h] = grid(rng, (1, h))
        item[:, h:] = grid(rng, (I, D - h))
        return [user, item, bias]
    if kind == "ucml":
        return [grid(rng, (U, D)), grid(rng, (I, D)), grid(rng, (I, 1), 1.0, 2.0 ** -8)]
    if kind == "wrmf":
        return [grid(rng, (U, D), 0.3, 0.25), grid(rng, (I, D), 0.3, 0.25), grid(rng, (I, 1), 0.5)]
    user[:, :h] = grid(rng, (U, h))        # gmf, wrmf_sig: u * i = 0 in every column
    item[:, h:] = grid(rng, (I, D - h))
    tabs = [user, item, bias]
    return tabs + [grid(rng, (1, D), 1.0)] if kind == "gmf" else tabs


def set_slots(c, rng):
    """Dyadic initial slots: Adagrad accumulators 1/8 (one per row of the user / item tables under ROWWISE), Adam m = 0
    (Keras's start) and v on the 2^-10 grid within (0, 1/4], momentum slots on 2^-8 within +-1/16.  Adam's m starts at 0
    because beta1 m + (1 - beta1) G may cancel, and the exact bar has no gradient term to cover the rounding of a
    cancelling blend on the zero halves of BPR / GMF rows (their values are 0, so their ulps are tiny)."""
    for n in c.names:
        t = c.tabs[n]
        if c.opt == O.OPT_SGD:
            c.slots[n] = (None, None)
        elif c.opt == O.OPT_ADAGRAD or (c.opt == RB.OPT_ROWWISE_ADAGRAD and not (n in RB.TABLES and c.D > 1)):
            c.slots[n] = (np.full_like(t, 0.125), None)
        elif c.opt == RB.OPT_ROWWISE_ADAGRAD:
            c.slots[n] = (np.full(len(t), 0.125), None)
        elif c.opt in MB.KINDS:
            c.slots[n] = (grid(rng, t.shape, 1 / 16, 2.0 ** -8), None)
        else:
            c.slots[n] = (np.zeros_like(t), np.maximum(np.abs(grid(rng, t.shape, 0.25, 2.0 ** -10)), 2.0 ** -10))
    return c


def make_case(kind, opt, D, B, pattern, seed, hot_seed=None, cap_B=None):
    """The exact Case of one (kind, opt, D, B, pattern).  hot_seed (default seed) draws the hot rows: two cases with the
    same hot_seed and different seeds share them."""
    rng = np.random.default_rng(seed)
    hot_rng = np.random.default_rng(seed if hot_seed is None else hot_seed)
    U, I, ids = (pair_ids if kind in S.PAIR_KINDS else point_ids)(pattern, B, rng, hot_rng, cap_B)
    return case_of(kind, opt, _tables(kind, D, U, I, rng), ids, rng)


def case_of(kind, opt, tabs, ids, rng):
    """The exact Case of a kind's tables (_tables) and a batch, with dyadic slots drawn from rng."""
    pair = kind in S.PAIR_KINDS
    B = len(ids[0])
    if kind in ("bpr", "gmf"):
        assert batch_exact(B), f"B = {B}: B * float32(1/B) is not 1 in float32"
        consts = dict(c_loss=float(B), c_l2=0.0)
    else:
        consts = dict(c_loss=1.0, c_l2=0.0)
    label = None if pair else (rng.random(B) < 0.4).astype(np.float32)
    sgd_opt = O.OPT_SGD if opt in MB.KINDS else O.OPT_ADAGRAD if opt == RB.OPT_ROWWISE_ADAGRAD else opt
    c = S.Case(kind[:4], sgd_opt, tabs, ids, label, lr=LR, sig=kind == "wrmf_sig", beta1=0.9, **consts)
    c.opt = opt
    if opt in MB.KINDS:
        c.P["beta1"] = MOMENTUM          # momentum_bar reads the momentum from beta1
    return set_slots(c, rng)


# ---- the exactness proof --------------------------------------------------------------------------------------------------
def _grid_exp(a):
    """The finest grid 2^-k all of a's values lie on (float64 scaling by 2^k is exact)."""
    a = np.abs(np.asarray(a, np.float64))
    m, e = np.frexp(a[a > 0])
    q = (m * 2.0 ** 53).astype(np.int64)           # the 53-bit mantissa: its lowest set bit is the value's grid
    return int((e - 53 + np.log2(q & -q).astype(np.int64)).min())


def _f32_exact(*arrs):
    return all(np.array_equal(x, S.f32(x)) for x in arrs)


def exact_bound(case):
    """-> {name: (e, units, exact_update)}: e the exponent of the finest grid of all the table's contributions, units the
    largest per-element sum of |contribution| in units of 2^e (< 2^24: every order of every partial sum is exact), and
    exact_update whether every product and sum of the SGD, momentum and Nesterov updates of the rows by their G
    (var - lr G, a1 = m a - lr G, var + a1, var + m a1 - lr G) is exact in float32."""
    st = case.state()
    _, rows = S.lookups(case, st)
    out = {}
    for name in case.names:
        idx, val = rows[name][:2]
        e = _grid_exp(val) if np.any(val) else 0
        uniq, inv = O.unique_first_occurrence(idx)
        mag = np.zeros((len(uniq), val.shape[1]))
        np.add.at(mag, inv, np.abs(val))
        G = np.zeros_like(mag)
        np.add.at(G, inv, val)
        units = float(mag.max() / 2.0 ** e) if mag.size else 0.0
        var = st[name][0][uniq]
        a = case.slots[name][0][uniq] if case.opt in MB.KINDS else grid(np.random.default_rng(0), var.shape, 1 / 16,
                                                                           2.0 ** -8)
        lg, m = LR * G, MOMENTUM
        a1 = m * a - lg
        ok = _f32_exact(G, lg, var - lg, m * a, a1, var + a1, m * a1, m * a1 - lg, var + (m * a1 - lg))
        out[name] = (e, units, ok)
    return out


def assert_exact(case):
    for name, (e, units, ok) in exact_bound(case).items():
        assert units < LIMIT and ok, f"{case}: {name} sums {units:.4g} units of 2^{e} (limit 2^24), updates exact: {ok}"


# ---- the exact bar ----------------------------------------------------------------------------------------------------------
class ExactBar(S.Bar):
    """step_bar.Bar, momentum_bar.MomBar or rowwise_bar.RowBar (by the case's optimizer) with every row's gradient error
    bound E = 0: a few float32 ulps and the MUFU divide only.  SGD / momentum / Nesterov tolerances are moot: those
    updates are compared bit for bit (exact_ref)."""

    def __init__(self, case):
        self.case = case
        st = case.state()
        _, rows = S.lookups(case, st)
        P, stp = S._opt_consts(case, None)
        self.ref, self.tol = {}, {}
        for name in case.names:
            idx, G, E = S.dedup(*rows[name])
            E = np.zeros_like(E)
            if case.opt in MB.KINDS:
                r = MB.update_bar(case.opt, case.lr, MB.momentum_of(case), st[name], idx, G, E)
            elif case.opt == RB.OPT_ROWWISE_ADAGRAD and name in RB.TABLES and case.D > 1:
                r = RB.row_update_bar(case.lr, P["eps"], st[name], idx, G, E)
            else:
                kind = O.OPT_ADAGRAD if case.opt == RB.OPT_ROWWISE_ADAGRAD else case.opt
                r = S.update_bar(kind, case.lr, st[name], idx, G, E, P, stp)
            self.ref[name], self.tol[name] = r

    def exact(self, got, what=""):
        """Bit-identity (as values) of every table and slot with the float64 reference (SGD, momentum, Nesterov)."""
        for name in self.case.names:
            for j, (g, r) in enumerate(zip(got[name], self.ref[name])):
                if r is None:
                    continue
                g = np.asarray(g, np.float64).reshape(r.shape)
                bad = np.flatnonzero((g != r).any(1) if r.ndim == 2 else g != r)
                assert not len(bad), f"{what} {self.case}: {name}/{('var', 's0', 's1')[j]} differs in rows {bad[:8]}"

    def judge(self, got, what=""):
        if self.case.opt in EXACT_OPTS:
            self.exact(got, what)
        else:
            self.check(got, what)


# ---- steps from per-lookup rows: the oracle (float64), the float32 emulation and the mutants ----------------------------
def apply_rows(case, st, rows):
    """The optimizer of the case on the per-lookup rows {name: (idx, val, ...)} from state st (arrays of one dtype, the
    arithmetic's), rows summed in the given order.  -> {name: (var, s0, s1)} as float64."""
    P, stp = S._opt_consts(case, None)
    new = {}
    for name in case.names:
        idx, val = rows[name][0], rows[name][1].reshape(len(rows[name][0]), -1)
        var, s0, s1 = (None if x is None else x.copy() for x in st[name])
        if case.opt in MB.KINDS:
            uniq, g = O.dedup(idx, val)
            if var.dtype == np.float32:
                var, s0 = (x.astype(np.float32) for x in MB.f32_update(var, s0, uniq, g, case.lr,
                                                                       MB.momentum_of(case),
                                                                       case.opt == MB.OPT_NESTEROV))
            else:
                MB._update(var, s0, uniq, g, case.lr, MB.momentum_of(case), case.opt == MB.OPT_NESTEROV)
        elif case.opt == RB.OPT_ROWWISE_ADAGRAD:
            if name in RB.TABLES and case.D > 1:
                RB.adagrad_rowwise_sparse(var, s0, idx, val, case.lr, P["eps"])
            else:
                O.adagrad_sparse(var, s0, idx, val, case.lr, P["eps"])
        else:
            O.apply_sparse(case.opt, var, s0, s1, idx, val, stp, case.lr, **P)
        new[name] = tuple(None if x is None else x.astype(np.float64) for x in (var, s0, s1))
    return new


def oracle_step(case):
    st = case.state()
    return apply_rows(case, st, S.lookups(case, st)[1])


def f32_step(case, rng=None):
    """The step in float32: per-lookup rows computed in float32, summed per row in a random order when rng is given."""
    st = case.state(np.float32)
    _, rows = S.lookups(case, st, np.float32)
    if rng is not None:
        rows = {n: tuple(x[p] for x in r) for n, r in rows.items()
                for p in [rng.permutation(len(r[0]))]}
    return apply_rows(case, st, rows)


MUTANTS = ("lose_hot", "double_hot", "neighbour_staged", "bias_one_side")


def _counts(idx):
    uniq, cnt = np.unique(idx, return_counts=True)
    return uniq, cnt


def hottest(case, rows, names=("user", "item")):
    """-> (name, row): the row of the tables `names` with the most lookups whose contributions are not all zero."""
    best = None
    for name in names:
        idx, val = rows[name][:2]
        live = np.any(val != 0, 1)
        uniq, cnt = _counts(idx[live])
        if len(cnt) and (best is None or cnt.max() > best[0]):
            best = (cnt.max(), name, uniq[cnt.argmax()])
    return best[1], best[2]


def mutant_rows(case, mutant, names=("user", "item")):
    """The per-lookup rows (float64) of a mutant of the staging sum, on the hottest row of the tables `names`."""
    st = case.state()
    _, rows = S.lookups(case, st)
    rows = {n: [np.array(x) for x in r] for n, r in rows.items()}
    if mutant == "bias_one_side":          # the hottest positive item's bias loses its contributions as a positive
        idx, val = rows["bias"][:2]
        B = case.B
        uniq, cnt = _counts(idx[:B][val[:B, 0] != 0])
        drop = np.zeros(len(idx), bool)
        drop[:B] = idx[:B] == uniq[cnt.argmax()]
        rows["bias"] = [x[~drop] for x in rows["bias"]]
        return rows
    name, r = hottest(case, rows, names)
    idx, val = rows[name][:2]
    k = np.flatnonzero((idx == r) & np.any(val != 0, 1))[-1]
    if mutant == "lose_hot":
        rows[name] = [np.delete(x, k, 0) for x in rows[name]]
    elif mutant == "double_hot":
        rows[name] = [np.concatenate([x, x[k:k + 1]]) for x in rows[name]]
    elif mutant == "neighbour_staged":     # the contribution lands on the next staged row of the table
        uniq, cnt = _counts(idx)
        staged = uniq[cnt > 1]
        rows[name][0][k] = staged[(np.searchsorted(staged, r) + 1) % len(staged)]
    else:
        raise ValueError(mutant)
    return rows


def mutant_step(case, mutant, names=("user", "item")):
    return apply_rows(case, case.state(), mutant_rows(case, mutant, names))


def staged_rows(case):
    """out4[3] of a step: the rows the batch index stages -- every distinct row of a side under dense Adam, else the rows
    referenced more than once (user side, then items over positives and negatives)."""
    sides = (case.ids[0], np.concatenate(case.ids[1:])) if case.kind in S.PAIR_KINDS else case.ids
    n = 0
    for ids in sides:
        cnt = np.unique(ids, return_counts=True)[1]
        n += len(cnt) if case.opt == O.OPT_ADAM_DENSE else int((cnt > 1).sum())
    return n


def loss_l2(case):
    """(loss, l2) of out4: the forward pass of the pre-step tables in float64."""
    t = {n: case.tabs[n] for n in case.names}
    if case.kind == "bpr":
        return O.bpr_forward(t["user"], t["item"], t["bias"], *case.ids)
    if case.kind == "ucml":
        return O.ucml_forward(t["user"], t["item"], t["bias"], *case.ids, case.P["margin"])
    if case.kind == "gmf":
        return O.gmf_forward(t["user"], t["item"], t["bias"], t["w"].reshape(-1, 1), *case.ids,
                             case.label.astype(np.float64))
    return O.wrmf_forward(t["user"], t["item"], t["bias"], *case.ids, case.label.astype(np.float64), case.P["a"],
                          case.P["b"], case.P["sig"])


# ---- the GPU grid -----------------------------------------------------------------------------------------------------------
SPECIAL_D, OTHER_D = (32, 64, 128, 256), (12, 260)
DIMS = SPECIAL_D + OTHER_D


def pair_specs():
    """(kind, opt, D, B, pattern, entry) of tests/test_gpu_hot_rows.py's pairwise steps.  entry: "step", "host"
    (orx_pairwise_step_host), "prefetch" (two consecutive prefetched steps whose batches share their hot rows)."""
    tail = tail_batch()
    out = [(k, o, D, 1024, "zipf", e) for k in S.PAIR_KINDS for o in OPTS for D in DIMS for e in ("step", "prefetch")]
    out += [("bpr", O.OPT_ADAGRAD, 128, 65536, "zipf", "step"), ("bpr", MB.OPT_MOMENTUM, 128, 65536, "one_row", "step")]
    j = 0
    for k in S.PAIR_KINDS:
        sizes = (1, tail, 4096) + (() if k == "bpr" else (203,))
        for p in PATTERNS:
            for B in sizes:
                for D in (128, 12):
                    out.append((k, OPTS[j % len(OPTS)], D, B, p, "step"))
                    j += 1
        out += [(k, o, D, 4096, "zipf", "host") for o in (O.OPT_ADAGRAD, MB.OPT_MOMENTUM) for D in (128, 12)]
    return out


def point_specs():
    tail = tail_batch()
    out = [(k, o, D, 1024, "zipf", "step") for k in ("gmf", "wrmf", "wrmf_sig") for o in OPTS for D in DIMS]
    out += [("gmf", O.OPT_ADAGRAD, 128, 65536, "zipf", "step")]
    j = 0
    for k in ("gmf", "wrmf", "wrmf_sig"):
        sizes = (1, tail, 4096) + (() if k == "gmf" else (237,))
        for p in PATTERNS:
            for B in sizes:
                for D in (128, 12):
                    out.append((k, OPTS[j % len(OPTS)], D, B, p, "step"))
                    j += 1
    return out


def build(spec, k=0):
    """The Case of one spec; k = 1: the second batch of a prefetched pair (its own tables, the same hot rows)."""
    kind, opt, D, B, pattern, _ = spec
    seed = seed_of("hot", *spec)
    return make_case(kind, opt, D, B, pattern, seed + k, hot_seed=seed)
