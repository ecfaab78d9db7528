"""Every table-indexing kernel on tables past 2^32 elements, and the row-space limits at 2^31 - 1.

The tables follow tests/far_tables.py: a float32 [rows, D] table of 2^32 + 2^29 elements and a little more (19.3 GB at
D = 128; D = 50 takes the generic / scalar paths), filled with a uniform background in [-0.05, 0.05], with planted far
rows from a disjoint range.  Id-driven kernels only ever see low rows and rows at or above 2^32 / D, whose 32-bit
truncated addresses (the row's alias) stay inside the table: a dropped int64 cast reads background values where planted
ones were expected, or writes an alias row no id named -- a wrong value at a known row, never an out-of-bounds access.
Only the full-table sweeps (k_adam_sweep, orx_fill_uniform, orx_rows_scale) cross the mid band, and their checks sample
every band.

The references only ever see the touched rows: they are copied out with index_select and the float64 oracle runs on the
compact problem (touched rows renumbered 0 .. n-1).  One far table set is alive at a time; each case skips, saying so,
when the device has less free memory than it needs plus 2 GB, and frees everything it allocated when it ends."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import dlrm_bags_np as NB
import far_tables as F
from dlrm_shard_np import lookup_bucket_np
from oracle import device_samplers as S
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N
from openrec_b200.sharded import loopback_sum, row_offsets, score_rank_sharded, score_topk_sharded
from test_gpu_kernels import PAIR_OP, POINT_OP, _check_step_dispatch, _staged

pytestmark = pytest.mark.gpu

GB = 1 << 30
DIMS = (128, 50)          # the D = 128 fast paths, and a D that is not a multiple of 4 (generic / scalar paths)
OPTS = {"sgd": (0, 0.05), "adagrad": (1, 0.05), "adam_lazy": (2, 0.01), "adam_dense": (3, 0.01)}
N_SLOTS = {0: 0, 1: 1, 2: 2, 3: 2}
# (background, planted) ranges of the variable and of each optimizer slot
RANGES = {"var": ((-0.05, 0.05), (1.0, 2.0)), 1: [((0.1, 0.2), (0.5, 0.6))],
          2: [((-0.01, 0.01), (0.02, 0.03)), ((1e-4, 2e-4), (3e-4, 4e-4))]}
INT32_MAX = 2 ** 31 - 1


@pytest.fixture(scope="module")
def eng():
    return N.engine()


_HELD = []


def big(t):
    """Registers a case's large tensor; -> t.  The case's teardown frees it."""
    _HELD.append(t)
    return t


@pytest.fixture(autouse=True)
def _release():
    """Every case frees its tables before the next one allocates.  The storage of each registered tensor is released
    explicitly: when an assertion fails, pytest keeps the traceback, whose frames still reference the tables, and the
    cases after it would otherwise find the device full and skip."""
    yield
    torch.cuda.synchronize()
    for t in _HELD:
        t.untyped_storage().resize_(0)
    _HELD.clear()
    gc.collect()
    torch.cuda.empty_cache()


def need(nbytes, what):
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes + 2 * GB:
        pytest.skip(f"{what} needs {(nbytes + 2 * GB) / GB:.1f} GB free on the device, {free / GB:.1f} GB are")


def table_bytes(D, n=1):
    return F.far_rows(D) * D * 4 * n


def idx(a):
    return torch.as_tensor(np.asarray(a, np.int64)).cuda()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def rows_of(t, r):
    """float32 host copy of rows r of t."""
    return t.index_select(0, idx(r)).cpu().numpy()


def plant(t, rows, lo, hi, rng):
    vals = rng.uniform(lo, hi, (len(rows),) + tuple(t.shape[1:])).astype(np.float32)
    t.index_copy_(0, idx(rows), dev(vals))


def close(got, want, what, atol=2e-5, rtol=1e-5):
    np.testing.assert_allclose(np.asarray(got, np.float64), want, atol=atol, rtol=rtol, err_msg=what)


def bits_equal(got, want, what):
    g, w = np.asarray(got), np.asarray(want)
    bad = (g.view(np.int32) != w.view(np.int32)).reshape(len(g), -1).any(1) if g.ndim else g != w
    assert g.shape == w.shape and not np.any(bad), f"{what}: {int(np.sum(bad))} rows differ, first {np.flatnonzero(bad)[:8]}"


def compact(ids, valid, rows):
    """ids renumbered into the compact problem over the sorted rows `valid`; padding stays -1, a bad id becomes
    len(valid) (out of range of the compact tables too)."""
    ids = np.asarray(ids, np.int64)
    ok = (ids >= 0) & (ids < rows)
    out = np.where(ids < 0, -1, len(valid)).astype(np.int64)
    out[ok] = np.searchsorted(valid, ids[ok])
    assert np.array_equal(valid[out[ok]], ids[ok])
    return out


class FarTable:
    """The far table of width D and n_slots optimizer slots of the same shape, background-filled, with mix.far planted
    in the variable and in every slot; .snap() copies the guard rows (and any extra rows) of all of them."""

    def __init__(self, eng, D, mix, n_slots=0, seed=1, opt=None):
        rng = np.random.default_rng(seed)
        self.rows, self.D = F.far_rows(D), D
        self.var = big(torch.empty(self.rows, D, device="cuda"))
        (blo, bhi), (plo, phi) = RANGES["var"]
        eng.fill_uniform(self.var, blo, bhi, seed)
        plant(self.var, mix.far, plo, phi, rng)
        self.slots = []
        for j in range(n_slots):
            (blo, bhi), (plo, phi) = RANGES[1 if opt == 1 else 2][j]
            s = big(torch.empty_like(self.var))
            eng.fill_uniform(s, blo, bhi, seed + 10 + j)
            plant(s, mix.far, plo, phi, rng)
            self.slots.append(s)

    @property
    def all(self):
        return [self.var] + self.slots

    def table(self):
        return N.table(self.var, *self.slots)

    def snap(self, rows):
        return [rows_of(t, rows) for t in self.all]


# ---------------------------------------------------------------------------------------------------------------------
# 1. gathers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", DIMS)
def test_gather(eng, D):
    """orx_gather with int32 and int64 ids, orx_gather_strided into out_ld > D: every row bit-equal to the host copy
    of the touched rows, bad ids zero rows counted in n_bad, the output's other columns untouched."""
    need(table_bytes(D), "a far table")
    m = F.Mix(D, seed=D)
    ft = FarTable(eng, D, m)
    host = rows_of(ft.var, m.valid)
    c = compact(m.ids, m.valid, m.rows)
    want = np.where((c >= 0)[:, None] & (c < len(m.valid))[:, None], host[np.clip(c, 0, len(m.valid) - 1)], 0)
    want = want.astype(np.float32)
    n_bad_want = int(((m.ids < 0) | (m.ids >= m.rows)).sum())
    for dtype in (torch.int32, torch.int64):
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = eng.gather(ft.var, dev(m.ids, dtype), n_bad)
        bits_equal(out.cpu().numpy(), want, f"orx_gather {dtype} D={D}")
        assert n_bad.item() == n_bad_want, (dtype, n_bad.item(), n_bad_want)
    n, F_, col = len(m.ids), 3, 1
    ids2d = np.full((n, F_), 7, np.int32)
    ids2d[:, col] = m.ids
    ld, c0 = 2 * D + 8, 4                      # a 16-byte aligned view: the float4 path at D = 128
    full = torch.full((n, ld), 7.0, device="cuda")
    out2d = full[:, c0:c0 + D]
    n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_ids = dev(ids2d, torch.int32)
    L.check(eng.lib.orx_gather_strided(eng.h, C.c_void_p(ft.var.data_ptr()), ft.rows, D,
                                       C.c_void_p(d_ids.data_ptr() + 4 * col), F_, n, C.c_void_p(out2d.data_ptr()), ld,
                                       C.c_void_p(n_bad.data_ptr()), eng.stream()), "orx_gather_strided")
    got = full.cpu().numpy()
    bits_equal(got[:, c0:c0 + D], want, f"orx_gather_strided D={D}")
    assert (got[:, :c0] == 7).all() and (got[:, c0 + D:] == 7).all()
    assert n_bad.item() == n_bad_want


@pytest.mark.parametrize("mode", [0, 1], ids=["sum", "mean"])
@pytest.mark.parametrize("Lbag", [1, 7, 33])
@pytest.mark.parametrize("D", DIMS)
def test_bag_gather(eng, D, Lbag, mode):
    """orx_bag_gather with the far table between two small ones: pooled rows bit-equal to pool_f32 over the touched
    rows, the exact n_bad."""
    need(table_bytes(D), "a far table")
    m = F.Mix(D, seed=D + Lbag)
    ft = FarTable(eng, D, m, seed=2)
    rng = np.random.default_rng(Lbag)
    small = [dev(rng.uniform(-1, 1, (r, D)).astype(np.float32)) for r in (1000, 77)]
    B = max(-(-len(m.ids) // Lbag), 8)
    far_ids = np.resize(rng.permutation(m.ids), B * Lbag).reshape(B, Lbag)
    far_ids[0] = -1                                        # a bag of padding only: the zero row
    col_off = [0, 2, 2 + Lbag, 2 + Lbag + 3]
    sparse = np.zeros((B, col_off[-1]), np.int64)
    sparse[:, 0:2] = rng.integers(-1, 1001, (B, 2))
    sparse[:, 2:2 + Lbag] = far_ids
    sparse[:, 2 + Lbag:] = rng.integers(-1, 78, (B, 3))
    tabs = [small[0], ft.var, small[1]]
    out = torch.full((B, 3 * D + 4), 7.0, device="cuda")
    n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    eng.bag_gather(tabs, dev(sparse, torch.int32), col_off, mode, out, n_bad)
    host = rows_of(ft.var, m.valid)
    csp = sparse.copy()
    csp[:, 2:2 + Lbag] = compact(far_ids, m.valid, m.rows).reshape(B, Lbag)
    Z, _, bad = NB.pool_f32([small[0].cpu().numpy(), host, small[1].cpu().numpy()], csp, col_off, mode == 1)
    got = out.cpu().numpy()
    bits_equal(got[:, :3 * D], Z.reshape(B, 3 * D), f"orx_bag_gather D={D} L={Lbag} mode={mode}")
    assert (got[:, 3 * D:] == 7).all()
    assert n_bad.item() == bad, (n_bad.item(), bad)


# ---------------------------------------------------------------------------------------------------------------------
# 2. sparse applies
# ---------------------------------------------------------------------------------------------------------------------
def _sweep_rows(D, m, rng):
    """Unnamed rows of every band for the whole-table checks (the guard rows among them)."""
    s = F.band_samples(D, 8, rng)
    rows = np.unique(np.concatenate(list(s.values()) + [m.guard]))
    rows = rows[~np.isin(rows, m.valid)]
    assert {F.row_bands(r, D)[0] for r in rows} == set(F.BANDS)
    return rows


def _check_untouched(ft, rows, before, opt, step, lr, what):
    """Rows no id named: bit-identical, or (Keras Adam) one Adam step with a zero gradient."""
    after = ft.snap(rows)
    if opt != O.OPT_ADAM_DENSE:
        for j, (a, b) in enumerate(zip(after, before)):
            bits_equal(a, b, f"{what}: unnamed rows of table {j} changed")
        return
    var, mm, vv = (x.astype(np.float64) for x in before)
    O.adam_dense(var, mm, vv, np.zeros_like(var), step, lr)
    for j, (a, r) in enumerate(zip(after, (var, mm, vv))):
        close(a, r, f"{what}: Keras Adam sweep, unnamed rows of table {j}")


@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("entry", ["apply", "strided", "bag_sum", "bag_mean"])
@pytest.mark.parametrize("D", DIMS)
def test_sparse_apply(eng, D, entry, optname):
    """orx_sparse_apply, orx_sparse_apply_strided and orx_bag_sparse_apply (sum, mean) on a far table under SGD,
    Adagrad, lazy Adam and Keras Adam: the named rows and their slots against O.apply_sparse on the compact rows; rows
    no id names bit-identical, or under Keras Adam (k_adam_sweep over every row) a zero-gradient Adam step, sampled in
    every band."""
    opt, lr = OPTS[optname]
    ns = N_SLOTS[opt]
    need(table_bytes(D, 1 + ns), f"a far table with {ns} slots")
    m = F.Mix(D, seed=D * 7 + opt)
    ft = FarTable(eng, D, m, ns, seed=3 + opt, opt=opt)
    rng = np.random.default_rng(opt)
    step = 3
    o = N.opt(opt, lr, step=step)
    sweep = _sweep_rows(D, m, rng)
    before_sweep = ft.snap(sweep)
    ref = [x.astype(np.float64) for x in ft.snap(m.valid)]
    n = len(m.ids)
    if entry in ("apply", "strided"):
        vals = rng.standard_normal((n, D)).astype(np.float32)
        if entry == "apply":
            eng.sparse_apply(ft.table(), dev(m.ids, torch.int32), dev(vals), o)
        else:
            ids2d = np.full((n, 2), -1, np.int32)
            ids2d[:, 1] = m.ids
            v3 = np.zeros((n, 2, D), np.float32)
            v3[:, 1] = vals
            eng.sparse_apply_strided(ft.table(), dev(ids2d, torch.int32), 1, dev(v3), o)
        c = compact(m.ids, m.valid, m.rows)
        ok = (c >= 0) & (c < len(m.valid))
        ids_c, rows_c = c[ok], vals[ok].astype(np.float64)
    else:
        Lb, mode = 5, int(entry == "bag_mean")
        B = -(-n // Lb)
        sparse = np.resize(rng.permutation(m.ids), B * Lb).reshape(B, Lb)
        dz = rng.standard_normal((B, D)).astype(np.float32)
        wide = np.full((B, Lb + 2), -1, np.int64)
        wide[:, 1:1 + Lb] = sparse
        eng.bag_sparse_apply(ft.table(), dev(wide, torch.int32), 1, Lb, dev(dz), mode, o)
        csp = compact(sparse, m.valid, m.rows).reshape(B, Lb)
        if mode:                               # the kernel divides in float32 (IEEE) before the rows enter
            v = (csp >= 0) & (csp < len(m.valid))
            dz_rows = np.repeat(dz[:, None, :], Lb, 1) / np.maximum(v.sum(1), 1).astype(np.float32)[:, None, None]
            ids_c, rows_c = csp[v], dz_rows[v].astype(np.float64)
        else:
            ids_c, rows_c = NB.bag_slices(csp, [0, Lb], 0, len(m.valid), dz.astype(np.float64), False)
    s = ref[1:] + [None] * (2 - ns)
    O.apply_sparse(opt, ref[0], s[0], s[1], ids_c, rows_c, step, lr)
    what = f"{entry} {optname} D={D}"
    for j, (got, want) in enumerate(zip(ft.snap(m.valid), ref)):
        close(got, want, f"{what}: named rows of table {j}")
    _check_untouched(ft, sweep, before_sweep, opt, step, lr, what)


# ---------------------------------------------------------------------------------------------------------------------
# 3. fused steps
# ---------------------------------------------------------------------------------------------------------------------
def _triplets(rng, far_ids, B, n_small):
    """(uid / pid / nid ids on the far side, the small side's ids): the far side cycles through the case's ids."""
    a = np.resize(rng.permutation(far_ids), B)
    b = np.resize(rng.permutation(far_ids), B)
    small = rng.integers(0, n_small, B)
    small[5], small[6] = -1, n_small          # bad ids on the small side too
    return a, b, small


def _hinge_ok(user, item, bias, cu, cp, cn, margin=0.5, tol=1e-3):
    h = margin - ((-((user[cu] - item[cp]) ** 2).sum(1) + bias[cp, 0]) - (-((user[cu] - item[cn]) ** 2).sum(1) +
                                                                         bias[cn, 0]))
    return not (np.abs(h) < tol).any()


@pytest.mark.parametrize("kind,side,prefetch", [("bpr", "item", False), ("bpr", "user", False), ("ucml", "item", False),
                                               ("ucml", "user", False), ("bpr", "item", True)])
@pytest.mark.parametrize("D", DIMS)
def test_pairwise_step(eng, D, kind, side, prefetch):
    """orx_pairwise_step under Adagrad with a far item table, then with a far user table (the prefetched form for BPR
    with a far item table): out4 against O.pairwise_train_step on the compact problem, the staged-row count exactly,
    the touched rows and slots, the guard rows bit-identical, and the dispatch record."""
    need(table_bytes(D, 2) + (F.far_rows(D) * 8 if side == "item" else 0), "a far table with its accumulator")
    m = F.Mix(D, seed=D + len(kind) + len(side))
    rng = np.random.default_rng(D + len(kind))
    ft = FarTable(eng, D, m, 1, seed=4, opt=1)
    n_small, B = 3000, 512
    sc = 0.05 if kind == "bpr" else 0.4
    small = dev(rng.uniform(-sc, sc, (n_small, D)).astype(np.float32))
    small_acc = torch.full_like(small, 0.1)
    if side == "item":
        user_t, item_t = N.table(small, small_acc), ft.table()
        I = ft.rows
    else:
        user_t, item_t = ft.table(), N.table(small, small_acc)
        I = n_small
    bias = big(torch.empty(I, 1, device="cuda"))
    eng.fill_uniform(bias, -0.05, 0.05, 9)
    bias_acc = torch.full_like(bias, 0.1)
    bias_t = N.table(bias, bias_acc)
    U = n_small if side == "item" else ft.rows
    for _ in range(50):
        a, b, s = _triplets(rng, m.ids, B, n_small)
        uid, pid, nid = (s, a, b) if side == "item" else (a, s, np.resize(rng.permutation(n_small), B))
        ok = (uid >= 0) & (uid < U) & (pid >= 0) & (pid < I) & (nid >= 0) & (nid < I)
        rows_u, rows_i = np.unique(uid[ok]), np.unique(np.concatenate([pid[ok], nid[ok]]))
        user = rows_of(ft.var if side == "user" else small, rows_u).astype(np.float64)
        item = rows_of(ft.var if side == "item" else small, rows_i).astype(np.float64)
        bias_c = rows_of(bias, rows_i).astype(np.float64)
        cu, cp, cn = (np.searchsorted(r, x[ok]) for r, x in ((rows_u, uid), (rows_i, pid), (rows_i, nid)))
        if kind == "bpr" or _hinge_ok(user, item, bias_c, cu, cp, cn):
            break
    far_rows = rows_i if side == "item" else rows_u
    guard_before = ft.snap(m.guard)
    st = {"user": (np.full_like(user, 0.1) if side == "item" else rows_of(ft.slots[0], rows_u).astype(np.float64),
                   None),
          "item": (rows_of(ft.slots[0], rows_i).astype(np.float64) if side == "item" else np.full_like(item, 0.1),
                   None),
          "bias": (np.full_like(bias_c, 0.1), None)}
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    d_ids = [dev(x, torch.int32) for x in (uid, pid, nid)]
    out4 = torch.zeros(4, device="cuda")
    eng.debug_dispatch_log()
    if prefetch:
        eng.pairwise_prefetch(user_t, item_t, *d_ids, 1, ids_ready=True)
    eng.pairwise_step(k, user_t, item_t, bias_t, *d_ids, N.opt(1, 0.05), out4, margin=0.5)
    _check_step_dispatch(eng, PAIR_OP, k, 1, B, D, "prefetch" if prefetch else 0)
    frac = ok.sum() / B if kind == "bpr" else 1.0
    loss, l2 = O.pairwise_train_step(kind, user, item, bias_c, cu, cp, cn, 1, st, 1, 0.05, margin=0.5, c_loss=frac)
    got = out4.cpu().numpy().astype(np.float64)
    what = f"{kind} far {side} D={D} prefetch={prefetch}"
    close(got[0], loss * frac, f"loss {what}", rtol=2e-5)
    close(got[1], l2, f"l2 {what}", rtol=2e-5)
    n_bad = sum(int(((x < 0) | (x >= r)).sum()) for x, r in ((uid, U), (pid, I), (nid, I)))
    assert got[2] == n_bad, (what, got[2], n_bad)
    assert got[3] == _staged(1, uid[ok], np.concatenate([pid[ok], nid[ok]])), (what, got[3])
    far_ref, far_acc = (item, st["item"][0]) if side == "item" else (user, st["user"][0])
    close(rows_of(ft.var, far_rows), far_ref, f"far rows {what}")
    close(rows_of(ft.slots[0], far_rows), far_acc, f"far accumulator rows {what}")
    close(rows_of(bias, rows_i), bias_c, f"bias {what}")
    for j, (a, b_) in enumerate(zip(ft.snap(m.guard), guard_before)):
        bits_equal(a, b_, f"{what}: guard rows of table {j}")


@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
@pytest.mark.parametrize("D", DIMS)
def test_pointwise_step(eng, D, kind):
    """orx_pointwise_step (GMF, WRMF) under Adagrad with a far item table, against O.pointwise_train_step on the compact
    problem: out4, the staged-row count, the touched rows and slots, GMF's w, the guard rows bit-identical."""
    need(table_bytes(D, 2) + F.far_rows(D) * 8, "a far item table with its accumulator")
    m = F.Mix(D, seed=D + 3 * len(kind))
    rng = np.random.default_rng(D + 5)
    ft = FarTable(eng, D, m, 1, seed=5, opt=1)
    U, B = 3000, 512
    I = ft.rows
    user = dev(rng.uniform(-0.3, 0.3, (U, D)).astype(np.float32))
    uacc = torch.full_like(user, 0.1)
    bias = big(torch.empty(I, 1, device="cuda"))
    eng.fill_uniform(bias, -0.3, 0.3, 11)
    bacc = torch.full_like(bias, 0.1)
    w = dev(rng.uniform(-0.3, 0.3, (1, D)).astype(np.float32))
    wacc = torch.full_like(w, 0.1)
    uid = rng.integers(0, U, B)
    uid[3], uid[4] = -1, U
    iid = np.resize(rng.permutation(m.ids), B)
    label = (rng.random(B) < 0.4).astype(np.float32)
    a, b, sig = (1.0, 1.0, False) if kind == "gmf" else (3.0, 0.5, False)
    ok = (uid >= 0) & (uid < U) & (iid >= 0) & (iid < I)
    rows_u, rows_i = np.unique(uid[ok]), np.unique(iid[ok])
    ref_u = rows_of(user, rows_u).astype(np.float64)
    ref_i = rows_of(ft.var, rows_i).astype(np.float64)
    ref_b = rows_of(bias, rows_i).astype(np.float64)
    ref_w = w.cpu().numpy().reshape(-1, 1).astype(np.float64)
    st = {"user": (np.full_like(ref_u, 0.1), None), "item": (rows_of(ft.slots[0], rows_i).astype(np.float64), None),
          "bias": (np.full_like(ref_b, 0.1), None), "w": (np.full_like(ref_w, 0.1), None)}
    guard_before = ft.snap(m.guard)
    k = N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF
    out4 = torch.zeros(4, device="cuda")
    eng.debug_dispatch_log()
    eng.pointwise_step(k, N.table(user, uacc), ft.table(), N.table(bias, bacc),
                       N.table(w, wacc) if kind == "gmf" else None, dev(uid, torch.int32), dev(iid, torch.int32),
                       dev(label), N.opt(1, 0.05), out4, a, b, sig)
    _check_step_dispatch(eng, POINT_OP, k, 1, B, D)
    frac = ok.sum() / B if kind == "gmf" else 1.0
    cu, ci = np.searchsorted(rows_u, uid[ok]), np.searchsorted(rows_i, iid[ok])
    loss, l2 = O.pointwise_train_step(kind, ref_u, ref_i, ref_b, ref_w if kind == "gmf" else None, cu, ci, label[ok], 1,
                                      st, 1, 0.05, a, b, sig, c_loss=frac)
    got = out4.cpu().numpy().astype(np.float64)
    what = f"{kind} far item D={D}"
    close(got[0], loss * frac, f"loss {what}", rtol=2e-5)
    close(got[1], l2, f"l2 {what}", rtol=2e-5)
    assert got[2] == int(((uid < 0) | (uid >= U)).sum() + ((iid < 0) | (iid >= I)).sum()), (what, got)
    assert got[3] == _staged(1, uid[ok], iid[ok]), (what, got)
    close(rows_of(ft.var, rows_i), ref_i, f"item rows {what}")
    close(rows_of(ft.slots[0], rows_i), st["item"][0], f"item accumulator {what}")
    close(rows_of(user, rows_u), ref_u, f"user rows {what}")
    close(rows_of(bias, rows_i), ref_b, f"bias {what}")
    if kind == "gmf":
        close(w.cpu().numpy().reshape(-1, 1), ref_w, f"w {what}")
    for j, (x, y) in enumerate(zip(ft.snap(m.guard), guard_before)):
        bits_equal(x, y, f"{what}: guard rows of table {j}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. censors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", DIMS)
def test_censor(eng, D):
    """orx_censor on far rows and their aliases in one id list, against O.censor on the compact rows."""
    need(table_bytes(D), "a far table")
    m = F.Mix(D, seed=D + 11)
    ft = FarTable(eng, D, m, seed=6)
    ref = rows_of(ft.var, m.valid).astype(np.float64)
    guard_before = ft.snap(m.guard)
    eng.censor(ft.var, dev(m.ids, torch.int32))
    c = compact(m.ids, m.valid, m.rows)
    O.censor(ref, c[(c >= 0) & (c < len(m.valid))])
    close(rows_of(ft.var, m.valid), ref, f"censor D={D}", atol=1e-6)
    bits_equal(ft.snap(m.guard)[0], guard_before[0], f"censor D={D}: guard rows")


@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("D", DIMS)
def test_censor_shard(eng, D, rank):
    """orx_censor_shard at world 2 with a far local shard (global id = 2 * local + rank <= 2^31 - 1): the owned ids
    against O.censor on the compact local rows, ids of the other rank and bad ids ignored, the dispatch record."""
    need(table_bytes(D), "a far shard")
    m = F.Mix(D, seed=D + 13 + rank)
    ft = FarTable(eng, D, m, seed=7)
    total = 2 * ft.rows
    assert N.shard_rows(total, rank, 2) == ft.rows and total - 1 <= INT32_MAX
    rng = np.random.default_rng(rank)
    loc = m.ids
    glob = np.where((loc >= 0) & (loc < m.rows), 2 * loc + rank, np.where(loc < 0, -1, total))
    other = 2 * rng.choice(m.far, 16) + (1 - rank)          # owned by the other rank: its far rows' twins
    ids = np.concatenate([glob, other, [total - 2 + rank]])  # the last row this rank owns
    ids = ids[rng.permutation(len(ids))]
    n_per, n_blocks, stride = -(-len(ids) // 2), 2, -(-len(ids) // 2) + 3
    flat = np.full(stride * 2, -1, np.int64)
    flat[:n_per] = ids[:n_per]
    flat[stride:stride + len(ids) - n_per] = ids[n_per:]
    valid = np.unique(np.concatenate([m.valid, [ft.rows - 1]]))
    ref = rows_of(ft.var, valid).astype(np.float64)
    guard_before = ft.snap(m.guard)
    eng.debug_dispatch_log()
    eng.censor_shard(ft.var, total, 2, rank, dev(flat, torch.int32), n_per, stride, n_blocks)
    rec = [r for r in eng.debug_dispatch_log() if r.op == L.ORX_OP_CENSOR_SHARD]
    variant = N.ORX_VARIANT_CENSOR_VEC if D % 4 == 0 and D <= 128 else N.ORX_VARIANT_CENSOR_SCALAR
    assert rec == [N.Dispatch(L.ORX_OP_CENSOR_SHARD, variant, rank, 0, n_per * n_blocks, ft.rows, D, 2)], rec
    used = np.concatenate([flat[:n_per], flat[stride:stride + n_per]])
    mine = used[(used >= 0) & (used < total) & (used % 2 == rank)] // 2
    O.censor(ref, np.searchsorted(valid, mine))
    close(rows_of(ft.var, valid), ref, f"censor_shard D={D} rank={rank}", atol=1e-6)
    bits_equal(ft.snap(m.guard)[0], guard_before[0], f"censor_shard D={D}: guard rows")


# ---------------------------------------------------------------------------------------------------------------------
# 5. row-sharded building blocks on a far local shard
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["user", "item"])
@pytest.mark.parametrize("D", DIMS)
def test_pointwise_serve(eng, D, side):
    """orx_pointwise_serve with the far shard as the user side, then as the item side: each served row bit-equal to
    the host copy of its row (the bias in column D for items), zeros elsewhere, the local row columns exact."""
    need(table_bytes(D) + F.far_rows(D) * 4, "a far shard and its bias")
    m = F.Mix(D, seed=D + 17)
    ft = FarTable(eng, D, m, seed=8)
    rng = np.random.default_rng(D)
    n_small, ld = 1000, D + 4
    small = dev(rng.uniform(-1, 1, (n_small, D)).astype(np.float32))
    if side == "user":
        Lu, lu, li = ft.rows + 3, ft.rows, n_small
        user, item = ft.var, small
        bias = dev(rng.uniform(-1, 1, n_small).astype(np.float32))
        far_req = m.ids
        small_req = Lu + rng.integers(0, n_small, 40)
    else:
        Lu, lu, li = n_small + 2, n_small, ft.rows
        user, item = small, ft.var
        bias = big(torch.empty(ft.rows, device="cuda"))
        eng.fill_uniform(bias, 3.0, 4.0, 12)
        far_req = np.where((m.ids >= 0) & (m.ids < m.rows), Lu + m.ids, np.where(m.ids < 0, -1, Lu + li))
        small_req = rng.integers(0, n_small, 40)
    assert Lu + li <= INT32_MAX
    req = np.concatenate([far_req, small_req, [lu, Lu - 1, Lu + li, -1]])     # gaps and past-the-end: zero rows
    req = req[np.random.default_rng(1).permutation(len(req))]
    rows, ul, il = eng.pointwise_serve(user, item, bias, lu, li, Lu, dev(req, torch.int32), ld)
    want = np.zeros((len(req), ld), np.float32)
    want_ul = np.where((req >= 0) & (req < lu), req, -1)
    want_il = np.where((req >= Lu) & (req < Lu + li), req - Lu, -1)
    u_rows, i_rows = want_ul[want_ul >= 0], want_il[want_il >= 0]
    hu = rows_of(user, u_rows) if len(u_rows) else np.zeros((0, D), np.float32)
    hi = rows_of(item, i_rows) if len(i_rows) else np.zeros((0, D), np.float32)
    want[want_ul >= 0, :D] = hu
    want[want_il >= 0, :D] = hi
    want[want_il >= 0, D] = bias.index_select(0, idx(i_rows)).cpu().numpy()
    bits_equal(rows.cpu().numpy(), want, f"pointwise_serve far {side} D={D}")
    assert np.array_equal(ul.cpu().numpy(), want_ul) and np.array_equal(il.cpu().numpy(), want_il)


@pytest.mark.parametrize("D", DIMS)
def test_rows_scale(eng, D):
    """orx_rows_scale over the whole far table: sampled rows of every band, the planted ones included, bit-equal to
    the float32 product."""
    need(table_bytes(D), "a far table")
    m = F.Mix(D, seed=D + 19)
    ft = FarTable(eng, D, m, seed=9)
    rng = np.random.default_rng(D)
    rows = np.unique(np.concatenate(list(F.band_samples(D, 16, rng).values()) + [m.far, [m.last]]))
    before = rows_of(ft.var, rows)
    scale = rng.uniform(0.5, 2.0, D).astype(np.float32)
    eng.rows_scale(ft.var, dev(scale))
    bits_equal(rows_of(ft.var, rows), before * scale[None, :], f"rows_scale D={D}")


def test_fill_uniform_far(eng):
    """orx_fill_uniform over a whole far table: the elements at 0, 2^31 - 16, 2^32 - 16, the far band's end and the
    last element, bit for bit against the host restatement of the stream (a truncated index would repeat an earlier
    draw)."""
    D = 128
    need(table_bytes(D), "a far table")
    t = big(torch.empty(F.far_rows(D), D, device="cuda"))
    flat = t.view(-1)
    n = flat.numel()
    for seed in (5, 2 ** 63 + 5):
        eng.fill_uniform(t, 0.0, 1.0, seed)
        for start in (0, 2 ** 31 - 16, 2 ** 32 - 16, 2 ** 32, F.FAR_END - 16, n - 16):
            got = flat[start:start + 32].cpu().numpy()
            want = S.fill_uniform_u(seed, start, min(start + 32, n))
            bits_equal(got, want, f"fill_uniform seed={seed} at {start}")


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_shard_step_far_item_shard(eng, kind):
    """orx_shard_step (the home-routed row-sharded step: route, request, serve, compute, apply) at world 1 with a far
    item shard (D = 128) under SGD, the optimizer it accepts with the fewest slots: the global loss against
    O.pairwise_train_step on the compact problem, the touched rows, the guard rows bit-identical."""
    from openrec_b200.sharded import LoopbackGroup
    D = 128
    need(table_bytes(D) + F.far_rows(D) * 4, "a far item shard and its bias")
    m = F.Mix(D, seed=31 + len(kind))
    rng = np.random.default_rng(37 + len(kind))
    ft = FarTable(eng, D, m, seed=13)
    U, B, I = 3000, 512, ft.rows
    sc = 0.05 if kind == "bpr" else 0.4
    user = dev(rng.uniform(-sc, sc, (U, D)).astype(np.float32))
    bias = big(torch.empty(I, 1, device="cuda"))
    eng.fill_uniform(bias, -0.05, 0.05, 14)
    for _ in range(50):
        pid, nid, uid = _triplets(rng, m.ids, B, U)
        ok = (uid >= 0) & (uid < U) & (pid >= 0) & (pid < I) & (nid >= 0) & (nid < I)
        rows_u, rows_i = np.unique(uid[ok]), np.unique(np.concatenate([pid[ok], nid[ok]]))
        ref_u = rows_of(user, rows_u).astype(np.float64)
        ref_i = rows_of(ft.var, rows_i).astype(np.float64)
        ref_b = rows_of(bias, rows_i).astype(np.float64)
        cu, cp, cn = (np.searchsorted(r, x[ok]) for r, x in ((rows_u, uid), (rows_i, pid), (rows_i, nid)))
        if kind == "bpr" or _hinge_ok(ref_u, ref_i, ref_b, cu, cp, cn):
            break
    assert np.isin(m.far, rows_i).sum() >= len(m.far) // 2 and np.isin(m.alias, rows_i).any()
    guard_before = ft.snap(m.guard)
    g = LoopbackGroup(1, U, I, D, B, kind=0 if kind == "bpr" else 1, opt_kind=0, lr=0.05, init=False,
                      tables=(user, ft.var, bias))
    try:
        out = g.step([tuple(dev(x, torch.int32) for x in (uid, pid, nid))])[0].cpu().numpy().astype(np.float64)
        g.check()
    finally:
        g.close()
    frac = ok.sum() / B if kind == "bpr" else 1.0     # BPR's 1/B is over the submitted batch
    loss, l2 = O.pairwise_train_step(kind, ref_u, ref_i, ref_b, cu, cp, cn, O.OPT_SGD, {}, 1, 0.05, margin=0.5,
                                     c_loss=frac)
    what = f"shard_step {kind} far item shard"
    np.testing.assert_allclose(out, [loss * frac, l2], rtol=3e-5, atol=1e-6, err_msg=what)
    tol = 2e-5 if kind == "bpr" else 2e-4              # UCML: the bar of tests/test_gpu_shard_loopback.py
    close(rows_of(ft.var, rows_i), ref_i, f"item rows {what}", atol=tol)
    close(rows_of(user, rows_u), ref_u, f"user rows {what}", atol=tol)
    close(rows_of(bias, rows_i), ref_b, f"bias {what}", atol=tol)
    bits_equal(ft.snap(m.guard)[0], guard_before[0], f"{what}: guard rows")


# ---------------------------------------------------------------------------------------------------------------------
# 6. evaluation and retrieval over a far item table (planted catalogue)
# ---------------------------------------------------------------------------------------------------------------------
class Planted:
    """A zeroed item table of I items (one or more shards) with planted items: item row c * e0, user rows e0, so the
    score of planted item j is exactly c_j (dot) or -(1 - c_j)^2 (neg_sqdist) and every other item scores the bulk value
    0 or -1.  `items` maps global item ids to their scores; `top` lists the items that outrank the bulk."""

    def __init__(self, kind, top_ids, low_ids):
        dot = kind == N.ORX_SCORE_DOT
        self.bulk = 0.0 if dot else -1.0
        ids = list(top_ids) + list(low_ids)
        n_top = len(top_ids)
        # distinct dyadic scores: top ids above the bulk value (descending), the others spread around it
        ks = np.arange(1, len(ids) + 1)
        if dot:
            c = np.where(ks <= n_top, (len(ids) + 10 - ks) / 64.0, (ks - n_top - (len(ids) - n_top) // 2 - 0.5) / 64.0)
            score = c
        else:
            k = np.where(ks <= n_top, ks, 1100 + ks)          # |1 - c| < 1: nearer the user than the bulk
            assert n_top < 1024
            sign = np.where(ks % 2 == 0, 1.0, -1.0)
            c = 1.0 + sign * k / 1024.0
            score = -(k / 1024.0) ** 2
        self.items = dict(zip((int(i) for i in ids), score.tolist()))
        self.c = dict(zip((int(i) for i in ids), c.astype(np.float32).tolist()))
        assert len(set(self.items.values())) == len(ids) and self.bulk not in self.items.values()
        if not dot:
            assert all(s > self.bulk for s in score[:n_top]) and all(s < self.bulk for s in score[n_top:])

    def fill(self, item_tab, ids_local, ids_global):
        """Plant the items ids_global at local rows ids_local of item_tab (zeroed)."""
        vals = np.zeros((len(ids_local), item_tab.shape[1]), np.float32)
        vals[:, 0] = [self.c[int(g)] for g in ids_global]
        item_tab.index_copy_(0, idx(ids_local), dev(vals))


def _csr(lists):
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    items = np.concatenate([np.asarray(x, np.int64) for x in lists]).astype(np.int32)
    return dev(off, torch.int64), dev(items, torch.int32)


def _user_lists(rng, pl, I, Bu, row_of=None, D=1):
    """Per user: sorted positives and exclusions (disjoint), each among the planted items and the bulk.  Bulk items
    whose row (row_of(item), the local row of a shard) lies in the mid band are not used: the kernels read the rows of
    a user's positives and exclusions by id."""
    planted = np.array(sorted(pl.items), np.int64)
    taken = set(planted.tolist())
    row_of = row_of or (lambda g: g)
    usable = lambda g: g not in taken and "mid" not in F.row_bands(row_of(g), D)
    pos, excl = [], []
    for u in range(Bu):
        pick = rng.permutation(planted)
        bulk = []
        while len(bulk) < 6:
            b = int(rng.integers(0, I))
            if usable(b) and b not in bulk:
                bulk.append(b)
        bulk += [I - 1] if u == 0 and usable(I - 1) else []
        p = set(pick[:5 + u].tolist()) | set(bulk[:3])
        e = set(pick[5 + u:12 + 2 * u].tolist()) | set(bulk[3:])
        pos.append(sorted(p))
        excl.append(sorted(e - p))
    return pos, excl


def _want_rank(pl, I, pos, excl, at):
    """AUC / NDCG / Recall of k_rank_metrics from the planted scores plus the count of bulk ties: AUC counts eval
    items e (neither positive nor excluded) with pred_e <= pred_p; rank_p counts non-excluded items with a larger
    expf(pred) (all scores are distinct dyadic values, far apart, so that is a larger pred)."""
    sc = pl.items
    auc, ndcg, rec = [], [], []
    for p_list, e_list in zip(pos, excl):
        P, E = set(p_list), set(e_list)
        n_bulk = I - len(sc)
        bulk_eval = n_bulk - sum(1 for x in P | E if x not in sc)
        bulk_open = n_bulk - sum(1 for x in E if x not in sc)
        pe = [s for i, s in sc.items() if i not in P and i not in E]
        po = [s for i, s in sc.items() if i not in E]
        n_eval = I - len(P | E)
        total, d, h = 0, np.zeros(len(at)), np.zeros(len(at))
        for p in p_list:
            v = sc.get(p, pl.bulk)
            total += bulk_eval * (pl.bulk <= v) + sum(1 for s in pe if s <= v)
            if p in E:
                continue
            r = bulk_open * (pl.bulk > v) + sum(1 for s in po if s > v)
            for j, k in enumerate(at):
                if r < k:
                    d[j] += 1.0 / np.log2(r + 2.0)
                    h[j] += 1
        auc.append(np.float32(total) / np.float32(len(p_list) * n_eval))
        ndcg.append(d)
        rec.append(h / len(p_list))
    return np.array(auc, np.float32), np.array(ndcg), np.array(rec)


def _check_rank(got, want, what):
    auc, ndcg, rec = (t.cpu().numpy() for t in got)
    np.testing.assert_allclose(auc, want[0], rtol=1e-6, err_msg=f"AUC {what}")
    np.testing.assert_allclose(ndcg, want[1], rtol=1e-5, err_msg=f"NDCG {what}")
    np.testing.assert_allclose(rec, want[2], rtol=1e-6, err_msg=f"Recall {what}")


def _want_topk(pl, excl, k):
    out = []
    for e in excl:
        cand = sorted(((-s, i) for i, s in pl.items.items() if i not in set(e)))
        out.append(([i for _, i in cand[:k]], [-s for s, _ in cand[:k]]))
    return out


def _check_topk(items, scores, want, what):
    items, scores = items.cpu().numpy(), scores.cpu().numpy()
    for u, (wi, ws) in enumerate(want):
        assert items[u].tolist() == wi, (what, u, items[u][:8], wi[:8])
        bits_equal(scores[u], np.array(ws, np.float32), f"{what} user {u}")


AT = (5, 50, 500)
TOPK = 48


def _far_and_alias(m):
    """(far items, their alias items): the planted rows' ids in the catalogue."""
    alias = sorted({a for r in m.far for a in F.alias_rows(r, m.D)})
    return m.far.tolist(), [a for a in alias if a not in set(m.far.tolist())]


@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_score_rank_topk_far(eng, kind):
    """orx_score_rank and orx_score_topk over a far item table (D = 128) with a planted catalogue: far-band items
    outrank everything, their aliases and the bulk tie; the metrics from the planted scores plus the bulk ties, the
    top-K the planted far items with their exact ids and scores."""
    D = 128
    need(table_bytes(D) + F.far_rows(D) * 4, "a far item table and its bias")
    m = F.Mix(D, seed=23, n_far=160)
    far, alias = _far_and_alias(m)
    pl = Planted(kind, far, alias)
    I = m.rows
    item = big(torch.zeros(I, D, device="cuda"))
    bias = big(torch.zeros(I, device="cuda"))
    pl.fill(item, list(pl.items), list(pl.items))
    Bu = 8
    user = torch.zeros(Bu, D, device="cuda")
    user[:, 0] = 1.0
    rng = np.random.default_rng(kind)
    pos, excl = _user_lists(rng, pl, I, Bu, D=D)
    po, pi = _csr(pos)
    eo, ei = _csr(excl)
    uid = dev(np.arange(Bu), torch.int32)
    got = eng.score_rank(kind, user, uid, item, bias, po, pi, eo, ei, max(len(p) for p in pos), at=AT)
    _check_rank(got, _want_rank(pl, I, pos, excl, AT), f"score_rank far kind={kind}")
    items, scores = eng.score_topk(kind, user, uid, item, bias, eo, ei, TOPK)
    _check_topk(items, scores, _want_topk(pl, excl, TOPK), f"score_topk far kind={kind}")
    assert set(items.cpu().numpy().reshape(-1).tolist()) <= set(far)


@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_score_rank_topk_shard_far(eng, kind):
    """orx_score_rank_shard / orx_score_topk_shard phase by phase at world 2 with both item shards far: the same
    planted-catalogue expectations on the global ids (global item = 2 * local + rank)."""
    D = 128
    need(table_bytes(D, 2) + F.far_rows(D) * 8, "two far item shards and their biases")
    rows_l = F.far_rows(D)
    I = 2 * rows_l
    assert I - 1 <= INT32_MAX
    mixes = [F.Mix(D, seed=29 + r, n_far=80) for r in range(2)]
    fa = [_far_and_alias(mm) for mm in mixes]
    far_g = [2 * x + r for r in range(2) for x in fa[r][0]]
    alias_g = [2 * x + r for r in range(2) for x in fa[r][1]]
    pl = Planted(kind, far_g, alias_g)
    shards, biases = [], []
    for r in range(2):
        t = big(torch.zeros(rows_l, D, device="cuda"))
        loc = fa[r][0] + fa[r][1]
        pl.fill(t, loc, [2 * x + r for x in loc])
        shards.append(t)
        biases.append(big(torch.zeros(rows_l, device="cuda")))
    Bu = 8
    user = torch.zeros(Bu, D, device="cuda")
    user[:, 0] = 1.0
    rng = np.random.default_rng(kind + 7)
    pos, excl = _user_lists(rng, pl, I, Bu, row_of=lambda g: g // 2, D=D)
    po, pi = _csr(pos)
    eo, ei = _csr(excl)
    uid = dev(np.arange(Bu), torch.int32)
    parts = [(eng, kind, user[r::2].contiguous(), shards[r], biases[r], N.rowshard(2, r, Bu, I)) for r in range(2)]
    outs = score_rank_sharded(parts, loopback_sum, uid, po, pi, eo, ei, max(len(p) for p in pos), at=AT)
    want = _want_rank(pl, I, pos, excl, AT)
    for r, o in enumerate(outs):
        _check_rank(o, want, f"score_rank_shard rank {r} kind={kind}")
    wt = _want_topk(pl, excl, TOPK)
    for r, (items, scores) in enumerate(score_topk_sharded(parts, loopback_sum, uid, eo, ei, TOPK)):
        _check_topk(items, scores, wt, f"score_topk_shard rank {r} kind={kind}")


@pytest.mark.parametrize("kind", [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST], ids=["dot", "neg_sqdist"])
def test_score_rank_topk_int32_max_items(eng, kind):
    """orx_score_rank / orx_score_topk over I = 2^31 - 1 items at D = 1 (a planted catalogue, with the bias): items
    at 2^31 - 2, 2^31 - 65, ... -- the item-id arithmetic of the last tile and the top-K key packing of the largest
    ids."""
    I, D = INT32_MAX, 1
    need(2 * I * 4, "an item table and a bias of 2^31 - 1 rows")
    top = [I - 1 - 1, I - 1 - 64, I - 1, I - 1 - 127, I - 1 - 1000, I - 1 - 4096] + [I - 1 - 63 * j for j in range(3, 40)]
    top = sorted(set(top), reverse=True)
    low = [0, 1, 2 ** 30, I - 1 - 2 ** 20] + [I - 1 - 5000 - 7 * j for j in range(20)]
    pl = Planted(kind, top, low)
    item = big(torch.zeros(I, D, device="cuda"))
    bias = big(torch.zeros(I, device="cuda"))
    pl.fill(item, list(pl.items), list(pl.items))
    Bu = 4
    user = torch.ones(Bu, D, device="cuda")
    rng = np.random.default_rng(kind + 11)
    pos, excl = _user_lists(rng, pl, I, Bu)
    po, pi = _csr(pos)
    eo, ei = _csr(excl)
    uid = dev(np.arange(Bu), torch.int32)
    got = eng.score_rank(kind, user, uid, item, bias, po, pi, eo, ei, max(len(p) for p in pos), at=AT)
    _check_rank(got, _want_rank(pl, I, pos, excl, AT), f"score_rank I=2^31-1 kind={kind}")
    k = 24
    items, scores = eng.score_topk(kind, user, uid, item, bias, eo, ei, k)
    _check_topk(items, scores, _want_topk(pl, excl, k), f"score_topk I=2^31-1 kind={kind}")


# ---------------------------------------------------------------------------------------------------------------------
# row-space limits at 2^31 - 1 rows (no large memory)
# ---------------------------------------------------------------------------------------------------------------------
ROW_OFF = [0, 5, INT32_MAX]


def _edge_sparse(rng, B):
    """[B, 2] ids of tables with vocabularies 5 and 2^31 - 6: the very top of the last table, row 0, padding, = vocab,
    and random ids; the top ids repeat across rows."""
    v1 = ROW_OFF[2] - ROW_OFF[1]
    s = np.zeros((B, 2), np.int64)
    s[:, 0] = rng.integers(-1, 6, B)
    s[:, 1] = rng.choice(np.array([v1 - 1, v1 - 2, v1 - 3, v1 - 1024, 0, -1, v1, 2 ** 30]), B)
    s[: B // 4, 1] = rng.integers(0, v1, B // 4)
    return s


@pytest.mark.parametrize("world", [1, 2, 3, 1000, 1024])
def test_lookup_bucket_row_space_edge(eng, world):
    """orx_lookup_bucket over the row space row_off = [0, 5, 2^31 - 1]: the sort key owner * L + local approaches
    2^32 and the radix sort runs all 32 bits; every output against lookup_bucket_np."""
    rng = np.random.default_rng(world)
    B = 3000
    s = _edge_sparse(rng, B)
    got = [t.cpu().numpy() for t in eng.lookup_bucket(dev(s, torch.int32), ROW_OFF, world)]
    counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(s, ROW_OFF, world)
    n_uniq, n_valid = len(send_local), int(grp_off[-1])
    assert np.array_equal(got[0], counts)
    assert np.array_equal(got[1][:n_uniq], send_local)
    assert np.array_equal(got[2], slot)
    assert np.array_equal(got[3][:n_uniq + 1], grp_off)
    assert np.array_equal(got[4][:n_valid], grp_idx)
    top = ROW_OFF[2] - 1                                   # the last row of the space is in the batch
    assert ((s[:, 1] + ROW_OFF[1]) == top).any()


def test_bag_shard_lookups_row_space_edge(eng):
    """orx_bag_shard_lookups with the same row space (bags of 2 and 3 columns): global rows exact, -1 for padding and
    bad ids; their bucket as [B*C, 1] with row_off = {0, G} equal to the T-table bucket's restatement; a row space of
    2^31 rows is refused."""
    rng = np.random.default_rng(3)
    B, col_off = 1000, [0, 2, 5]
    s = np.concatenate([_edge_sparse(rng, B)[:, :1], _edge_sparse(rng, B)[:, :1],
                        _edge_sparse(rng, B)[:, 1:], _edge_sparse(rng, B)[:, 1:], _edge_sparse(rng, B)[:, 1:]], 1)
    out = eng.bag_shard_lookups(dev(s, torch.int32), col_off, ROW_OFF).cpu().numpy()
    want = np.full_like(s, -1)
    for k in range(2):
        v = ROW_OFF[k + 1] - ROW_OFF[k]
        blk = s[:, col_off[k]:col_off[k + 1]]
        want[:, col_off[k]:col_off[k + 1]] = np.where((blk >= 0) & (blk < v), ROW_OFF[k] + blk, -1)
    assert np.array_equal(out, want)
    assert out.max() == INT32_MAX - 1
    for world in (2, 1024):
        got = [t.cpu().numpy() for t in eng.lookup_bucket(dev(out.reshape(-1, 1), torch.int32), [0, INT32_MAX],
                                                          world)]
        counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(out.reshape(-1, 1), [0, INT32_MAX], world)
        assert np.array_equal(got[0], counts) and np.array_equal(got[2], slot)
        assert np.array_equal(got[1][:len(send_local)], send_local)
        assert np.array_equal(got[4][:int(grp_off[-1])], grp_idx)
    with pytest.raises(RuntimeError, match=r"\(status -1\)"):
        eng.bag_shard_lookups(dev(s, torch.int32), col_off, [0, 5, 2 ** 31])


@pytest.mark.parametrize("world", [1, 2, 3])
def test_pointwise_shard_limits(eng, world):
    """The row-sharded GMF / WRMF row space at its limit world * Lu + I = 2^31 - 1 (Lu = ceil(U / world)): the model's
    row offsets accept it and refuse one more item; orx_pointwise_shard_lookups at U, I = 2^31 - 1 with ids at the
    top (and refuses U = 2^31); orx_owner_bucket_combined with the largest user and item ids of the space."""
    rng = np.random.default_rng(world)
    U = 2 ** 30 + 7
    Lu = -(-U // world)
    I = INT32_MAX - world * Lu
    assert row_offsets([world * Lu, I])[-1] == INT32_MAX
    with pytest.raises(ValueError):
        row_offsets([world * Lu, I + 1])
    B = 600
    uid = rng.integers(0, U, B)
    iid = rng.integers(0, I, B)
    uid[:4], iid[:4] = [U - 1, U - 2, 0, U], [I - 1, 0, I, I - 2]
    uid[4:8] = [-1, U - 1, U - 1, INT32_MAX]
    iid[8:12] = [I - 1, I - 1, -1, INT32_MAX]
    got = eng.pointwise_shard_lookups(dev(uid, torch.int32), dev(iid, torch.int32), U, I).cpu().numpy()
    ok = (uid >= 0) & (uid < U) & (iid >= 0) & (iid < I)
    want = np.where(ok[:, None], np.stack([uid, iid], 1), -1)
    assert np.array_equal(got, want)
    # the same lookups through the row space {0, world * Lu, world * Lu + I}: the global rows reach 2^31 - 2
    buck = [t.cpu().numpy() for t in eng.lookup_bucket(dev(got, torch.int32), row_offsets([world * Lu, I]), world)]
    counts, send_local, slot, grp_off, grp_idx = lookup_bucket_np(got, row_offsets([world * Lu, I]), world)
    assert np.array_equal(buck[0], counts) and np.array_equal(buck[2], slot)
    assert np.array_equal(buck[1][:len(send_local)], send_local)
    top = INT32_MAX
    uu = np.array([top - 1, top - 2, top - 3, 0, 1, 5], np.int64)
    got = eng.pointwise_shard_lookups(dev(uu, torch.int32), dev(uu, torch.int32), top, top).cpu().numpy()
    assert np.array_equal(got, np.stack([uu, uu], 1))
    with pytest.raises(RuntimeError, match=r"\(status -1\)"):
        eng.pointwise_shard_lookups(dev(uu, torch.int32), dev(uu, torch.int32), 2 ** 31, top)
    # orx_owner_bucket_combined: users then items of one space of U + I = 2^31 - 1 rows per world
    Uc = 2 ** 30 + 3
    Ic = INT32_MAX - world * (-(-Uc // world))
    n_user = 300
    ids = np.concatenate([np.concatenate([[Uc - 1, Uc - 2, 0], rng.integers(0, Uc, n_user - 3)]),
                          np.concatenate([[Ic - 1, Ic - 2, 0], rng.integers(0, Ic, 297)])]).astype(np.int64)
    counts, send_local, slot = (t.cpu().numpy() for t in eng.owner_bucket_combined(dev(ids, torch.int32), n_user, Uc,
                                                                                    world))
    owner = ids % world
    user_rows = (Uc - owner + world - 1) // world
    want_local = ids // world + np.where(np.arange(len(ids)) >= n_user, user_rows, 0)
    assert want_local.max() <= INT32_MAX
    assert np.array_equal(counts, np.bincount(owner, minlength=world))
    assert sorted(slot.tolist()) == list(range(len(ids)))
    assert np.array_equal(send_local[slot], want_local)
