"""The per-triplet records of a prefetched pairwise batch (k_index_resolve) and the step that reads them in place of the
index probes: records against a numpy oracle, the record path against the probing path (ORX_PAIR_RESOLVE=0) and the
un-prefetched step, and the records through the prefetch lifecycle (alternating sets, a dropped prefetch, the host-buffer
entry point)."""
import os

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

OPTS = {"sgd": (L.ORX_OPT_SGD, 0.05), "adagrad": (L.ORX_OPT_ADAGRAD, 0.05), "adam_lazy": (L.ORX_OPT_ADAM_LAZY, 0.01),
        "adam_dense": (L.ORX_OPT_ADAM_DENSE, 0.01)}
PAIR_OP = L.ORX_OP_PAIRWISE_STEP


def _engine(resolve):
    """A handle of its own, created with ORX_PAIR_RESOLVE set (the handle reads it once, at creation)."""
    old = os.environ.get("ORX_PAIR_RESOLVE")
    os.environ["ORX_PAIR_RESOLVE"] = "1" if resolve else "0"
    try:
        return N.Engine(torch.cuda.current_device())
    finally:
        if old is None:
            del os.environ["ORX_PAIR_RESOLVE"]
        else:
            os.environ["ORX_PAIR_RESOLVE"] = old


@pytest.fixture(scope="module")
def engines():
    e = {True: _engine(True), False: _engine(False)}
    yield e
    for x in e.values():
        x.close()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def _valid(ids, U, I):
    uid, pid, nid = ids
    return (uid >= 0) & (uid < U) & (pid >= 0) & (pid < I) & (nid >= 0) & (nid < I)


def _counts(ids, U, I):
    """-> (user, item) occurrence counts of every row over the valid triplets."""
    uid, pid, nid = ids
    ok = _valid(ids, U, I)
    return (np.bincount(uid[ok], minlength=U),
            np.bincount(np.concatenate([pid[ok], nid[ok]]), minlength=I))


def check_records(rec, ids, U, I, dense, what=""):
    """rec (int32 [B, 4]) against the oracle of the ids.  Staging indices depend on the order of the index build's
    atomics, so they are checked for what they must be: -1 exactly for rows seen once (mode 0), else one index per
    distinct row, the indices of a side being 0 .. n_staged - 1.  -> staged rows of both sides."""
    rec = rec.cpu().numpy()
    uid, pid, nid = ids
    ok = _valid(ids, U, I)
    cu, ci = _counts(ids, U, I)
    flags = ok.astype(np.int64)
    if not dense:
        flags |= ok * ((cu[np.clip(uid, 0, U - 1)] == 1) * 2 + (ci[np.clip(pid, 0, I - 1)] == 1) * 4
                       + (ci[np.clip(nid, 0, I - 1)] == 1) * 8)
    np.testing.assert_array_equal(rec[:, 0], flags, err_msg=f"flags {what}")
    assert (rec[~ok, 1:] == -1).all(), f"an invalid triplet has a staging index {what}"
    staged = 0
    for side, cols in (((uid,), (1,)), ((pid, nid), (2, 3))):
        x = np.concatenate([s[ok] for s in side])
        d = np.concatenate([rec[ok, c] for c in cols])
        cnt = cu if cols == (1,) else ci
        st = (cnt[x] > 1) if not dense else np.ones(len(x), bool)
        assert (d[~st] == -1).all(), f"a row seen once has a staging index {what}"
        assert (d[st] >= 0).all(), f"a staged row has no staging index {what}"
        pairs = np.unique(np.stack([x[st], d[st]], 1), axis=0) if st.any() else np.zeros((0, 2), np.int64)
        n = len(np.unique(x[st]))
        assert len(pairs) == n, f"row -> staging index is not one to one {what}"
        np.testing.assert_array_equal(np.sort(pairs[:, 1]), np.arange(n), err_msg=f"staging indices {what}")
        staged += n
    return staged


def make_ids(rng, case, U, I, B):
    if case == "owned":        # every row referenced once
        uid = rng.choice(U, B, replace=False)
        it = rng.choice(I, 2 * B, replace=False)
        return [x.astype(np.int32) for x in (uid, it[:B], it[B:])]
    if case == "staged":       # every row referenced at least twice
        uid = rng.permutation(np.repeat(rng.choice(U, B // 2, replace=False), 2))
        pid = rng.choice(I, B, replace=False)
        return [x.astype(np.int32) for x in (uid, pid, rng.permutation(pid))]
    uid, pid, nid = (rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
    uid[1] = uid[2]
    nid[3] = pid[3]
    uid[4], uid[5], pid[6], pid[7], nid[8], nid[9] = -1, U, -3, I, -1, I + 7   # a bad id in every position
    uid[10], pid[10], nid[10] = -1, I, -2
    nid[B - 1] = I                                                              # and in the last triplet
    return uid, pid, nid


class Tables:
    """Device user / item / bias tables and the slot rows optimizer `opt` keeps, all from one seed."""

    def __init__(self, opt, U, I, D, seed, scale=0.05):
        rng = np.random.default_rng(seed)
        self.var = [rng.uniform(-scale, scale, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1))]
        self.opt = opt
        self.t = [dev(a) for a in self.var]
        self.s = []
        for a in self.var:
            if opt == L.ORX_OPT_SGD:
                self.s.append(())
            elif opt == L.ORX_OPT_ADAGRAD:
                self.s.append((dev(np.full_like(a, 0.1)),))
            else:
                self.s.append((dev(np.abs(a) * 0.01), dev(a * a * 0.02 + 1e-4)))
        self.tt = [N.table(t, *s) for t, s in zip(self.t, self.s)]

    def arrays(self):
        return [[t.cpu().numpy()] + [x.cpu().numpy() for x in s] for t, s in zip(self.t, self.s)]


def _step(eng, kind, tabs, dids, optname, prefetch, margin=0.5):
    """One step (prefetched or not) -> (out4, dispatch record)."""
    opt, lr = OPTS[optname]
    eng.debug_dispatch_log()
    if prefetch:
        eng.pairwise_prefetch(tabs.tt[0], tabs.tt[1], *dids, opt, ids_ready=True)
    out = torch.zeros(4, device="cuda")
    eng.pairwise_step(kind, *tabs.tt, *dids, N.opt(opt, lr, step=1), out, margin=margin)
    rec = eng.debug_dispatch_log()
    assert len(rec) == 1, rec
    return out, rec[0]


CASES = ["mixed", "owned", "staged"]


@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("case", CASES)
def test_records_match_oracle(engines, case, optname):
    """The records of a prefetched batch, field by field, at B = 1003 / 517 / 600 (no multiple of 8 or 64 among the
    first two), with bad ids in every position, all-owned and all-staged batches, for every optimizer (ADAM_DENSE
    builds a mode-1 index: every row staged, no owned bits)."""
    eng = engines[True]
    U, I, D = 2000, 3000, 32
    B = {"mixed": 1003, "owned": 517, "staged": 600}[case]
    opt = OPTS[optname][0]
    rng = np.random.default_rng([7, CASES.index(case), opt])
    ids = make_ids(rng, case, U, I, B)
    tabs = Tables(opt, U, I, D, seed=3)
    out, rec = _step(eng, N.ORX_PAIR_BPR, tabs, [dev(x, torch.int32) for x in ids], optname, prefetch=True)
    assert rec.s in (1, 2), rec
    staged = check_records(eng.debug_pair_records(rec.s, B), ids, U, I, opt == L.ORX_OPT_ADAM_DENSE,
                           f"{case} {optname}")
    got = out.cpu().numpy()
    n_bad = sum(int(((x < 0) | (x >= n)).sum()) for x, n in zip(ids, (U, I, I)))
    assert got[2] == n_bad and got[3] == staged, (got, n_bad, staged)
    cu, ci = _counts(ids, U, I)
    if case == "owned" and opt != L.ORX_OPT_ADAM_DENSE:
        assert staged == 0
    if case == "staged":
        assert staged == int((cu > 0).sum() + (ci > 0).sum())


def test_no_records_without_resolve(engines):
    """A handle created with ORX_PAIR_RESOLVE=0 resolves nothing: its prefetched steps probe the index."""
    eng = engines[False]
    U, I, D, B = 500, 700, 32, 64
    ids = make_ids(np.random.default_rng(1), "mixed", U, I, B)
    _, rec = _step(eng, N.ORX_PAIR_BPR, Tables(L.ORX_OPT_ADAGRAD, U, I, D, 4), [dev(x, torch.int32) for x in ids],
                   "adagrad", prefetch=True)
    assert rec.s in (1, 2)
    with pytest.raises(RuntimeError):
        eng.debug_pair_records(rec.s, B)


@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D", [32, 64, 128, 256])
@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_paths_agree(engines, kind, D, optname):
    """The same step three ways from the same tables and ids: prefetched with records, prefetched without
    (ORX_PAIR_RESOLVE=0) and built on the step's stream.  Same dispatch record apart from the index set, same out4;
    tables, slots and bias equal to fp32 summation order (the staging rows' atomics), bit-equal on every row the batch
    references at most once."""
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    U, I, B = 3000, 5000, 1003
    rng = np.random.default_rng([11, D, OPTS[optname][0], k])
    ids = make_ids(rng, "mixed", U, I, B)
    dids = [dev(x, torch.int32) for x in ids]
    scale = 0.05 if kind == "bpr" else 0.4
    runs = []
    for eng, pf in ((engines[True], True), (engines[False], True), (engines[True], False)):
        tabs = Tables(OPTS[optname][0], U, I, D, seed=5, scale=scale)
        out, rec = _step(eng, k, tabs, dids, optname, prefetch=pf)
        runs.append((out.cpu().numpy(), rec, tabs.arrays()))
    (o0, r0, t0) = runs[0]
    assert r0.s in (1, 2) and runs[1][1].s in (1, 2) and runs[2][1].s == 0, [r for _, r, _ in runs]
    cu, ci = _counts(ids, U, I)
    once = (cu <= 1, ci <= 1, ci <= 1)
    for o, r, t in runs[1:]:
        assert r._replace(s=0) == r0._replace(s=0), (r, r0)
        np.testing.assert_array_equal(o, o0)
        for name, a, b, m in zip(("user", "item", "bias"), t, t0, once):
            for j, (x, y) in enumerate(zip(a, b)):
                what = f"{kind} D={D} {optname} {name} slot {j}"
                np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-6, err_msg=what)
                np.testing.assert_array_equal(x[m], y[m], err_msg=what + " (rows seen at most once)")


def test_lifecycle(engines):
    """Consecutive prefetched steps alternate sets 1 / 2 and each set's records stay those of its batch until the set is
    reused; an unconsumed prefetch is dropped (the step after it builds its own index, set 0) and the alternation goes
    on after it; orx_pairwise_step_host resolves its own uploads the same way."""
    eng = engines[True]
    U, I, D, B = 3000, 5000, 64, 777
    rng = np.random.default_rng(21)
    tabs = Tables(L.ORX_OPT_ADAGRAD, U, I, D, seed=6)
    opt = N.opt(L.ORX_OPT_ADAGRAD, 0.05)
    batches = [make_ids(rng, "mixed", U, I, B) for _ in range(6)]
    dids = [[dev(x, torch.int32) for x in b] for b in batches]
    out = torch.zeros(4, device="cuda")

    def step(i, prefetch_next=None):
        eng.pairwise_step(N.ORX_PAIR_BPR, *tabs.tt, *dids[i], opt, out)
        rec = eng.debug_dispatch_log()
        assert len(rec) == 1 and rec[0].op == PAIR_OP, rec
        if prefetch_next is not None:
            eng.pairwise_prefetch(tabs.tt[0], tabs.tt[1], *dids[prefetch_next], opt.kind, ids_ready=True)
        return rec[0].s

    def records_are(s, i):
        check_records(eng.debug_pair_records(s, B), batches[i], U, I, False, f"set {s} batch {i}")

    eng.debug_dispatch_log()
    eng.pairwise_prefetch(tabs.tt[0], tabs.tt[1], *dids[0], opt.kind, ids_ready=True)
    a = step(0, prefetch_next=1)
    b = step(1, prefetch_next=2)                 # batch 2's prefetch goes to set a and is never consumed
    assert {a, b} == {1, 2}, (a, b)
    records_are(b, 1)
    assert step(3) == 0                          # other ids: the dangling prefetch is dropped, the index built here
    eng.pairwise_prefetch(tabs.tt[0], tabs.tt[1], *dids[4], opt.kind, ids_ready=True)
    assert step(4, prefetch_next=5) == b         # the set after the dropped one
    records_are(b, 4)
    assert step(5) == a
    records_are(a, 5)
    records_are(b, 4)                            # still intact: nothing has been prefetched into b since
    torch.cuda.synchronize()

    host = [make_ids(rng, "mixed", U, I, B) for _ in range(2)]
    sets = []
    for h in host:
        pinned = [torch.from_numpy(x).pin_memory() for x in h]
        out_h = torch.zeros(4).pin_memory()
        eng.pairwise_step_host(N.ORX_PAIR_BPR, *tabs.tt, *pinned, opt, out_h)
        rec = eng.debug_dispatch_log()
        assert len(rec) == 1 and rec[0].s in (1, 2), rec
        sets.append(rec[0].s)
        staged = check_records(eng.debug_pair_records(rec[0].s, B), h, U, I, False, f"host set {rec[0].s}")
        torch.cuda.synchronize()
        assert out_h[3].item() == staged
    assert sets[0] != sets[1], sets
