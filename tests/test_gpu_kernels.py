"""GPU parity: every liborx entry point vs the oracle, through the C-ABI (ctypes).
Bar: indices bit-exact (out-of-range / duplicate handling), loss / gradients / updated rows
within 1e-5 (fp32) of the oracle evaluated in float64 on identical weights and ids."""
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

ATOL = 1e-5
OPTS = {"sgd": (0, 0.05), "adagrad": (1, 0.05), "adam_lazy": (2, 0.01), "adam_dense": (3, 0.01)}
LAZY, DENSE = L.ORX_OPT_ADAM_LAZY, L.ORX_OPT_ADAM_DENSE
PAIR_OP, POINT_OP = L.ORX_OP_PAIRWISE_STEP, L.ORX_OP_POINTWISE_STEP
SPECIAL_D = (32, 64, 128, 256)     # the dims with a specialised k_pair_step / k_point_step


# ---- dispatch of the sparse steps --------------------------------------------------------------------------------
# Every pairwise / pointwise step a test runs asserts its dispatch record {op, variant, kind, optimizer, B, D, MINB,
# index set} against the rule below (orx_pairwise.cu launch_pair_step_kind_opt, orx_pointwise.cu launch_point_kind_opt).
def _pair_rule(D, opt):
    """(variant, CTAs/SM bound) of the fused pairwise kernel: lazy Adam (nine rows per triplet) never double-buffers,
    D = 128 runs one register buffer at 4 CTAs/SM (3 for lazy Adam), the other specialised dims 2 CTAs/SM."""
    if D == 128:
        return L.ORX_VARIANT_STEP, 3 if opt == LAZY else 4
    if D in SPECIAL_D:
        return (L.ORX_VARIANT_STEP if opt == LAZY else L.ORX_VARIANT_STEP_PIPE), 2
    return L.ORX_VARIANT_STEP_GENERIC, 0


def _point_rule(D):
    return (L.ORX_VARIANT_STEP if D in SPECIAL_D else L.ORX_VARIANT_STEP_GENERIC), 0


def _check_step_dispatch(eng, op, kind, opt, B, D, index_set=0):
    """Asserts the one record of the step just launched; index_set "prefetch" accepts set 1 or 2.  -> the set."""
    v, minb = _pair_rule(D, opt) if op == PAIR_OP else _point_rule(D)
    got = eng.debug_dispatch_log()
    assert len(got) == 1, got
    want = N.Dispatch(op, v, kind, opt, B, D, minb, got[0].s if index_set == "prefetch" else index_set)
    assert got[0] == want, (got[0], want)
    if index_set == "prefetch":
        assert got[0].s in (1, 2), got[0]
    return got[0].s


def _staged(opt, *sides):
    """Rows the batch index gives a staging slot (out4[3]): every unique row of a side under ADAM_DENSE, else the rows
    referenced more than once.  `sides` hold the ids of the VALID samples only."""
    n = 0
    for ids in sides:
        c = np.unique(ids, return_counts=True)[1]
        n += len(c) if opt == DENSE else int((c > 1).sum())
    return n


@pytest.fixture(scope="module")
def eng():
    from openrec_b200 import native
    return native.engine()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())   # hash() is randomised per process


def avoid_hinge_ties(rng, user, item, bias, uid, pid, nid, margin=0.5, tol=1e-3):
    """UCML's hinge is discontinuous in its gradient: a triplet with |h| ~ 1e-7 may be active in
    float32 and inactive in float64.  Parity is only defined away from the kink, so resample the
    negatives of such triplets (the reference has the same measure-zero ambiguity)."""
    for _ in range(20):
        u, p, n = user[uid], item[pid], item[nid]
        h = margin - ((-((u - p) ** 2).sum(1) + bias[pid, 0]) - (-((u - n) ** 2).sum(1) + bias[nid, 0]))
        bad = np.abs(h) < tol
        if not bad.any():
            return nid
        nid = nid.copy()
        nid[bad] = rng.integers(0, len(item), bad.sum())
    raise AssertionError("could not avoid hinge ties")


def make_problem(rng, U, I, D, B, scale=0.05):
    user = rng.uniform(-scale, scale, (U, D))
    item = rng.uniform(-scale, scale, (I, D))
    bias = rng.uniform(-scale, scale, (I, 1))
    uid = rng.integers(0, U, B).astype(np.int32)
    pid = rng.integers(0, I, B).astype(np.int32)
    nid = rng.integers(0, I, B).astype(np.int32)
    if B >= 4:
        nid[1] = pid[1]   # same item as positive and negative of one triplet
        uid[2] = uid[3]   # guaranteed duplicate user
    return user, item, bias, uid, pid, nid


def slots(opt_kind, *arrs):
    """float64 oracle state + device tensors for the given optimizer."""
    st, dv = {}, {}
    for name, a in arrs:
        if opt_kind == 0:
            st[name], dv[name] = (None, None), (None, None)
        elif opt_kind == 1:
            s0 = np.full_like(a, 0.1)
            st[name], dv[name] = (s0, None), (dev(s0), None)
        else:
            s0, s1 = np.abs(a) * 0.01, a * a * 0.02 + 1e-4   # non-trivial m, v
            st[name], dv[name] = (s0.copy(), s1.copy()), (dev(s0), dev(s1))
    return st, dv


def close(t, ref, atol=ATOL, rtol=1e-5, what=""):
    got = t.detach().cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(got, np.asarray(ref, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol,
                               err_msg=what)


# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_pairwise_golden_fwd_grad(eng, golden_dir, kind):
    from openrec_b200 import native as N
    g = dict(np.load(os.path.join(golden_dir, f"pairwise_{kind}.npz")))
    tu, ti, tb = dev(g["user"]), dev(g["item"]), dev(g["bias"])
    U, D = g["user"].shape
    B = len(g["uid"])
    uid, pid, nid = dev(g["uid"], torch.int32), dev(g["pid"], torch.int32), dev(g["nid"], torch.int32)
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    out4 = torch.zeros(4, device="cuda")
    eng.pairwise_fwd(k, N.table(tu), N.table(ti), N.table(tb), uid, pid, nid, out4, margin=0.5)
    close(out4[0], g["loss"], what="loss")
    close(out4[1], g["l2"], what="l2")
    du, dp, dn = (torch.empty(B, D, device="cuda") for _ in range(3))
    dbp, dbn = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    eng.pairwise_grad(k, N.table(tu), N.table(ti), N.table(tb), uid, pid, nid, 0.5, 1.0, 1.0, d_user=du, d_pos=dp,
                      d_neg=dn, d_bp=dbp, d_bn=dbn)
    dense_u = torch.zeros_like(tu).index_add_(0, uid.long(), du)
    dense_i = torch.zeros_like(ti).index_add_(0, pid.long(), dp).index_add_(0, nid.long(), dn)
    dense_b = torch.zeros(len(g["bias"]), device="cuda").index_add_(0, pid.long(), dbp).index_add_(0, nid.long(), dbn)
    tol = 2e-4 if kind == "ucml" else ATOL   # the ucml fixture scales embeddings x8 (values ~O(10))
    close(dense_u, g["g_user"], atol=tol, what="g_user")
    close(dense_i, g["g_item"], atol=tol, what="g_item")
    close(dense_b, g["g_bias"], atol=tol, what="g_bias")


def _ids(rng, mode, U, I, B):
    """One pairwise batch.  "owned": every row referenced once (U >= B, I >= 2B); "staged": every row referenced at
    least twice (B >= 2); "mixed": uniform ids."""
    if mode == "owned":
        items = rng.permutation(I)[:2 * B]
        ids = rng.permutation(U)[:B], items[:B], items[B:]
    elif mode == "staged":
        users = np.resize(rng.permutation(U)[:max(1, B // 2)], B)
        items = np.resize(rng.permutation(I)[:B], 2 * B)
        rng.shuffle(users), rng.shuffle(items)
        ids = users, items[:B], items[B:]
    else:
        ids = rng.integers(0, U, B), rng.integers(0, I, B), rng.integers(0, I, B)
    return tuple(np.asarray(x, np.int32) for x in ids)


BIG = 2 ** 31 - 1


def _bad_pair_ids(rng, U, I, B):
    """Uniform triplets over all but the last two rows of each table, then bad ids (-1, the row count, 2^31-1) in uid,
    pid and nid, one triplet with two of them, one in the last (partial) warp of the batch, and
      (a) user U-1 and item I-1 referenced by one skipped and by one valid triplet;
      (b) user U-2 and item I-2 (and so its bias) referenced twice, only by skipped triplets."""
    uid, pid, nid = (np.asarray(rng.integers(0, n - 2, B), np.int32) for n in (U, I, I))
    uid[0], pid[0], nid[0] = U - 1, I - 1, -1          # (a)
    uid[1], pid[1] = U - 1, I - 1
    uid[2], pid[2], nid[2] = U - 2, I - 2, I           # (b)
    uid[3], pid[3], nid[3] = U - 2, BIG, I - 2
    uid[4], uid[5], pid[6], nid[7] = -1, U, -1, BIG
    uid[8], pid[8] = BIG, I
    nid[B - 1] = -1
    return uid, pid, nid


class PairProb:
    """One pairwise problem: device tables + optimizer slots and their float64 oracle twins (from the float32-rounded
    device values).  run() launches one step and checks its dispatch record; verify() runs the oracle on the valid
    triplets and checks out4, and the tables and every slot.  It runs the default constants (margin 0.5, c_l2 1, Keras
    betas / eps) under the value bar; cases with other constants, slot initialisations and tie tables, judged by their
    per-element updates, are built in tests/step_bar.py (plain numpy, shared with the CPU proof of that bar)."""

    def __init__(self, kind, optname, D, U, I, seed, scale=None):
        self.kind, self.optname, self.D, self.U, self.I = kind, optname, D, U, I
        self.opt, self.lr = OPTS[optname]
        self.k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
        rng = np.random.default_rng(seed)
        sc = scale or (0.05 if kind == "bpr" else 0.4)
        arrs = [rng.uniform(-sc, sc, s) for s in ((U, D), (I, D), (I, 1))]
        st, self.dv = slots(self.opt, *zip(("user", "item", "bias"), arrs))
        self.tabs = [dev(a) for a in arrs]
        self.ref = [t.cpu().numpy().astype(np.float64) for t in self.tabs]
        self.st = {k: tuple(None if s is None else dev(s).cpu().numpy().astype(np.float64) for s in v)
                   for k, v in st.items()}
        self.tt = [N.table(t, *self.dv[n]) for t, n in zip(self.tabs, ("user", "item", "bias"))]
        self.n = 0
        self.pinned = []

    def valid(self, uid, pid, nid):
        return (uid >= 0) & (uid < self.U) & (pid >= 0) & (pid < self.I) & (nid >= 0) & (nid < self.I)

    def ties(self, uid, pid, nid, tol=1e-3):
        """UCML's hinge has a kink: a valid triplet with |h| < tol may be active in float32 and not in float64."""
        if self.kind != "ucml":
            return False
        ok = self.valid(uid, pid, nid)
        user, item, bias = self.ref
        u, p, n, bp, bn = user[uid[ok]], item[pid[ok]], item[nid[ok]], bias[pid[ok], 0], bias[nid[ok], 0]
        h = 0.5 - ((-((u - p) ** 2).sum(1) + bp) - (-((u - n) ** 2).sum(1) + bn))
        return bool((np.abs(h) < tol).any())

    def draw(self, rng, make):
        """make(rng) -> ids, redrawn while a UCML triplet sits on the hinge's kink."""
        for _ in range(50):
            ids = make(rng)
            if not self.ties(*ids):
                return ids
        raise AssertionError("could not avoid hinge ties")

    def run(self, eng, ids, dids=None, index_set=0, host=False):
        """-> (out4 tensor, step number, index set the record shows)."""
        self.n += 1
        o = N.opt(self.opt, self.lr, step=self.n)
        eng.debug_dispatch_log()
        if host:   # the pinned ids must outlive the asynchronous upload: they are kept until verify() synchronises
            out = torch.zeros(4).pin_memory()
            self.pinned.append([torch.from_numpy(x).pin_memory() for x in ids])
            eng.pairwise_step_host(self.k, *self.tt, *self.pinned[-1], o, out)
        else:
            out = torch.zeros(4, device="cuda")
            eng.pairwise_step(self.k, *self.tt, *(dids or [dev(x, torch.int32) for x in ids]), o, out, margin=0.5)
        s = _check_step_dispatch(eng, PAIR_OP, self.k, self.opt, len(ids[0]), self.D, index_set)
        return out, self.n, s

    def verify(self, out, ids, n, tables=True, what=""):
        torch.cuda.synchronize()
        self.pinned = []
        uid, pid, nid = ids
        ok = self.valid(*ids)
        frac = ok.sum() / len(uid) if self.kind == "bpr" else 1.0   # BPR's 1/B is over the submitted batch
        loss, l2 = O.pairwise_train_step(self.kind, *self.ref, uid[ok], pid[ok], nid[ok], self.opt, self.st, n, self.lr,
                                         margin=0.5, c_loss=frac)
        got = out.cpu().numpy().astype(np.float64)
        what = f"{self.kind} {self.optname} D={self.D} B={len(uid)} step {n} {what}"
        np.testing.assert_allclose(got[0], loss * frac, rtol=2e-5, atol=ATOL, err_msg=f"loss {what}")
        np.testing.assert_allclose(got[1], l2, rtol=2e-5, atol=ATOL, err_msg=f"l2 {what}")
        n_bad = sum(int(((x < 0) | (x >= r)).sum()) for x, r in ((uid, self.U), (pid, self.I), (nid, self.I)))
        assert got[2] == n_bad, (what, got[2], n_bad)
        if tables:
            self.check_tables(what)
        assert got[3] == _staged(self.opt, uid[ok], np.concatenate([pid[ok], nid[ok]])), (what, got[3])
        return got

    def check_tables(self, what=""):
        for t, r, name in zip(self.tabs, self.ref, ("user", "item", "bias")):
            close(t, r, what=f"{name} {what}")
            for j in (0, 1):
                if self.st[name][j] is not None:
                    close(self.dv[name][j], self.st[name][j], what=f"{name} slot{j} {what}")

    def step(self, eng, ids, **kw):
        out, n, s = self.run(eng, ids, **kw)
        return self.verify(out, ids, n), s


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D,U,I,B", [(1, 40, 60, 100), (12, 37, 53, 96), (50, 300, 500, 257), (260, 300, 500, 203),
                                     (32, 64, 64, 200), (32, 300, 2000, 203), (64, 2000, 3000, 1000),
                                     (128, 5000, 9000, 4096), (256, 500, 700, 333)])
def test_pairwise_step(eng, kind, optname, D, U, I, B):
    """Three steps of uniform batches (workspace, hash and staging must be clean between steps).  D = 32: 64 x 64 rows
    (nearly every row staged) and 300 x 2000 rows (owned users and items occur); D = 1 / 12 / 50 / 260 run the generic
    kernel and the scalar and >32-float4 paths of the tail."""
    rng = np.random.default_rng(seed_of(kind, optname, D, U))
    p = PairProb(kind, optname, D, U, I, seed_of("tabs", kind, optname, D, U))

    def make(r):
        ids = _ids(r, "mixed", U, I, B)
        ids[2][1] = ids[1][1]   # same item as positive and negative of one triplet
        ids[0][2] = ids[0][3]   # a duplicated user
        return ids

    for _ in range(3):
        p.step(eng, p.draw(rng, make))


TAIL_B = (1, 3, 201, 237, 391)   # a batch smaller than one warp's 8 triplets; B % 8 = 1, 5, 7 with B % 64 != 0


@pytest.mark.parametrize("D", SPECIAL_D)
@pytest.mark.parametrize("B", TAIL_B)
def test_pairwise_batch_tails(eng, D, B):
    """Partial warps and blocks on every specialised kernel: the bench kernel (BPR Adagrad) and UCML lazy Adam (the
    single-buffer variant at D != 128), three steps each."""
    for kind, optname in (("bpr", "adagrad"), ("ucml", "adam_lazy")):
        rng = np.random.default_rng(seed_of("tail", kind, D, B))
        U, I = max(4, B // 2), max(6, B)             # about half of the rows referenced more than once
        p = PairProb(kind, optname, D, U, I, seed_of("tail-tabs", kind, D, B))
        for _ in range(3):
            p.step(eng, p.draw(rng, lambda r: _ids(r, "mixed", U, I, B)))


ALL_D = (1, 7, 32, 64, 128, 256, 260)


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("mode", ["owned", "staged"])
def test_pairwise_ownership_extremes(eng, kind, optname, mode):
    """All rows owned by their triplet (optimizer in registers, no staging: out4[3] = 0, or every unique row under
    ADAM_DENSE) and all rows staged (out4[3] = every unique row), on every kernel variant, three steps each."""
    for D in ALL_D:
        B = 203 if D in (7, 260) else 200
        U, I = (B + 57, 2 * B + 91) if mode == "owned" else (3 * B, 5 * B)
        rng = np.random.default_rng(seed_of("own", kind, optname, mode, D))
        p = PairProb(kind, optname, D, U, I, seed_of("own-tabs", kind, optname, mode, D))
        for _ in range(3):
            uid, pid, nid = ids = p.draw(rng, lambda r: _ids(r, mode, U, I, B))
            got, _ = p.step(eng, ids)
            unique = len(np.unique(uid)) + len(np.unique(np.concatenate([pid, nid])))
            if mode == "owned":
                assert unique == 3 * B and got[3] == (unique if p.opt == DENSE else 0), (D, got)
            else:
                assert got[3] == unique, (D, got, unique)


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
@pytest.mark.parametrize("optname", list(OPTS))
def test_pairwise_bad_ids(eng, kind, optname):
    """Bad ids on every kernel variant: counted one by one in out4[2], their triplets skipped, BPR's 1/B kept over the
    submitted batch; a row referenced only by skipped triplets is not touched (under lazy Adam an optimizer step with
    g = 0 would still move it), nor staged."""
    for D in (13, 32, 64, 128, 256):
        B = 203
        U, I = 150, 400
        rng = np.random.default_rng(seed_of("bad", kind, optname, D))
        p = PairProb(kind, optname, D, U, I, seed_of("bad-tabs", kind, optname, D))
        for _ in range(3):
            p.step(eng, p.draw(rng, lambda r: _bad_pair_ids(r, U, I, B)))


def test_pairwise_weighted_objective_and_bad_ids(eng):
    """tape.gradient(loss + 0.25*l2) and out-of-range ids (counted, triplet skipped)."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(5)
    U, I, D, B = 100, 150, 64, 300
    user, item, bias, uid, pid, nid = make_problem(rng, U, I, D, B)
    tu, ti, tb = dev(user), dev(item), dev(bias)
    user, item, bias = (t.cpu().numpy().astype(np.float64) for t in (tu, ti, tb))
    bad = uid.copy()
    bad[7], bad[9] = U + 3, -1
    out4 = torch.zeros(4, device="cuda")
    eng.debug_dispatch_log()
    eng.pairwise_step(N.ORX_PAIR_BPR, N.table(tu), N.table(ti), N.table(tb), dev(bad, torch.int32),
                      dev(pid, torch.int32), dev(nid, torch.int32), N.opt(0, 0.1), out4, c_loss=2.0, c_l2=0.25)
    _check_step_dispatch(eng, PAIR_OP, N.ORX_PAIR_BPR, 0, B, D)
    assert out4[2].item() == 2
    keep = np.ones(B, bool)
    keep[[7, 9]] = False
    gr = O.bpr_grads(user, item, bias, uid[keep], pid[keep], nid[keep], c_loss=2.0 * keep.sum() / B, c_l2=0.25)
    for var, name in ((user, "user"), (item, "item"), (bias, "bias")):
        idx, val = gr[name]
        O.sgd_sparse(var, idx, val.reshape(len(idx), -1), 0.1)
    close(tu, user), close(ti, item), close(tb, bias)


def test_pairwise_step_host_buffers(eng):
    from openrec_b200 import native as N
    rng = np.random.default_rng(6)
    U, I, D, B = 400, 600, 128, 1024
    user, item, bias, uid, pid, nid = make_problem(rng, U, I, D, B)
    tu, ti, tb = dev(user), dev(item), dev(bias)
    au, ai, ab = (torch.full_like(t, 0.1) for t in (tu, ti, tb))
    user, item, bias = (t.cpu().numpy().astype(np.float64) for t in (tu, ti, tb))
    st = {k: (np.full_like(v, 0.1), None) for k, v in (("user", user), ("item", item), ("bias", bias))}
    hu, hp, hn = (torch.from_numpy(x).pin_memory() for x in (uid, pid, nid))
    out_h = torch.zeros(4).pin_memory()
    eng.debug_dispatch_log()
    eng.pairwise_step_host(N.ORX_PAIR_BPR, N.table(tu, au), N.table(ti, ai), N.table(tb, ab), hu, hp, hn,
                           N.opt(1, 0.05), out_h)
    _check_step_dispatch(eng, PAIR_OP, N.ORX_PAIR_BPR, 1, B, D, "prefetch")
    torch.cuda.synchronize()
    loss, l2 = O.pairwise_train_step("bpr", user, item, bias, uid, pid, nid, 1, st, 1, 0.05)
    np.testing.assert_allclose(out_h[0].item(), loss, rtol=2e-5)
    np.testing.assert_allclose(out_h[1].item(), l2, rtol=2e-5)
    close(tu, user), close(ti, item), close(tb, bias), close(ai, st["item"][0])


def _adagrad_problem(rng, U, I, D):
    user, item, bias = (rng.uniform(-0.05, 0.05, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1)))
    tabs = [dev(a) for a in (user, item, bias)]
    accs = [torch.full_like(t, 0.1) for t in tabs]
    ref = [a.astype(np.float64) for a in (user, item, bias)]
    st = {k: (np.full_like(v, 0.1), None) for k, v in zip(("user", "item", "bias"), ref)}
    return tabs, accs, ref, st


# (kind, optimizer) of the prefetch / host-path tests beyond BPR Adagrad.  UCML runs at scale 0.05 there: its hinge then
# sits far from the kink for every triplet (h ~ 0.5 +- 0.06), since the ids of a pipelined sequence are fixed before the
# tables move.
PIPE_CASES = [("ucml", "sgd"), ("bpr", "adam_dense"), ("ucml", "adam_lazy")]


def test_pairwise_step_host_runs_ahead(eng):
    """Eight host-buffer steps enqueued back to back (no sync in between): the id upload and the index build of step t
    run on the side stream under step t-1; staging buffers and index sets alternate and must not be reused early.
    Every step consumes its side-stream index (set 1 or 2, alternating).  BPR Adagrad, the bench configuration."""
    _host_runs_ahead(eng, "bpr", "adagrad")


@pytest.mark.parametrize("kind,optname", PIPE_CASES)
def test_pairwise_step_host_runs_ahead_kinds(eng, kind, optname):
    """test_pairwise_step_host_runs_ahead for UCML and the other optimizers, ADAM_DENSE (mode-1 index) included."""
    _host_runs_ahead(eng, kind, optname)


def _host_runs_ahead(eng, kind, optname):
    rng = np.random.default_rng(seed_of("host", kind, optname))
    U, I, D, B = 700, 900, 128, 4096            # few rows: most lookups are duplicates (staging + tail every step)
    p = PairProb(kind, optname, D, U, I, seed_of("host-tabs", kind, optname), scale=0.05)
    ids = [_ids(rng, "mixed", U, I, B) for _ in range(8)]
    runs = [p.run(eng, x, host=True, index_set="prefetch") for x in ids]
    assert all(a[2] != b[2] for a, b in zip(runs, runs[1:])), [r[2] for r in runs]
    for x, (out, n, _) in zip(ids, runs):
        p.verify(out, x, n, tables=False)
    p.check_tables()


def test_pairwise_prefetch_pipeline(eng):
    """orx_pairwise_prefetch: the index of batch i+1 is built on the side stream while step i runs; a prefetch nobody
    consumes (different ids) is dropped; results equal the plain sequence of steps.  The dispatch record shows the
    consumed prefetch's set (1 or 2) and set 0 for the step after the dropped one.  BPR Adagrad."""
    _prefetch_pipeline(eng, "bpr", "adagrad")


@pytest.mark.parametrize("kind,optname", PIPE_CASES)
def test_pairwise_prefetch_pipeline_kinds(eng, kind, optname):
    """test_pairwise_prefetch_pipeline for UCML and the other optimizers, ADAM_DENSE (mode-1 index) included."""
    _prefetch_pipeline(eng, kind, optname)


def _prefetch_pipeline(eng, kind, optname):
    rng = np.random.default_rng(seed_of("pf", kind, optname))
    U, I, D, B = 600, 800, 128, 2048
    p = PairProb(kind, optname, D, U, I, seed_of("pf-tabs", kind, optname), scale=0.05)
    ids = [_ids(rng, "mixed", U, I, B) for _ in range(6)]
    dids = [[dev(x, torch.int32) for x in b] for b in ids]
    torch.cuda.synchronize()                         # the id tensors are complete: ids_ready=True below is honest
    eng.pairwise_prefetch(p.tt[0], p.tt[1], *dids[0], p.opt, ids_ready=True)
    runs = []
    for k in range(6):
        # consumes the index prefetched for batch k, except k == 3: the prefetch issued at k == 2 is for batch 0
        runs.append(p.run(eng, ids[k], dids=dids[k], index_set=0 if k == 3 else "prefetch"))
        nxt = dids[(k + 1) % 6] if k != 2 else dids[0]                    # k == 2: nobody consumes this one -> dropped
        eng.pairwise_prefetch(p.tt[0], p.tt[1], *nxt, p.opt, ids_ready=(k % 2 == 0))
    assert runs[0][2] != runs[1][2] and runs[1][2] != runs[2][2] and runs[4][2] != runs[5][2]
    for x, (out, n, _) in zip(ids, runs):
        p.verify(out, x, n, tables=False)
    p.check_tables()
    # the dangling prefetch (batch 0) is dropped by the next call that builds its own index
    p.step(eng, ids[3], dids=dids[3])


def test_pairwise_prefetch_mode_mismatch(eng):
    """A prefetch built for mode 0 (rows staged when seen twice) must not serve an ADAM_DENSE step (mode 1: every row
    staged), nor the reverse: such a step builds its own index (set 0) and still matches the oracle.  Lazy and dense
    Adam share the m / v slots, so one problem runs both."""
    rng = np.random.default_rng(19)
    U, I, D, B = 300, 500, 64, 777
    for kind in ("bpr", "ucml"):
        p = PairProb(kind, "adam_lazy", D, U, I, seed_of("mm", kind), scale=0.05)
        for pf_opt, step_opt, want in ((LAZY, DENSE, 0), (DENSE, LAZY, 0), (LAZY, LAZY, "prefetch"),
                                       (DENSE, DENSE, "prefetch")):
            ids = _ids(rng, "mixed", U, I, B)
            dids = [dev(x, torch.int32) for x in ids]
            torch.cuda.synchronize()
            eng.pairwise_prefetch(p.tt[0], p.tt[1], *dids, pf_opt, ids_ready=True)
            p.opt, p.optname = step_opt, f"prefetch {pf_opt} step {step_opt}"
            p.step(eng, ids, dids=dids, index_set=want)


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
@pytest.mark.parametrize("optname", list(OPTS))
def test_pairwise_prefetch_every_variant(eng, kind, optname):
    """Each kernel variant consumes a prefetched index from both prefetch sets, then a plain step (set 0) follows."""
    for D in (32, 64, 128, 256, 50):
        rng = np.random.default_rng(seed_of("pfv", kind, optname, D))
        U, I, B = 120, 250, 333
        p = PairProb(kind, optname, D, U, I, seed_of("pfv-tabs", kind, optname, D), scale=0.05)
        sets = []
        for k in range(3):
            ids = _ids(rng, "mixed", U, I, B)
            dids = [dev(x, torch.int32) for x in ids]
            if k < 2:
                torch.cuda.synchronize()
                eng.pairwise_prefetch(p.tt[0], p.tt[1], *dids, p.opt, ids_ready=True)
            sets.append(p.step(eng, ids, dids=dids, index_set="prefetch" if k < 2 else 0)[1])
        assert sorted(sets[:2]) == [1, 2], sets


def test_epoch_wrap():
    """The batch-index epoch has 31 bits: starting just below 2^31 the counter wraps, the hash tables are emptied and
    duplicates are still detected (a stale epoch compare would turn every step into hogwild updates)."""
    from openrec_b200 import native as N
    e = N.Engine(0)
    try:
        rng = np.random.default_rng(18)
        U, I, D, B = 50, 70, 64, 512               # every row is hit many times
        tabs, accs, ref, st = _adagrad_problem(rng, U, I, D)
        tt = [N.table(t, a) for t, a in zip(tabs, accs)]
        out4 = torch.zeros(4, device="cuda")
        ids0 = [rng.integers(0, n, B).astype(np.int32) for n in (U, I, I)]
        e.pairwise_step(N.ORX_PAIR_BPR, *tt, *[dev(x, torch.int32) for x in ids0], N.opt(1, 0.05), out4)   # allocates
        O.pairwise_train_step("bpr", *ref, *ids0, 1, st, 1, 0.05)
        e.debug_set_epoch(2 ** 31 - 3)
        e.debug_dispatch_log()
        for k in range(5):                           # epochs 2^31-2, 2^31-1, wrap -> 1, 2, 3
            ids = [rng.integers(0, n, B).astype(np.int32) for n in (U, I, I)]
            e.pairwise_step(N.ORX_PAIR_BPR, *tt, *[dev(x, torch.int32) for x in ids], N.opt(1, 0.05), out4)
            _check_step_dispatch(e, PAIR_OP, N.ORX_PAIR_BPR, 1, B, D)
            loss, l2 = O.pairwise_train_step("bpr", *ref, *ids, 1, st, k + 2, 0.05)
            np.testing.assert_allclose(out4[0].item(), loss, rtol=2e-5)
        for t, r in zip(tabs, ref):
            close(t, r)
    finally:
        e.close()


@pytest.mark.parametrize("case", ["prefetch", "host", "set0_under_prefetch", "apply_censor"])
def test_epoch_wrap_per_set(case):
    """Every index table takes its own epoch, and a wrap empties only that table, on the stream that builds into it.
    Every table starts 3 below 2^31 (its third build wraps), with few rows so that every row is hit many times:
      prefetch            -- prefetched steps, sets 1 and 2 alternating, each set wrapping;
      host                -- orx_pairwise_step_host run ahead, its side-stream sets wrapping under the previous step;
      set0_under_prefetch -- set 0 wraps under pointwise steps and censors while a prefetch is outstanding, and the
                             pairwise step then consumes that prefetch;
      apply_censor        -- orx_sparse_apply_strided and orx_censor, which use set 0's user table only.
    Each step matches the oracle, with its dispatch record."""
    e = N.Engine(0)
    try:
        rng = np.random.default_rng(seed_of("wrap", case))
        U, I, D, B = 50, 70, 64, 512
        if case == "apply_censor":
            ok, lr = OPTS["adagrad"]
            var = rng.uniform(-0.3, 0.3, (U, D))
            st, dv = slots(ok, ("v", var))
            tv = dev(var)
            var, s0 = tv.cpu().numpy().astype(np.float64), dv["v"][0].cpu().numpy().astype(np.float64)
            tc = dev(rng.uniform(-0.3, 0.3, (U, D)))
            cref = tc.cpu().numpy().astype(np.float64)
            for k in range(5):                       # the user table's epochs: k = 0 allocates, then 2^31-2 ... wrap
                ids = rng.integers(0, U, B).astype(np.int32)
                vals = rng.standard_normal((B, 2, D)).astype(np.float32)
                e.sparse_apply_strided(N.table(tv, dv["v"][0]), dev(np.stack([ids, ids[::-1]], 1), torch.int32), 1,
                                       dev(vals), N.opt(ok, lr, step=k + 1))
                O.apply_sparse(ok, var, s0, None, ids[::-1], vals[:, 1].astype(np.float64), k + 1, lr)
                e.censor(tc, dev(ids, torch.int32))
                O.censor(cref, ids)
                close(tv, var, atol=2e-5, what=f"sparse apply {k}")
                close(dv["v"][0], s0, atol=2e-5, what=f"accumulator {k}")
                close(tc, cref, what=f"censor {k}")
                if k == 0:
                    e.debug_set_epoch(2 ** 31 - 3)
            return
        p = PairProb("bpr", "adagrad", D, U, I, seed_of("wrap-tabs", case), scale=0.05)
        p.step(e, _ids(rng, "mixed", U, I, B))       # allocates the workspace (epochs restart there)
        e.debug_set_epoch(2 ** 31 - 3)
        ids = [_ids(rng, "mixed", U, I, B) for _ in range(8)]
        if case == "host":
            runs = [p.run(e, x, host=True, index_set="prefetch") for x in ids]
            for x, (out, n, _) in zip(ids, runs):
                p.verify(out, x, n, tables=False)
            p.check_tables()
            sets = [r[2] for r in runs]
        else:
            if case == "set0_under_prefetch":
                q = PointProb("gmf", "adagrad", D, U, I, seed_of("wrap-point"))
                tc = dev(rng.uniform(-0.3, 0.3, (U, D)))
                cref = tc.cpu().numpy().astype(np.float64)
            sets = []
            for x in ids:
                dids = [dev(a, torch.int32) for a in x]
                torch.cuda.synchronize()             # the id tensors are complete: ids_ready=True is honest
                e.pairwise_prefetch(p.tt[0], p.tt[1], *dids, p.opt, ids_ready=True)
                if case == "set0_under_prefetch":    # set 0: two user-table and one item-table epochs per batch
                    q.step(e, _point_ids(rng, "mixed", U, I, B), (rng.random(B) < 0.4).astype(np.float32))
                    e.censor(tc, dids[0])
                    O.censor(cref, x[0])
                    close(tc, cref, what="censor")
                sets.append(p.step(e, x, dids=dids, index_set="prefetch")[1])
        assert all(a != b for a, b in zip(sets, sets[1:])), sets   # sets 1 and 2 alternate
    finally:
        e.close()


# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
def test_pointwise_golden_fwd_grad(eng, golden_dir, kind):
    from openrec_b200 import native as N
    g = dict(np.load(os.path.join(golden_dir, f"pointwise_{kind}.npz")))
    tu, ti, tb = dev(g["user"]), dev(g["item"]), dev(g["bias"])
    B, D = len(g["uid"]), g["user"].shape[1]
    uid, iid, lab = dev(g["uid"], torch.int32), dev(g["iid"], torch.int32), dev(g["label"])
    k = N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF
    w = dev(g["w"].reshape(1, -1)) if kind == "gmf" else None
    wt = N.table(w) if w is not None else None
    a, b = float(g["a"]), float(g["b"])
    out4 = torch.zeros(4, device="cuda")
    eng.pointwise_fwd(k, N.table(tu), N.table(ti), N.table(tb), wt, uid, iid, lab, out4, a, b)
    close(out4[0], g["loss"], what="loss")
    close(out4[1], g["l2"], what="l2")
    du, di = torch.empty(B, D, device="cuda"), torch.empty(B, D, device="cuda")
    db = torch.empty(B, device="cuda")
    dw = torch.empty(D, device="cuda") if kind == "gmf" else None
    eng.pointwise_grad(k, N.table(tu), N.table(ti), N.table(tb), wt, uid, iid, lab, a, b, False, 1.0, 1.0,
                       d_user=du, d_item=di, d_bias=db, d_w=dw)
    close(torch.zeros_like(tu).index_add_(0, uid.long(), du), g["g_user"], atol=3e-5)
    close(torch.zeros_like(ti).index_add_(0, iid.long(), di), g["g_item"], atol=3e-5)
    close(torch.zeros(len(g["bias"]), device="cuda").index_add_(0, iid.long(), db), g["g_bias"], atol=3e-5)
    if kind == "gmf":
        close(dw, g["g_w"], what="g_w")


class PointProb:
    """One pointwise problem (GMF: with its dense weight w), as PairProb (non-default constants: tests/step_bar.py)."""

    def __init__(self, kind, optname, D, U, I, seed, sig=False):
        self.kind, self.optname, self.D, self.U, self.I = kind, optname, D, U, I
        self.opt, self.lr = OPTS[optname]
        self.k = N.ORX_POINT_GMF if kind == "gmf" else N.ORX_POINT_WRMF
        self.a, self.b, self.sig = (1.0, 1.0, False) if kind == "gmf" else (3.0, 0.5, sig)
        rng = np.random.default_rng(seed)
        arrs = [rng.uniform(-0.3, 0.3, s) for s in ((U, D), (I, D), (I, 1), (1, D))]
        names = ("user", "item", "bias", "w")
        st, self.dv = slots(self.opt, *zip(names, arrs))
        self.tabs = [dev(x) for x in arrs]
        self.ref = [t.cpu().numpy().astype(np.float64) for t in self.tabs]
        self.st = {k: tuple(None if s is None else dev(s).cpu().numpy().astype(np.float64) for s in v)
                   for k, v in st.items()}
        self.tt = [N.table(t, *self.dv[n]) for t, n in zip(self.tabs, names)]
        self.n = 0

    def valid(self, uid, iid):
        return (uid >= 0) & (uid < self.U) & (iid >= 0) & (iid < self.I)

    def step(self, eng, ids, label):
        uid, iid = ids
        B = len(uid)
        self.n += 1
        out = torch.zeros(4, device="cuda")
        eng.debug_dispatch_log()
        eng.pointwise_step(self.k, *self.tt[:3], self.tt[3] if self.kind == "gmf" else None, dev(uid, torch.int32),
                           dev(iid, torch.int32), dev(label), N.opt(self.opt, self.lr, step=self.n), out, self.a,
                           self.b, self.sig)
        _check_step_dispatch(eng, POINT_OP, self.k, self.opt, B, self.D)
        ok = self.valid(uid, iid)
        frac = ok.sum() / B if self.kind == "gmf" else 1.0   # GMF's mean is over the submitted batch
        user, item, bias, w = self.ref
        st = {**self.st, "w": tuple(None if s is None else s.reshape(-1, 1) for s in self.st["w"])}
        loss, l2 = O.pointwise_train_step(self.kind, user, item, bias, w.reshape(-1, 1) if self.kind == "gmf" else None,
                                          uid[ok], iid[ok], label[ok], self.opt, st, self.n, self.lr, self.a, self.b,
                                          self.sig, c_loss=frac)
        got = out.cpu().numpy().astype(np.float64)
        what = f"{self.kind} {self.optname} D={self.D} B={B} sig={self.sig} step {self.n}"
        np.testing.assert_allclose(got[0], loss * frac, rtol=2e-5, atol=ATOL, err_msg=f"loss {what}")
        np.testing.assert_allclose(got[1], l2, rtol=2e-5, atol=ATOL, err_msg=f"l2 {what}")
        assert got[2] == int(((uid < 0) | (uid >= self.U)).sum() + ((iid < 0) | (iid >= self.I)).sum()), (what, got)
        names = ("user", "item", "bias", "w") if self.kind == "gmf" else ("user", "item", "bias")
        for t, r, name in zip(self.tabs, self.ref, names):
            close(t, r, what=f"{name} {what}")
            for j in (0, 1):
                if self.st[name][j] is not None:
                    close(self.dv[name][j], self.st[name][j], what=f"{name} slot{j} {what}")
        assert got[3] == _staged(self.opt, uid[ok], iid[ok]), (what, got)
        return got


def _point_ids(rng, mode, U, I, B):
    """As _ids: "owned" every row once (U, I >= B), "staged" every row at least twice (B >= 2), else uniform."""
    if mode == "owned":
        ids = rng.permutation(U)[:B], rng.permutation(I)[:B]
    elif mode == "staged":
        ids = (np.resize(rng.permutation(U)[:max(1, B // 2)], B), np.resize(rng.permutation(I)[:max(1, B // 2)], B))
        rng.shuffle(ids[0]), rng.shuffle(ids[1])
    else:
        ids = rng.integers(0, U, B), rng.integers(0, I, B)
    return tuple(np.asarray(x, np.int32) for x in ids)


def _bad_point_ids(rng, U, I, B):
    """As _bad_pair_ids: (a) user U-1 / item I-1 in one skipped and one valid sample, (b) user U-2 / item I-2 twice,
    only in skipped samples; bad ids in uid and iid, one in the last (partial) warp."""
    uid, iid = (np.asarray(rng.integers(0, n - 2, B), np.int32) for n in (U, I))
    uid[0], iid[0], uid[1], iid[1] = U - 1, -1, U - 1, I - 1     # (a)
    iid[2], uid[2] = I - 1, BIG
    uid[3], iid[3], uid[4], iid[4] = U - 2, I, U - 2, BIG        # (b)
    uid[5], iid[5], uid[6], iid[6] = -1, I - 2, U, I - 2
    uid[7], iid[7] = BIG, -1
    iid[B - 1] = I
    return uid, iid


POINT_CASES = [(10, 29, 41, 80), (64, 700, 900, 1000), (128, 3000, 4000, 2048), (260, 300, 400, 203),
               (32, 300, 500, 237), (256, 400, 500, 391)]
POINT_SIGMOID_D = (64, 256, 260)   # WRMF with use_sigmoid: two specialised kernels and the generic one


@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D,U,I,B", POINT_CASES)
def test_pointwise_step(eng, kind, optname, D, U, I, B):
    """Two steps of uniform batches on every pointwise kernel (D = 10 / 260 generic, 32 / 64 / 128 / 256 specialised,
    with batch tails); WRMF with use_sigmoid at POINT_SIGMOID_D, without it at the other dims."""
    rng = np.random.default_rng(seed_of(kind, optname, D))
    p = PointProb(kind, optname, D, U, I, seed_of("point-tabs", kind, optname, D), D in POINT_SIGMOID_D)
    for _ in range(2):
        p.step(eng, _point_ids(rng, "mixed", U, I, B), (rng.random(B) < 0.4).astype(np.float32))


@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("mode", ["owned", "staged"])
def test_pointwise_ownership_extremes(eng, kind, optname, mode):
    """All rows owned (the in-register optimizer and the owned write-back of k_point_step) and all rows staged, on
    every pointwise kernel, at batch sizes that end in a partial warp."""
    for D, B in ((7, 203), (32, 201), (64, 237), (128, 391), (256, 203), (260, 201)):
        rng = np.random.default_rng(seed_of("pown", kind, optname, mode, D))
        U, I = (B + 31, B + 57) if mode == "owned" else (3 * B, 3 * B)
        p = PointProb(kind, optname, D, U, I, seed_of("pown-tabs", kind, optname, mode, D), sig=D == 64)
        for _ in range(2):
            uid, iid = ids = _point_ids(rng, mode, U, I, B)
            got = p.step(eng, ids, (rng.random(B) < 0.4).astype(np.float32))
            unique = len(np.unique(uid)) + len(np.unique(iid))
            if mode == "owned":
                assert unique == 2 * B and got[3] == (unique if p.opt == DENSE else 0), (D, got)
            else:
                assert got[3] == unique, (D, got, unique)


@pytest.mark.parametrize("kind", ["gmf", "wrmf"])
@pytest.mark.parametrize("optname", list(OPTS))
def test_pointwise_bad_ids(eng, kind, optname):
    """Bad ids on every pointwise kernel: counted, their samples skipped, GMF's 1/B kept over the submitted batch, rows
    referenced only by skipped samples untouched."""
    for D in (13, 32, 64, 128, 256):
        B, U, I = 203, 120, 260
        rng = np.random.default_rng(seed_of("pbad", kind, optname, D))
        p = PointProb(kind, optname, D, U, I, seed_of("pbad-tabs", kind, optname, D), sig=D == 64)
        for _ in range(2):
            p.step(eng, _bad_point_ids(rng, U, I, B), (rng.random(B) < 0.4).astype(np.float32))


def test_workspace_regrowth():
    """One fresh handle: B grows, then D grows (while a prefetched index is outstanding), then both shrink, mixing
    pairwise and pointwise steps and optimizers.  A regrowth reallocates and zeroes the index sets and the staging
    buffers and invalidates the prefetch: the step meant to consume it builds its own index (set 0)."""
    e = N.Engine(0)
    try:
        rng = np.random.default_rng(20)
        pa = PairProb("bpr", "adagrad", 64, 300, 500, 21)
        pb = PointProb("gmf", "adam_lazy", 64, 400, 500, 22)
        pc = PairProb("ucml", "adam_dense", 256, 200, 300, 23, scale=0.05)
        pd = PointProb("wrmf", "sgd", 32, 100, 150, 24, sig=True)
        pe = PairProb("bpr", "adam_lazy", 32, 80, 120, 25)

        def pf(p, ids):
            dids = [dev(x, torch.int32) for x in ids]
            torch.cuda.synchronize()
            e.pairwise_prefetch(p.tt[0], p.tt[1], *dids, p.opt, ids_ready=True)
            return dids

        ids = _ids(rng, "mixed", 300, 500, 100)
        pa.step(e, ids)                                                        # allocates: B = 100, D = 64
        ids = _ids(rng, "mixed", 300, 500, 100)
        pa.step(e, ids, dids=pf(pa, ids), index_set="prefetch")                # control: the prefetch is used
        ids = _ids(rng, "mixed", 300, 500, 100)
        dids = pf(pa, ids)
        pb.step(e, _point_ids(rng, "mixed", 400, 500, 700), (rng.random(700) < 0.4).astype(np.float32))   # B grows
        pa.step(e, ids, dids=dids, index_set=0)                                # its prefetch died with the regrowth
        ids = _ids(rng, "mixed", 200, 300, 500)
        dids = pf(pc, ids)                                                     # built for D = 256: grows D
        pa.step(e, _ids(rng, "mixed", 300, 500, 100))
        pc.step(e, ids, dids=dids, index_set=0)                                # dropped by the step above
        ids = _ids(rng, "mixed", 200, 300, 500)
        dids = pf(pc, ids)
        pc.step(e, ids, dids=dids, index_set="prefetch")
        ids = _ids(rng, "mixed", 300, 500, 1200)
        dids = pf(pa, ids)                                                     # grows B before its index is built
        pa.step(e, ids, dids=dids, index_set="prefetch")
        ids = _ids(rng, "mixed", 80, 120, 3000)
        dids = pf(pe, ids)                                                     # grows B again: reallocates ...
        pd.step(e, _point_ids(rng, "mixed", 100, 150, 5000), (rng.random(5000) < 0.4).astype(np.float32))  # ... and here
        pe.step(e, ids, dids=dids, index_set=0)
        for _ in range(2):                                                     # both shrink
            pd.step(e, _point_ids(rng, "staged", 100, 150, 37), (rng.random(37) < 0.4).astype(np.float32))
            ids = _ids(rng, "mixed", 80, 120, 7)
            pe.step(e, ids, dids=pf(pe, ids), index_set="prefetch")
            pb.step(e, _point_ids(rng, "mixed", 400, 500, 5), (rng.random(5) < 0.4).astype(np.float32))
    finally:
        e.close()


def test_sparse_step_dispatch_coverage():
    """The cases above reach every (op, variant, kind, optimizer, specialised D or generic, index set) combination the
    dispatch can choose: pairwise steps on sets 0, 1 and 2, pointwise steps (always set 0)."""
    dcls = lambda D: D if D in SPECIAL_D else "generic"
    seen = set()

    def pair(D, opt, kinds=(0, 1), sets=(0,)):
        for k in kinds:
            for s in sets:
                seen.add((PAIR_OP, _pair_rule(D, opt)[0], k, opt, dcls(D), s))

    for opt, _ in OPTS.values():
        for D in (1, 12, 50, 260, 32, 64, 128, 256) + ALL_D + (13, 32, 64, 128, 256):   # step, ownership, bad ids
            pair(D, opt)
        for D in (32, 64, 128, 256, 50):                                                # prefetch, every variant
            pair(D, opt, sets=(1, 2))
        for D, *_ in POINT_CASES:
            for k in (0, 1):
                seen.add((POINT_OP, _point_rule(D)[0], k, opt, dcls(D), 0))
    want = {(PAIR_OP, _pair_rule(D, opt)[0], k, opt, dcls(D), s)
            for D in SPECIAL_D + (1,) for opt in range(4) for k in (0, 1) for s in (0, 1, 2)}
    want |= {(POINT_OP, _point_rule(D)[0], k, opt, dcls(D), 0) for D in SPECIAL_D + (1,) for opt in range(4)
             for k in (0, 1)}
    assert seen == want, sorted(want - seen)


# ---------------------------------------------------------------------------------------
def test_gather_bit_exact(eng):
    rng = np.random.default_rng(1)
    tab = rng.standard_normal((1000, 50)).astype(np.float32)
    ids = rng.integers(0, 1000, 777)
    for dt in (torch.int32, torch.int64):
        out = eng.gather(dev(tab), dev(ids, dt))
        assert np.array_equal(out.cpu().numpy(), tab[ids])   # gather must be bit-exact
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ids2 = ids.copy()
    ids2[3] = 5000
    out = eng.gather(dev(tab), dev(ids2, torch.int32), bad)
    assert bad.item() == 1 and not out[3].any()


def test_censor(eng, golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "pairwise_ucml.npz")))
    tu, ti = dev(g["user"]), dev(g["item"])
    eng.censor(tu, dev(g["uid"], torch.int32))
    eng.censor(ti, dev(g["pid"], torch.int32))
    eng.censor(ti, dev(g["nid"], torch.int32))
    close(tu, g["user_censored"]), close(ti, g["item_censored"])
    rng = np.random.default_rng(2)
    tab = rng.standard_normal((50, 128)) * 0.001   # tiny rows: max(norm, 0.1) branch
    t = dev(tab)
    ids = rng.integers(0, 50, 400).astype(np.int32)   # many duplicates: each row scaled exactly once
    eng.censor(t, dev(ids, torch.int32))
    ref = t.new_tensor(tab).cpu().numpy().astype(np.float64)
    O.censor(ref, ids)
    close(t, ref)


def test_score_all_and_metrics(eng, golden_dir):
    from openrec_b200 import native as N
    for kind, name in ((N.ORX_SCORE_DOT, "pairwise_bpr"), (N.ORX_SCORE_NEG_SQDIST, "pairwise_ucml")):
        g = dict(np.load(os.path.join(golden_dir, f"{name}.npz")))
        s = eng.score_all(kind, dev(g["user"]), dev(g["uid"][:5], torch.int32), dev(g["item"]), dev(g["bias"]))
        close(s, g["inference"], atol=1e-4 if kind else ATOL)
    g = dict(np.load(os.path.join(golden_dir, "pointwise_gmf.npz")))
    s = eng.score_all(N.ORX_SCORE_DOT, dev(g["user"]), dev(g["uid"][:5], torch.int32), dev(g["item"]),
                      dev(g["bias"]), scale=dev(g["w"].reshape(-1)))
    close(s, g["inference"])
    m = dict(np.load(os.path.join(golden_dir, "metrics.npz")))
    auc, ndcg, rec = eng.rank_metrics(dev(m["pred"]), dev(m["pos"], torch.uint8), dev(m["excl"], torch.uint8),
                                      at=(5, 20))
    close(auc, m["auc"], atol=1e-6), close(ndcg, m["ndcg"], atol=1e-5), close(rec, m["recall"], atol=1e-6)
    # bigger random case against the oracle
    rng = np.random.default_rng(3)
    R, I = 9, 17000
    pred = rng.standard_normal((R, I)).astype(np.float32)
    pos = rng.random((R, I)) < 0.002
    pos[:, 7] = True
    excl = (rng.random((R, I)) < 0.01) & ~pos
    auc, ndcg, rec = eng.rank_metrics(dev(pred), dev(pos, torch.uint8), dev(excl, torch.uint8), at=(50, 100))
    close(auc, O.auc(pos, pred, excl), atol=1e-6)
    close(ndcg, O.ndcg(pos, pred, excl, (50, 100)), atol=1e-4)
    close(rec, O.recall(pos, pred, excl, (50, 100)), atol=1e-6)


def test_dense_apply_and_fill(eng):
    from openrec_b200 import native as N
    rng = np.random.default_rng(4)
    n = 5000
    for ok, lr in OPTS.values():
        var, grad = rng.standard_normal(n), rng.standard_normal(n)
        s0, s1 = np.abs(rng.standard_normal(n)) * 0.1 + 0.1, np.abs(rng.standard_normal(n)) * 0.1 + 0.01
        tv, tg, t0, t1 = dev(var), dev(grad), dev(s0), dev(s1)
        var, grad, s0, s1 = (t.cpu().numpy().astype(np.float64) for t in (tv, tg, t0, t1))
        eng.dense_apply(tv, t0 if ok else None, t1 if ok >= 2 else None, tg, N.opt(ok, lr, step=4))
        O.apply_dense(ok, var, s0, s1, grad, 4, lr)
        close(tv, var)
    t = torch.empty(1 << 20, device="cuda")
    eng.fill_uniform(t, -0.05, 0.05, 123)
    assert t.min().item() >= -0.05 and t.max().item() < 0.05
    assert abs(t.mean().item()) < 2e-4 and abs(t.std().item() - 0.1 / 12 ** 0.5) < 2e-4
    t2 = torch.empty_like(t)
    eng.fill_uniform(t2, -0.05, 0.05, 123)
    assert torch.equal(t, t2)


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_full_size_pairwise_adagrad(eng, kind):
    """BASELINE.json configs[1] (BPR) and configs[2] (UCML, margin 0.5, censor_vec after the step): 1M x 1M, D=128,
    B=65536; oracle on the touched rows, untouched rows bit-identical."""
    from openrec_b200 import native as N
    U = I = 1_000_000
    D, B = 128, 65536
    scale = 0.05 if kind == "bpr" else 0.4        # ucml: rows longer than 1 so that the censor has work
    tu, ti = torch.empty(U, D, device="cuda"), torch.empty(I, D, device="cuda")
    tb = torch.empty(I, 1, device="cuda")
    eng.fill_uniform(tu, -scale, scale, 1), eng.fill_uniform(ti, -scale, scale, 2), eng.fill_uniform(tb, -0.05, 0.05, 3)
    au, ai, ab = (torch.full_like(t, 0.1) for t in (tu, ti, tb))
    g = torch.Generator(device="cpu").manual_seed(1)
    uid, pid, nid = (torch.randint(0, U, (B,), generator=g, dtype=torch.int32).numpy() for _ in range(3))
    rows_u, rows_i = np.unique(uid), np.unique(np.concatenate([pid, nid]))
    # compact oracle problem over the touched rows only
    cu, cp, cn = np.searchsorted(rows_u, uid).astype(np.int32), np.searchsorted(rows_i, pid).astype(np.int32), \
        np.searchsorted(rows_i, nid).astype(np.int32)
    user = tu[torch.from_numpy(rows_u).cuda()].cpu().numpy().astype(np.float64)
    item = ti[torch.from_numpy(rows_i).cuda()].cpu().numpy().astype(np.float64)
    bias = tb[torch.from_numpy(rows_i).cuda()].cpu().numpy().astype(np.float64)
    if kind == "ucml":                            # away from the hinge's kink (resampled negatives stay inside rows_i)
        cn = avoid_hinge_ties(np.random.default_rng(4), user, item, bias, cu, cp, cn).astype(np.int32)
        nid = rows_i[cn].astype(np.int32)
    st = {k: (np.full_like(v, 0.1), None) for k, v in (("user", user), ("item", item), ("bias", bias))}
    untouched_before = ti[:1000].clone()
    out4 = torch.zeros(4, device="cuda")
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    d_uid, d_pid, d_nid = (torch.from_numpy(a).cuda() for a in (uid, pid, nid))
    eng.debug_dispatch_log()
    eng.pairwise_step(k, N.table(tu, au), N.table(ti, ai), N.table(tb, ab), d_uid, d_pid, d_nid, N.opt(1, 0.05), out4,
                      margin=0.5)
    _check_step_dispatch(eng, PAIR_OP, k, 1, B, D)       # the bench kernel: k_pair_step<.., 128, 8, 4, false>, set 0
    loss, l2 = O.pairwise_train_step(kind, user, item, bias, cu, cp, cn, 1, st, 1, 0.05, margin=0.5)
    close(out4[0], loss, rtol=2e-5), close(out4[1], l2, rtol=2e-5)
    n_dup = int((np.unique(uid, return_counts=True)[1] > 1).sum()
                + (np.unique(np.concatenate([pid, nid]), return_counts=True)[1] > 1).sum())
    assert out4[3].item() == n_dup   # exactly the duplicated rows were staged
    if kind == "ucml":               # UCML.censor_vec (recommenders/ucml.py:39-46): the caller's three censors after the step
        eng.censor(tu, d_uid), eng.censor(ti, d_pid), eng.censor(ti, d_nid)
        O.censor(user, cu), O.censor(item, cp), O.censor(item, cn)
    close(tu[torch.from_numpy(rows_u).cuda()], user)
    close(ti[torch.from_numpy(rows_i).cuda()], item)
    close(tb[torch.from_numpy(rows_i).cuda()], bias)
    close(ai[torch.from_numpy(rows_i).cuda()], st["item"][0])
    mask = torch.ones(1000, dtype=torch.bool)
    mask[torch.from_numpy(rows_i[rows_i < 1000])] = False
    assert torch.equal(ti[:1000][mask.cuda()], untouched_before[mask.cuda()])   # untouched rows bit-identical


# ---------------------------------------------------------------------------------------
# un-fused sparse apply + sharded building blocks
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D,rows,n", [(1, 300, 500), (50, 400, 1000), (128, 3000, 4096)])
def test_sparse_apply(eng, optname, D, rows, n):
    from openrec_b200 import native as N
    rng = np.random.default_rng(seed_of("sparse", optname, D))
    ok, lr = OPTS[optname]
    var = rng.uniform(-0.3, 0.3, (rows, D))
    st, dv = slots(ok, ("v", var))
    tv = dev(var)
    var = tv.cpu().numpy().astype(np.float64)
    s = tuple(None if x is None else dev(x).cpu().numpy().astype(np.float64) for x in st["v"])
    for step in (1, 2):
        ids = rng.integers(0, rows, n).astype(np.int32)
        vals = rng.standard_normal((n, D)).astype(np.float32)
        eng.sparse_apply(N.table(tv, *dv["v"]), dev(ids, torch.int32), dev(vals), N.opt(ok, lr, step=step))
        O.apply_sparse(ok, var, s[0], s[1], ids, vals.astype(np.float64), step, lr)
        close(tv, var, atol=2e-5, what=f"var step {step}")
        for j in (0, 1):
            if s[j] is not None:
                close(dv["v"][j], s[j], atol=2e-5, what=f"slot{j}")


def test_owner_bucket(eng):
    """Owner bucketing of plain lookups: orx_owner_bucket_combined with every lookup a user lookup (n_user = n) puts row r
    on rank r % world at local row r / world."""
    rng = np.random.default_rng(8)
    for world in (2, 3, 8):
        ids = rng.integers(0, 100000, 5000).astype(np.int32)
        counts, send_local, slot = (t.cpu().numpy() for t in eng.owner_bucket_combined(dev(ids, torch.int32), len(ids),
                                                                                        100000, world))
        assert np.array_equal(counts, np.bincount(ids % world, minlength=world))
        assert sorted(slot.tolist()) == list(range(len(ids)))            # a permutation
        assert np.array_equal(send_local[slot], ids // world)            # lookup i sits at slot[i]
        owner_of_slot = np.repeat(np.arange(world), counts)
        assert np.array_equal(owner_of_slot[slot], ids % world)          # buckets are contiguous per owner


@pytest.mark.parametrize("kind", ["bpr", "ucml"])
def test_pairwise_grad_rows(eng, kind):
    """Row-form gradients (the compact form of the NCCL sharded step): every lookup of the batch has its own fetched row
    of width D+4 (item bias in column D); the gradient overwrites the lookup's row of d_rows, padding included."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(9)
    B, D, R = 300, 64, 4
    sc = 0.05 if kind == "bpr" else 0.4
    rows = np.zeros((3 * B, D + 4))
    rows[:, :D + 1] = rng.uniform(-sc, sc, (3 * B, D + 1))
    perm = rng.permutation(3 * B).astype(np.int32)
    us, ps, ns = perm[:B], perm[B:2 * B], perm[2 * B:]
    trows = dev(rows)
    r64 = trows.cpu().numpy().astype(np.float64)
    d_rows = torch.full_like(trows, 7.0)       # every touched entry must be overwritten (incl. the padding)
    out4 = torch.zeros(4, device="cuda")
    k = N.ORX_PAIR_BPR if kind == "bpr" else N.ORX_PAIR_UCML
    eng.pairwise_grad_rows(k, trows, D, dev(us, torch.int32), dev(ps, torch.int32), dev(ns, torch.int32),
                           1.0 / (B * R), d_rows, out4, 0.5, 1.0, 1.0)
    emb, bias = r64[:, :D], r64[:, D:D + 1]
    if kind == "bpr":
        loss, l2 = O.bpr_forward(emb, emb, bias, us, ps, ns)
        gr = O.bpr_grads(emb, emb, bias, us, ps, ns, 1.0 / R, 1.0)
        loss = loss / R
    else:
        loss, l2 = O.ucml_forward(emb, emb, bias, us, ps, ns, 0.5)
        gr = O.ucml_grads(emb, emb, bias, us, ps, ns, 0.5)
    close(out4[0], loss, rtol=2e-5), close(out4[1], l2, rtol=2e-5)
    ref = np.zeros_like(r64)
    ref[gr["user"][0], :D], ref[gr["item"][0], :D] = gr["user"][1], gr["item"][1]
    ref[gr["bias"][0], D] = gr["bias"][1].reshape(-1)
    close(d_rows, ref, atol=1e-4 if kind == "ucml" else ATOL)


def test_owner_bucket_combined_and_grad_rows(eng):
    """The combined-table form of the sharded step: (owner, combined local row) lookups and row-form gradients."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(10)
    U, I, B, D, R = 1003, 2005, 400, 64, 3
    uid, pid, nid = (rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
    ids = np.concatenate([uid, pid, nid])
    counts, send_local, slot = (t.cpu().numpy() for t in eng.owner_bucket_combined(dev(ids, torch.int32), B, U, R))
    owner = ids % R
    assert np.array_equal(counts, np.bincount(owner, minlength=R))
    assert sorted(slot.tolist()) == list(range(3 * B))
    user_rows = (U - owner + R - 1) // R
    want_local = ids // R + np.where(np.arange(3 * B) >= B, user_rows, 0)
    assert np.array_equal(send_local[slot], want_local)
    assert np.array_equal(np.repeat(np.arange(R), counts)[slot], owner)
    # gradients on fetched rows (width D+4, bias in column D)
    W = D + 4
    rows = np.zeros((3 * B, W))
    rows[:, :D + 1] = rng.uniform(-0.05, 0.05, (3 * B, D + 1))
    perm = rng.permutation(3 * B).astype(np.int32)
    us, ps, ns = perm[:B], perm[B:2 * B], perm[2 * B:]
    trows = dev(rows)
    r64 = trows.cpu().numpy().astype(np.float64)
    d_rows = torch.full_like(trows, 7.0)       # every touched entry must be overwritten (incl. the padding)
    out4 = torch.zeros(4, device="cuda")
    eng.pairwise_grad_rows(N.ORX_PAIR_BPR, trows, D, dev(us, torch.int32), dev(ps, torch.int32), dev(ns, torch.int32),
                           1.0 / (B * R), d_rows, out4, 0.5, 1.0, 1.0)
    emb, bias = r64[:, :D], r64[:, D:D + 1]
    loss, l2 = O.bpr_forward(emb, emb, bias, us, ps, ns)
    gr = O.bpr_grads(emb, emb, bias, us, ps, ns, 1.0 / R, 1.0)
    ref = np.zeros_like(r64)
    ref[gr["user"][0], :D], ref[gr["item"][0], :D] = gr["user"][1], gr["item"][1]
    ref[gr["bias"][0], D] = gr["bias"][1].reshape(-1)
    close(out4[0], loss / R, rtol=2e-5), close(out4[1], l2, rtol=2e-5)
    close(d_rows, ref)


# ---- optimizer kind and slot rows: every entry point that applies an optimizer checks them before it launches -------
# An optimizer needs slot s0 unless it is SGD, and s1 when it is an Adam (ADAM_DENSE keeps m and v there too).
MISSING_SLOT = [(opt, j) for opt in (1, 2, 3) for j in (0, 1) if j == 0 or opt >= 2]
BAD_KINDS = (-1, 4)


def _rejected(call):
    with pytest.raises(RuntimeError, match=r"\(status -1\)"):    # ORX_ERR_INVALID
        call()


class _Tabs:
    """Tables (var, s0, s1) of the given shapes; .t(i, opt, drop) is table i with the slots `opt` needs minus `drop`."""

    def __init__(self, rng, *shapes):
        self.v = [tuple(dev(rng.uniform(0.1, 0.3, s)) for _ in range(3)) for s in shapes]
        self.before = [tuple(x.clone() for x in t) for t in self.v]

    def t(self, i, opt, drop=None):
        from openrec_b200 import native as N
        var, s0, s1 = self.v[i]
        keep0 = opt != 0 and drop != (i, 0)
        keep1 = opt in (2, 3) and drop != (i, 1)
        return N.table(var, s0 if keep0 else None, s1 if keep1 else None)

    def unchanged(self):
        return all(torch.equal(a, b) for t, u in zip(self.v, self.before) for a, b in zip(t, u))


@pytest.mark.parametrize("entry", ["pairwise_step", "pairwise_prefetch", "pointwise_step", "sparse_apply",
                                   "sparse_apply_strided", "dense_apply", "shard_step"])
def test_optimizer_kind_and_slots_checked(eng, entry):
    """A table missing a slot row its optimizer keeps, or an unknown optimizer kind, is rejected with ORX_ERR_INVALID
    and nothing is written; SGD with no slot rows is accepted."""
    from openrec_b200 import native as N
    rng = np.random.default_rng(seed_of("slots", entry))
    U, I, D, B = 40, 50, 32, 64
    ids = lambda n: dev(rng.integers(0, n, B), torch.int32)
    uid, pid, nid = ids(U), ids(I), ids(I)
    out4 = torch.zeros(4, device="cuda")
    if entry == "shard_step":
        from openrec_b200.sharded import LoopbackGroup
        g = LoopbackGroup(1, U, I, D, B, kind=0, opt_kind=2, lr=0.05, seed=1)
        try:
            m = g.ranks[0]
            full = (m._tabs, m.opt_kind)
            vars_ = [m.user, m.item, m.bias] + [x for x in m.user_slots + m.item_slots + m.bias_slots]
            before = [x.clone() for x in vars_]

            def shard(opt, drop=None):
                def tab(i, var, slots):
                    keep0 = opt != 0 and drop != (i, 0)
                    keep1 = opt in (2, 3) and drop != (i, 1)
                    return N.table(var, slots[0] if keep0 else None, slots[1] if keep1 else None)
                m._tabs = (tab(0, m.user, m.user_slots), tab(1, m.item, m.item_slots), tab(2, m.bias, m.bias_slots))
                m.opt_kind = opt
                m.iterations = 1
                m._call(uid, pid, nid, 1.0, 1.0, 0, 5)

            for opt, j in MISSING_SLOT:
                if opt == 3:
                    continue                # the sharded step rejects ADAM_DENSE whatever the slots
                for i in range(3):
                    _rejected(lambda: shard(opt, (i, j)))
            for bad in BAD_KINDS + (3,):
                _rejected(lambda: shard(bad))
            torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(vars_, before))
            shard(0)                        # SGD, no slot rows
            g.check()
            m._tabs, m.opt_kind = full
        finally:
            g.close()
        return

    if entry in ("pairwise_step", "pairwise_prefetch"):
        T = _Tabs(rng, (U, D), (I, D), (I, 1))

        def call(opt, drop=None):
            if entry == "pairwise_step":
                eng.pairwise_step(N.ORX_PAIR_BPR, T.t(0, opt, drop), T.t(1, opt, drop), T.t(2, opt, drop), uid, pid,
                                  nid, N.opt(opt, 0.05), out4)
            else:
                eng.pairwise_prefetch(T.t(0, opt, drop), T.t(1, opt, drop), uid, pid, nid, opt)
        n_tabs = 3
    elif entry == "pointwise_step":
        T = _Tabs(rng, (U, D), (I, D), (I, 1), (1, D))
        label = dev(rng.integers(0, 2, B))

        def call(opt, drop=None):                   # GMF: the dense weight w is checked like the tables
            eng.pointwise_step(N.ORX_POINT_GMF, T.t(0, opt, drop), T.t(1, opt, drop), T.t(2, opt, drop),
                               T.t(3, opt, drop), uid, pid, label, N.opt(opt, 0.05), out4)
        n_tabs = 4
    elif entry in ("sparse_apply", "sparse_apply_strided"):
        T = _Tabs(rng, (U, D))
        vals = dev(rng.standard_normal((B, 1, D)))

        def call(opt, drop=None):
            if entry == "sparse_apply":
                eng.sparse_apply(T.t(0, opt, drop), uid, vals.reshape(B, D), N.opt(opt, 0.05))
            else:
                eng.sparse_apply_strided(T.t(0, opt, drop), uid.reshape(B, 1), 0, vals, N.opt(opt, 0.05))
        n_tabs = 1
    else:
        T = _Tabs(rng, (300,))
        grad = dev(rng.standard_normal(300))

        def call(opt, drop=None):
            t = T.t(0, opt, drop)
            var, s0, s1 = T.v[0]
            eng.dense_apply(var, s0 if t.s0 else None, s1 if t.s1 else None, grad, N.opt(opt, 0.05))
        n_tabs = 1

    if entry != "pairwise_prefetch":                # the prefetch reads no slot row: the step that consumes it checks
        for opt, j in MISSING_SLOT:
            for i in range(n_tabs):
                _rejected(lambda: call(opt, (i, j)))
    for bad in BAD_KINDS:
        _rejected(lambda: call(bad))
    torch.cuda.synchronize()
    assert T.unchanged()
    call(0)                                         # SGD, no slot rows
    if entry == "pairwise_prefetch":                # consume the prefetched index
        eng.pairwise_step(N.ORX_PAIR_BPR, T.t(0, 0), T.t(1, 0), T.t(2, 0), uid, pid, nid, N.opt(0, 0.05), out4)
    torch.cuda.synchronize()
    eng.debug_dispatch_log()
