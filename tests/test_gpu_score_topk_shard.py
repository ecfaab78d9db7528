"""GPU parity of the sharded top-K retrieval (orx_score_topk_shard, openrec_b200/csrc/orx_eval.cu) and of Retriever on
ShardedBPR / ShardedUCML.

R virtual ranks on one device (openrec_b200.sharded.score_topk_sharded with loopback_sum): every rank's items and score
bits must equal rank 0's, and rank 0's must equal orx_score_topk on the global tables -- items equal, scores bit for bit
(both decode the same keys), whatever R is.  A NaN row would be dropped by the top-K as ineligible, so the dummy row of
an empty item shard is a zero row with bias +inf instead: a read of it would put an item id >= I first in the list."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N
from openrec_b200.sharded import loopback_sum, score_topk_sharded
from _ranks import run_ranks
from test_gpu_score_topk import F32, SHAPES, Problem, dev, make_problem, seed_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST]


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def shard(t, R, r, dummy):
    """Rows r, r + R, ... of t; an empty shard is one row of `dummy` (never to be read)."""
    if t is None:
        return None
    s = t[r::R].contiguous()
    return s if s.shape[0] else torch.full((1,) + tuple(t.shape[1:]), dummy, device=t.device)


def parts_of(pb, R, engines):
    return [(engines[r], pb.kind, shard(pb.user, R, r, float("nan")), shard(pb.item, R, r, 0.0),
             shard(pb.bias, R, r, float("inf")), N.rowshard(R, r, pb.U, pb.I)) for r in range(R)]


def sharded(pb, R, k, engines=None, uid=None):
    uid = pb.uid if uid is None else uid
    outs = score_topk_sharded(parts_of(pb, R, engines or [N.engine()] * R), loopback_sum, dev(uid, torch.int32),
                              pb.excl_off, pb.excl_items, k)
    return [(it.cpu().numpy(), sc.cpu().numpy()) for it, sc in outs]


def check_ranks(outs, want, what=""):
    """every rank's output bit-identical to rank 0's, and rank 0's equal to orx_score_topk's"""
    for r, (it, sc) in enumerate(outs):
        np.testing.assert_array_equal(it, outs[0][0], err_msg=f"rank {r} items differ from rank 0 {what}")
        np.testing.assert_array_equal(sc.view(np.int32), outs[0][1].view(np.int32), err_msg=f"rank {r} {what}")
    np.testing.assert_array_equal(outs[0][0], want[0], err_msg=f"items {what}")
    np.testing.assert_array_equal(outs[0][1].view(np.int32), want[1].view(np.int32), err_msg=f"score bits {what}")


def shard_dispatch(eng):
    return [r for r in eng.debug_dispatch_log() if r.op == L.ORX_OP_SCORE_TOPK_SHARD]


def ks_for(I):
    """k = 1, 7, 100, ORX_MAX_TOPK and one k > I (where <= ORX_MAX_TOPK)"""
    return sorted({k for k in (1, 7, 100, L.ORX_MAX_TOPK, I + 3) if k <= L.ORX_MAX_TOPK})


# (Bu, I, D, U): the single-device shapes, plus I < R and U < R (ranks without items or without users)
SMALL = [(6, 2, 4, 3), (40, 5, 16, 3), (9, 300, 8, 3)]
CASES = [s + (None,) for s in SHAPES] + SMALL


@pytest.mark.parametrize("Bu,I,D,U", CASES)
@pytest.mark.parametrize("biased", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_loopback_parity(eng, R, kind, biased, Bu, I, D, U):
    """Exact ties and one-ulp neighbours on items of different ranks, bad and duplicate uids and ignored exclusion
    entries (make_problem), over R virtual ranks sharing one handle; one dispatch record per rank's phase 1."""
    rng = np.random.default_rng(seed_of("topk-shard", R, kind, biased, Bu, I, D, U))
    pb = make_problem(rng, kind, Bu, I, D, biased=biased, U=U)
    for k in ks_for(I):
        eng.debug_dispatch_log()
        check_ranks(sharded(pb, R, k), pb.fused(eng, k), f"R={R} k={k}")
        rec = shard_dispatch(eng)
        assert [(r.variant, r.ta, r.tb, r.m, r.n, r.k) for r in rec] == \
            [(L.ORX_VARIANT_TOPK, kind, r, Bu, (I - r + R - 1) // R, D) for r in range(R)]
        assert all((r.s > 0) == (r.n > 0) for r in rec)


@pytest.mark.parametrize("R", [3, 8])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_special_values_and_exclusions(eng, kind, R):
    """test_gpu_score_topk.test_special_values_and_exclusions over R ranks: NaN biases (never returned), +-inf biases,
    zero scores of both signs, rows with fewer than k eligible items in total and a row with every item excluded, list
    entries -1 and I, duplicate uids, uids -1 and U; then the same users with excl_off = NULL."""
    rng = np.random.default_rng(seed_of("special", kind))
    U, I, D = 8, 300, 16
    user = rng.uniform(-1, 1, (U, D)).astype(F32)
    item = rng.uniform(-1, 1, (I, D)).astype(F32)
    bias = rng.uniform(-1, 1, I).astype(F32)
    bias[rng.choice(I, 30, replace=False)] = np.nan
    bias[rng.choice(I, 10, replace=False)] = np.inf
    bias[rng.choice(I, 10, replace=False)] = -np.inf
    zero = rng.choice(I, 40, replace=False)
    item[zero] = 0.0
    bias[zero] = np.where(np.arange(40) % 2, F32(-0.0), F32(0.0))
    user[3] = 0.0                                             # with DOT: exact zeros of both bias signs
    allI = list(range(I))
    excl = {0: allI[5:], 1: [-1] + allI[:290] + [I], 2: [], 3: [-1, 5, 6, I], 4: allI, 5: [7]}
    uid = [0, 1, 2, 3, 4, 4, -1, U, 1, 2, 5, 6, 3]
    pb = Problem(kind, user, item, bias, None, excl, uid)
    for k in (1, 7, 50, 400):
        got = sharded(pb, R, k)
        check_ranks(got, pb.fused(eng, k), f"k={k}")
        assert not np.isnan(got[0][1]).any()
        assert (got[0][0][4] == -1).all() and np.isneginf(got[0][1][4]).all()          # everything excluded
    noex = Problem(kind, user, item, bias, None, None, uid)
    for k in (10, 400):
        check_ranks(sharded(noex, R, k), noex.fused(eng, k), f"no exclusions k={k}")


@pytest.mark.parametrize("R", [2, 3, 8])
def test_equal_scores_across_ranks(eng, R):
    """Every item row and bias equal (and a bad uid under DOT without bias, which scores 0 everywhere): every score
    ties, so the answer is the first k eligible global ids, which lie on every rank."""
    rng = np.random.default_rng(seed_of("equal", R))
    U, I, D = 6, 5000, 32
    item = np.repeat(rng.uniform(-1, 1, (1, D)).astype(F32), I, axis=0)
    bias = np.full(I, F32(0.25))
    excl = {0: [0, 1, 2, 9, 10], 1: list(range(1, 4000, 2))}
    for b in (bias, None):
        pb = Problem(N.ORX_SCORE_DOT, rng.uniform(-1, 1, (U, D)).astype(F32), item, b, None, excl, [0, 1, 2, -1, U])
        for k in (1, 100, L.ORX_MAX_TOPK):
            got = sharded(pb, R, k)
            check_ranks(got, pb.fused(eng, k), f"k={k}")
            assert (got[0][0][2] == np.arange(k)).all()


def test_no_state_across_phases(eng):
    """One handle for every virtual rank gives the bits of one handle per rank; so does a run in which an
    orx_score_topk call that grows the handle's scratch comes between two ranks' phase-1 calls."""
    rng = np.random.default_rng(seed_of("phases"))
    pb = make_problem(rng, N.ORX_SCORE_NEG_SQDIST, 300, 5000, 24)
    big = make_problem(rng, N.ORX_SCORE_DOT, 1000, 100003, 64)
    R, k = 3, 100
    shared = sharded(pb, R, k)
    own = [N.Engine(torch.cuda.current_device()) for _ in range(R)]
    try:
        apart = sharded(pb, R, k, engines=own)
        torch.cuda.synchronize()
    finally:
        for e in own:
            e.close()
    fresh = N.Engine(torch.cuda.current_device())     # a handle whose scratch the big call has to grow
    try:
        parts = parts_of(pb, R, [fresh] * R)
        uid = dev(pb.uid, torch.int32)
        Bu = len(pb.uid)
        bufs = [(torch.empty(Bu * pb.D, dtype=torch.int32, device="cuda"),
                 torch.empty(Bu * R * k, dtype=torch.int64, device="cuda")) for _ in range(R)]
        mixed = [None] * R
        for phase in range(3):
            for r, ((e, kind, user, item, bias, g), b) in enumerate(zip(parts, bufs)):
                if phase == 1 and r == 1:
                    big.fused(fresh, L.ORX_MAX_TOPK)
                mixed[r] = e.score_topk_shard(kind, phase, g, user, item, bias, uid, pb.excl_off, pb.excl_items, k,
                                              *b)
            if phase < 2:
                loopback_sum([b[phase] for b in bufs])
        mixed = [(it.cpu().numpy(), sc.cpu().numpy()) for it, sc in mixed]
    finally:
        torch.cuda.synchronize()
        fresh.close()
    want = pb.fused(eng, k)
    for outs in (shared, apart, mixed):
        check_ranks(outs, want)


def test_argument_refusals(eng):
    """Each bad argument returns ORX_ERR_INVALID and leaves the buffers untouched (no device work)."""
    rng = np.random.default_rng(seed_of("refuse"))
    pb = make_problem(rng, N.ORX_SCORE_DOT, 16, 100, 8, U=20)
    lib = L.lib()
    Bu, D, k = 16, 8, 10
    user, item, bias = pb.user[0::2].contiguous(), pb.item[0::2].contiguous(), pb.bias[0::2].contiguous()
    uid = dev(pb.uid, torch.int32)
    xrows = torch.full((Bu * D,), 7, dtype=torch.int32, device="cuda")
    xkeys = torch.full((Bu * 2 * k,), 7, dtype=torch.int64, device="cuda")
    items = torch.full((Bu, k), 7, dtype=torch.int32, device="cuda")
    scores = torch.full((Bu, k), 7.0, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731

    def call(phase=0, g=(2, 0, 20, 100, 10, 50), Bu=Bu, k=k, kind=0, dim=D, u=uid, us=user, it=item, xr=xrows,
             xk=xkeys, ti=items):
        geo = L.OrxRowShard(*g)
        return lib.orx_score_topk_shard(eng.h, kind, phase, C.byref(geo), p(us), p(it), p(bias), dim, p(u), Bu,
                                        p(pb.excl_off), p(pb.excl_items), k, p(xr), p(xk), p(ti), p(scores),
                                        eng.stream())

    bad = {"local_users": dict(g=(2, 0, 20, 100, 11, 50)), "local_items": dict(g=(2, 1, 20, 100, 10, 49)),
           "rank = world": dict(g=(2, 2, 20, 100, 9, 49)), "rank < 0": dict(g=(2, -1, 20, 100, 10, 50)),
           "world 0": dict(g=(0, 0, 20, 100, 20, 100)), "phase 3": dict(phase=3), "phase -1": dict(phase=-1),
           "kind": dict(kind=2), "dim 0": dict(dim=0), "Bu < 0": dict(Bu=-1), "k 0": dict(k=0),
           "k > ORX_MAX_TOPK": dict(k=L.ORX_MAX_TOPK + 1),
           "total_items > 2^31 - 1": dict(g=(1, 0, 20, 1 << 31, 20, 1 << 31)),
           "Bu * world * k": dict(Bu=1 << 21, k=L.ORX_MAX_TOPK), "null uid": dict(u=None),
           "phase 0 null user_shard": dict(us=None), "phase 0 null xrows": dict(xr=None),
           "phase 1 null item_shard": dict(phase=1, it=None), "phase 1 null xrows": dict(phase=1, xr=None),
           "phase 1 null xkeys": dict(phase=1, xk=None), "phase 2 null xkeys": dict(phase=2, xk=None),
           "phase 2 null top_items": dict(phase=2, ti=None)}
    for name, kw in bad.items():
        assert call(**kw) == -1, name   # ORX_ERR_INVALID
    torch.cuda.synchronize()
    assert (xrows == 7).all() and (xkeys == 7).all() and (items == 7).all() and (scores == 7.0).all()
    assert call(Bu=0, u=None, xr=None, xk=None, ti=None) == 0
    assert call(k=L.ORX_MAX_TOPK, xk=None) == 0       # k > total_items is allowed; phase 0 does not need xkeys


def test_catalogue_shape(eng):
    """I = 1 000 000, D = 128, Bu = 1 024, k = 100, exclusions ~ Poisson(100) per user, over R = 2."""
    rng = np.random.default_rng(seed_of("catalogue"))
    I, D, Bu, U = 1_000_000, 128, 1024, 1024
    user = rng.uniform(-0.1, 0.1, (U, D)).astype(F32)
    item = rng.uniform(-0.1, 0.1, (I, D)).astype(F32)
    bias = rng.uniform(-0.1, 0.1, I).astype(F32)
    excl = {u: np.unique(rng.integers(0, I, rng.poisson(100))).tolist() for u in range(U)}
    pb = Problem(N.ORX_SCORE_DOT, user, item, bias, None, excl, rng.permutation(U)[:Bu])
    check_ranks(sharded(pb, 2, 100), pb.fused(eng, 100))


# ---- end to end through openrec.tf2 over NCCL ------------------------------------------------------------------------
def _run_workers(world):
    outs = run_ranks(world, [os.path.join(ROOT, "tests", "_score_topk_shard_worker.py")], "gpu_score_topk_shard", timeout=600)
    for rc, o in outs:
        assert rc == 0, o
    assert "retrieval ok" in outs[0][1], outs[0][1]


def test_end_to_end_world_one():
    """ShardedBPR / ShardedUCML in a single-rank NCCL group, three Adagrad steps, then Retriever.recommend equals
    recommend on BPR / UCML holding the same tables."""
    _run_workers(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu():
    """One process per GPU over NCCL (world 2 to 4): train, recommend on every rank (identical results), and on rank 0
    compare with Retriever on the gathered tables."""
    _run_workers(min(torch.cuda.device_count(), 4))
