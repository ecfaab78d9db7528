"""GPU parity of the sharded catalogue evaluation (orx_score_rank_shard, openrec_b200/csrc/orx_eval.cu) and of
RankingEvaluator on ShardedBPR / ShardedUCML.

R virtual ranks on one device (openrec_b200.sharded.score_rank_sharded with loopback_sum): every rank's outputs must
equal each other bit for bit and equal orx_score_rank on the global tables -- AUC and Recall bit for bit, NDCG within
one float32 ulp, the bar of tests/test_gpu_score_rank.py.  The dummy row of an empty shard is NaN, so any read of it
shows up in the outputs."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N
from openrec_b200.sharded import loopback_sum, score_rank_sharded
from _ranks import run_ranks
from test_gpu_score_rank import SHAPES, Problem, check_equal, dev, make_problem, seed_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST]
EIGHT = (1, 2, 3, 5, 10, 50, 100, 1 << 30)


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def shard(t, R, r):
    """Rows r, r + R, ... of t; an empty shard is one NaN row (never to be read)."""
    if t is None:
        return None
    s = t[r::R].contiguous()
    return s if s.shape[0] else torch.full((1,) + tuple(t.shape[1:]), float("nan"), device=t.device)


def parts_of(pb, R, engines):
    return [(engines[r], pb.kind, shard(pb.user, R, r), shard(pb.item, R, r), shard(pb.bias, R, r),
             N.rowshard(R, r, pb.U, pb.I)) for r in range(R)]


def sharded(pb, R, at, engines=None, max_pos=None):
    engines = engines or [N.engine()] * R
    return score_rank_sharded(parts_of(pb, R, engines), loopback_sum, dev(pb.uid, torch.int32), pb.pos_off,
                              pb.pos_items, pb.excl_off, pb.excl_items, pb.max_pos() if max_pos is None else max_pos,
                              at=at)


def bits(outs):
    return [t.cpu().numpy().view(np.int32) for t in outs]


def check_ranks(outs, want, what=""):
    """every rank's outputs bit-identical to rank 0's, and rank 0's equal to orx_score_rank's"""
    first = bits(outs[0])
    for r, o in enumerate(outs[1:], 1):
        for x, y in zip(first, bits(o)):
            np.testing.assert_array_equal(x, y, err_msg=f"rank {r} differs from rank 0 {what}")
    check_equal(outs[0], want, what)


def last_shard_dispatch(eng):
    return [r for r in eng.debug_dispatch_log() if r.op == L.ORX_OP_SCORE_RANK_SHARD]


# (Bu, I, D, U): the single-device shapes, plus I < R and U < R (ranks without items or without users)
SMALL = [(6, 2, 4, 3), (40, 5, 16, 3), (9, 300, 8, 3)]
CASES = [s + (None,) for s in SHAPES] + SMALL


@pytest.mark.parametrize("Bu,I,D,U", CASES)
@pytest.mark.parametrize("biased", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_loopback_parity(eng, R, kind, biased, Bu, I, D, U):
    """Ties, one-ulp neighbours, expf overflow / underflow, excluded positives, bad uids and ignored entries
    (make_problem), over R virtual ranks sharing one handle."""
    rng = np.random.default_rng(seed_of("shard", R, kind, biased, Bu, I, D, U))
    pb = make_problem(rng, kind, Bu, I, D, biased=biased, U=U)
    eng.debug_dispatch_log()
    check_ranks(sharded(pb, R, EIGHT), pb.fused(eng, EIGHT), f"R={R}")
    rec = last_shard_dispatch(eng)
    assert [(r.ta, r.tb, r.m, r.n, r.k) for r in rec] == [(kind, r, Bu, (I - r + R - 1) // R, D) for r in range(R)]
    assert all((r.s > 0) == (r.n > 0) for r in rec)


@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_special_rows(eng, kind):
    """test_gpu_score_rank.test_special_rows under R = 3: empty rows, every item positive, duplicate and bad uids,
    ignored entries, the max_pos cut and excl_off = NULL."""
    rng = np.random.default_rng(seed_of("special", kind))
    U, I, D = 8, 300, 16
    pb = make_problem(rng, kind, 1, I, D, U=U, maxp=5, maxe=5)
    allI = list(range(I))
    pb.pos_rows.update({0: [], 1: [3, 7, 11], 2: allI, 3: [-1, 5, I], 4: sorted(rng.choice(I, 40, replace=False))})
    pb.excl_rows.update({0: [1, 2], 1: [i for i in allI if i not in (3, 7, 11)], 2: [], 3: [-1, 5, 6, I], 4: [0]})
    uid = [0, 1, 2, 3, 4, 4, -1, U, 1, 2, 5, 6]
    tabs = (pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy())
    pb = Problem(kind, *tabs, None, pb.pos_rows, pb.excl_rows, uid)
    at = (1, 10, 100, I + 1)
    check_ranks(sharded(pb, 3, at), pb.fused(eng, at), "special")
    check_ranks(sharded(pb, 3, at, max_pos=39), pb.fused(eng, at, max_pos=39), "max_pos = 39")
    noex = Problem(kind, *tabs, None, pb.pos_rows, None, uid)
    check_ranks(sharded(noex, 3, at), noex.fused(eng, at), "no exclusions")


def test_global_variant(eng):
    """One user with 30 000 positives at I = 100 003 over R = 2: the local pass keeps its thresholds in global
    scratch (RANK_GLOBAL)."""
    rng = np.random.default_rng(seed_of("global", "one_long_user"))
    kind = N.ORX_SCORE_DOT
    pb = make_problem(rng, kind, 1, 100003, 64, U=2, maxp=5, maxe=100)
    pb.pos_rows[0] = sorted(rng.choice(100003, 30000, replace=False).tolist())
    pb = Problem(kind, pb.user.cpu().numpy(), pb.item.cpu().numpy(), pb.bias.cpu().numpy(), None, pb.pos_rows,
                 pb.excl_rows, [0])
    at = (10, 100, 1000)
    eng.debug_dispatch_log()
    check_ranks(sharded(pb, 2, at), pb.fused(eng, at))
    rec = last_shard_dispatch(eng)
    assert [r.variant for r in rec] == [L.ORX_VARIANT_RANK_GLOBAL] * 2 and [r.n for r in rec] == [50002, 50001]


def test_no_state_across_phases(eng):
    """One handle for every virtual rank gives the bits of one handle per rank; so does a run in which an orx_score_rank
    call that grows the handle's scratch comes between two ranks' phase-2 calls."""
    rng = np.random.default_rng(seed_of("phases"))
    pb = make_problem(rng, N.ORX_SCORE_NEG_SQDIST, 300, 5000, 24)
    big = make_problem(rng, N.ORX_SCORE_DOT, 1000, 16980, 50, maxp=400)
    at = (5, 50)
    R = 3
    shared = sharded(pb, R, at)
    own = [N.Engine(torch.cuda.current_device()) for _ in range(R)]
    try:
        apart = sharded(pb, R, at, engines=own)
        torch.cuda.synchronize()
    finally:
        for e in own:
            e.close()
    fresh = N.Engine(torch.cuda.current_device())     # a handle whose scratch the big call has to grow
    try:
        parts = parts_of(pb, R, [fresh] * R)
        uid, max_pos = dev(pb.uid, torch.int32), pb.max_pos()
        bufs = []
        for e, kind, user, item, bias, g in parts:
            n3 = e.score_rank_shard_sizes(len(pb.uid), user.shape[1], max_pos)
            bufs.append((torch.empty(n3[0], dtype=torch.int32, device="cuda"),
                         torch.empty(n3[1], dtype=torch.int32, device="cuda"),
                         torch.empty(n3[2], dtype=torch.int64, device="cuda")))
        mixed = [None] * R
        for phase in range(4):
            for r, ((e, kind, user, item, bias, g), b) in enumerate(zip(parts, bufs)):
                if phase == 2 and r == 1:
                    big.fused(fresh, at)
                mixed[r] = e.score_rank_shard(kind, phase, g, user, item, bias, uid, pb.pos_off, pb.pos_items,
                                              pb.excl_off, pb.excl_items, max_pos, *b, at=at)
            if phase < 3:
                loopback_sum([b[phase] for b in bufs])
        torch.cuda.synchronize()
    finally:
        fresh.close()
    want = bits(shared[0])
    for outs in (shared, apart, mixed):
        for o in outs:
            for x, y in zip(want, bits(o)):
                np.testing.assert_array_equal(x, y)
    check_equal(shared[0], pb.fused(eng, at))


def test_exact_exchange(eng):
    """User and item tables holding -0.0, NaN (with payloads) and +-inf: the summed phase-0 rows are the bits of the
    global rows (0 for bad uids), and the outputs still equal orx_score_rank's."""
    rng = np.random.default_rng(seed_of("exchange"))
    U, I, D, Bu, R = 40, 500, 12, 64, 3
    pb = make_problem(rng, N.ORX_SCORE_DOT, Bu, I, D, U=U)
    user, item = pb.user.cpu().numpy(), pb.item.cpu().numpy()
    specials = np.array([-0.0, np.inf, -np.inf], np.float32)
    nans = np.array([0x7fc00001, 0xffc12345, 0x7f800001], np.uint32).view(np.float32)
    for t in (user, item):
        flat = t.reshape(-1)
        at_ = rng.choice(flat.size, 12, replace=False)
        flat[at_[:6]] = np.resize(specials, 6)
        flat[at_[6:]] = np.resize(nans, 6)
    pb = Problem(N.ORX_SCORE_DOT, user, item, pb.bias.cpu().numpy(), None, pb.pos_rows, pb.excl_rows, pb.uid)
    parts = parts_of(pb, R, [eng] * R)
    uid = dev(pb.uid, torch.int32)
    xrows = []
    for e, kind, u, it, b, g in parts:
        x = torch.full((Bu * D,), 7, dtype=torch.int32, device="cuda")
        z = torch.zeros(1, dtype=torch.int32, device="cuda")
        e.score_rank_shard(kind, 0, g, u, it, b, uid, pb.pos_off, pb.pos_items, pb.excl_off, pb.excl_items,
                           pb.max_pos(), x, z, z.to(torch.int64))
        xrows.append(x)
    loopback_sum(xrows)
    want = np.zeros((Bu, D), np.float32)
    ok = (pb.uid >= 0) & (pb.uid < U)
    want[ok] = user[pb.uid[ok]]
    np.testing.assert_array_equal(xrows[0].cpu().numpy(), want.view(np.int32).reshape(-1))
    check_ranks(sharded(pb, R, (10, 100)), pb.fused(eng, (10, 100)), "specials")


@pytest.mark.parametrize("D", [1, 7, 50, 128])
def test_dimensions(eng, D):
    """Any D (the sharded step needs D % 4 == 0; the evaluation does not)."""
    rng = np.random.default_rng(seed_of("dims", D))
    for kind in KINDS:
        pb = make_problem(rng, kind, 200, 1000, D)
        check_ranks(sharded(pb, 3, (10, 100)), pb.fused(eng, (10, 100)), f"D={D}")


def test_argument_refusals(eng):
    """Each bad argument returns ORX_ERR_INVALID and leaves the buffers untouched (no device work)."""
    rng = np.random.default_rng(seed_of("refuse"))
    pb = make_problem(rng, N.ORX_SCORE_DOT, 16, 100, 8, U=20)
    lib = L.lib()
    Bu, D, mp = 16, 8, pb.max_pos()
    P = mp + 1
    user, item, bias = pb.user[0::2].contiguous(), pb.item[0::2].contiguous(), pb.bias[0::2].contiguous()
    uid = dev(pb.uid, torch.int32)
    xrows = torch.full((Bu * D,), 7, dtype=torch.int32, device="cuda")
    xpred = torch.full((Bu * P,), 7, dtype=torch.int32, device="cuda")
    xcnt = torch.full((Bu * P,), 7, dtype=torch.int64, device="cuda")
    auc = torch.full((Bu,), 7.0, device="cuda")
    at = (C.c_int32 * 8)(*range(1, 9))
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731

    def call(phase=0, g=(2, 0, 20, 100, 10, 50), Bu=Bu, max_pos=mp, n_at=1, kind=0, xr=xrows, dim=D):
        geo = L.OrxRowShard(*g)
        return lib.orx_score_rank_shard(eng.h, kind, phase, C.byref(geo), p(user), p(item), p(bias), dim, p(uid), Bu,
                                        p(pb.pos_off), p(pb.pos_items), p(pb.excl_off), p(pb.excl_items), max_pos, at,
                                        n_at, p(xr), p(xpred), p(xcnt), p(auc), None, None, eng.stream())

    bad = {"local_users": dict(g=(2, 0, 20, 100, 11, 50)), "local_items": dict(g=(2, 1, 20, 100, 10, 49)),
           "rank = world": dict(g=(2, 2, 20, 100, 9, 49)), "rank < 0": dict(g=(2, -1, 20, 100, 10, 50)),
           "world 0": dict(g=(0, 0, 20, 100, 20, 100)), "phase 4": dict(phase=4), "phase -1": dict(phase=-1),
           "kind": dict(kind=2), "n_at 9": dict(n_at=9), "max_pos < 0": dict(max_pos=-1), "dim 0": dict(dim=0),
           "total_items > 2^31 - 1": dict(g=(1, 0, 20, 1 << 31, 20, 1 << 31)),
           "Bu * P": dict(Bu=1 << 20, max_pos=4096), "null xrows": dict(xr=None)}
    for name, kw in bad.items():
        assert call(**kw) == -1, name   # ORX_ERR_INVALID
    torch.cuda.synchronize()
    assert (xrows == 7).all() and (xpred == 7).all() and (xcnt == 7).all() and (auc == 7.0).all()
    assert call(Bu=0) == 0
    n3 = (C.c_int64 * 3)()
    assert lib.orx_score_rank_shard_sizes(Bu, D, mp, n3) == 0 and list(n3) == [Bu * D, Bu * P, Bu * P]
    assert lib.orx_score_rank_shard_sizes(-1, D, mp, n3) == -1


def _run_workers(world):
    outs = run_ranks(world, [os.path.join(ROOT, "tests", "_score_rank_shard_worker.py")], "gpu_score_rank_shard", timeout=600)
    for rc, o in outs:
        assert rc == 0, o
    assert "evaluation ok" in outs[0][1], outs[0][1]


def test_end_to_end_world_one():
    """ShardedBPR / ShardedUCML in a single-rank NCCL group, three Adagrad steps, then RankingEvaluator.evaluate equals
    evaluate on BPR / UCML holding the same tables."""
    _run_workers(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu():
    """One process per GPU over NCCL: train, evaluate on every rank (identical results), and on rank 0 compare with
    orx_score_rank on the gathered tables."""
    _run_workers(min(torch.cuda.device_count(), 4))
