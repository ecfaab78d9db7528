"""GPU parity of the sharded listed-candidate evaluation (orx_score_rank_listed_shard, openrec_b200/csrc/orx_eval.cu)
and of CandidateEvaluator on row-sharded models.

R virtual ranks on one device (openrec_b200.sharded.score_rank_listed_sharded with loopback_sum): every rank's outputs
must equal each other bit for bit and equal orx_score_rank_listed on the global tables -- AUC and Recall bit for bit,
NDCG within one float32 ulp.  The dummy row of an empty shard is NaN, so any read of it shows up in the outputs."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N
from openrec_b200.sharded import loopback_sum, score_rank_listed_sharded
from _ranks import run_ranks
from test_gpu_score_rank import check_equal, dev, seed_of
from test_gpu_score_rank_listed import Listed, make_listed
from test_gpu_score_rank_shard import bits, shard

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = [N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST]
EIGHT = (1, 2, 3, 5, 10, 50, 100, 1 << 30)


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def sharded(pb, R, at, engines=None, max_pos=None, scaled=False):
    """The four phases over R virtual ranks; with `scaled` the user rows are scaled by pb.scale (GMF) between phases."""
    engines = engines or [N.engine()] * R
    parts = [(engines[r], pb.kind, shard(pb.user, R, r), shard(pb.item, R, r), shard(pb.bias, R, r),
              N.rowshard(R, r, pb.U, pb.I)) for r in range(R)]
    return score_rank_listed_sharded(parts, loopback_sum, dev(pb.uid, torch.int32), pb.pos_off, pb.pos_items,
                                     pb.neg_off, pb.neg_items, pb.excl_off, pb.excl_items,
                                     pb.max_pos() if max_pos is None else max_pos, at=at,
                                     scale=[pb.scale] * R if scaled else None)


def check_ranks(outs, want, what=""):
    first = bits(outs[0])
    for r, o in enumerate(outs[1:], 1):
        for x, y in zip(first, bits(o)):
            np.testing.assert_array_equal(x, y, err_msg=f"rank {r} differs from rank 0 {what}")
    check_equal(outs[0], want, what)


# (Bu, I, D, U): I < R and U < R give ranks without items or without users
CASES = [(1, 1, 1, None), (37, 129, 33, None), (1000, 16980, 50, None), (37, 16980, 128, None), (6, 2, 4, 3),
         (40, 5, 16, 3), (9, 300, 8, 3)]


@pytest.mark.parametrize("Bu,I,D,U", CASES)
@pytest.mark.parametrize("biased", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_loopback_parity(eng, R, kind, biased, Bu, I, D, U):
    """Ties, one-ulp neighbours, expf overflow / underflow, excluded positives, listed items that are positives or
    excluded, bad uids and ignored entries over R virtual ranks whose phases interleave on one handle."""
    rng = np.random.default_rng(seed_of("listed-shard", R, kind, biased, Bu, I, D, U))
    pb = make_listed(rng, kind, Bu, I, D, biased=biased, U=U)
    check_ranks(sharded(pb, R, EIGHT), pb.listed(eng, EIGHT), f"R={R}")


@pytest.mark.parametrize("R", [1, 3, 8])
def test_gmf_scale(eng, R):
    """GMF: the summed user rows scaled by w between phases 0 and 1 equal the single-device call with scale = w."""
    rng = np.random.default_rng(seed_of("listed-shard-gmf", R))
    pb = make_listed(rng, N.ORX_SCORE_DOT, 300, 4000, 32, scaled=True)
    check_ranks(sharded(pb, R, (5, 50), scaled=True), pb.listed(eng, (5, 50)), f"R={R}")


@pytest.mark.parametrize("kind", KINDS, ids=["dot", "neg_sqdist"])
def test_special_rows(eng, kind):
    """The crafted rows of test_gpu_score_rank_listed.test_special_rows under R = 3, with the max_pos cut."""
    rng = np.random.default_rng(seed_of("listed-shard-special", kind))
    pb = make_listed(rng, kind, 1, 300, 16, U=8, maxp=5, maxe=5)
    pb.pos_rows.update({0: [], 1: [3, 7, 11], 2: list(range(40)), 3: [-1, 5, 300]})
    pb.neg_rows.update({0: [1, 2], 1: [], 2: [50, 51], 3: [-1, 5, 6, 7, 300]})
    pb.excl_rows.update({0: [1], 1: [3], 2: [], 3: [-1, 6, 300]})
    u, i, b, _ = pb.tables()
    uid = [0, 1, 2, 3, 4, 4, -1, 8, 5, 6]
    pb = Listed(kind, u, i, b, None, pb.pos_rows, pb.neg_rows, pb.excl_rows, uid)
    at = (1, 10, 301)
    check_ranks(sharded(pb, 3, at), pb.listed(eng, at), "special")
    check_ranks(sharded(pb, 3, at, max_pos=39), pb.listed(eng, at, max_pos=39), "max_pos = 39")
    noex = Listed(kind, u, i, b, None, pb.pos_rows, pb.neg_rows, None, uid)
    check_ranks(sharded(noex, 3, at), noex.listed(eng, at), "no exclusions")


def test_no_state_across_phases(eng):
    """One handle per virtual rank gives the bits of one shared handle; so does a run in which a single-device call
    that grows a fresh handle's scratch comes between two ranks' phase-2 calls on that handle."""
    rng = np.random.default_rng(seed_of("listed-phases"))
    pb = make_listed(rng, N.ORX_SCORE_NEG_SQDIST, 300, 5000, 24)
    big = make_listed(rng, N.ORX_SCORE_DOT, 1000, 16980, 50, maxp=400)
    at, R = (5, 50), 3
    shared = sharded(pb, R, at)
    own = [N.Engine(torch.cuda.current_device()) for _ in range(R)]
    try:
        apart = sharded(pb, R, at, engines=own)
        torch.cuda.synchronize()
    finally:
        for e in own:
            e.close()
    fresh = N.Engine(torch.cuda.current_device())
    try:
        parts = [(fresh, pb.kind, shard(pb.user, R, r), shard(pb.item, R, r), shard(pb.bias, R, r),
                  N.rowshard(R, r, pb.U, pb.I)) for r in range(R)]
        uid, max_pos = dev(pb.uid, torch.int32), pb.max_pos()
        n3 = fresh.score_rank_shard_sizes(len(pb.uid), pb.user.shape[1], max_pos)
        bufs = [(torch.empty(n3[0], dtype=torch.int32, device="cuda"), torch.empty(n3[1], dtype=torch.int32,
                 device="cuda"), torch.empty(n3[2], dtype=torch.int64, device="cuda")) for _ in range(R)]
        mixed = [None] * R
        for phase in range(4):
            for r, ((e, kind, user, item, bias, g), b) in enumerate(zip(parts, bufs)):
                if phase == 2 and r == 1:
                    big.listed(fresh, at)
                mixed[r] = e.score_rank_listed_shard(kind, phase, g, user, item, bias, uid, pb.pos_off, pb.pos_items,
                                                     pb.neg_off, pb.neg_items, pb.excl_off, pb.excl_items, max_pos,
                                                     *b, at=at)
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
    check_equal(shared[0], pb.listed(eng, at))


def test_argument_refusals(eng):
    """Each bad argument returns ORX_ERR_INVALID and leaves the buffers untouched (no device work)."""
    rng = np.random.default_rng(seed_of("listed-shard-refuse"))
    pb = make_listed(rng, N.ORX_SCORE_DOT, 16, 100, 8, U=20)
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

    def call(phase=0, g=(2, 0, 20, 100, 10, 50), Bu=Bu, max_pos=mp, n_at=1, kind=0, xr=xrows, xc=xcnt, dim=D,
             neg_off=pb.neg_off, pos_off=pb.pos_off):
        geo = L.OrxRowShard(*g)
        return lib.orx_score_rank_listed_shard(eng.h, kind, phase, C.byref(geo), p(user), p(item), p(bias), dim,
                                               p(uid), Bu, p(pos_off), p(pb.pos_items), p(neg_off), p(pb.neg_items),
                                               p(pb.excl_off), p(pb.excl_items), max_pos, at, n_at, p(xr), p(xpred),
                                               p(xc), p(auc), None, None, eng.stream())

    bad = {"local_users": dict(g=(2, 0, 20, 100, 11, 50)), "local_items": dict(g=(2, 1, 20, 100, 10, 49)),
           "rank = world": dict(g=(2, 2, 20, 100, 9, 49)), "rank < 0": dict(g=(2, -1, 20, 100, 10, 50)),
           "world 0": dict(g=(0, 0, 20, 100, 20, 100)), "phase 4": dict(phase=4), "phase -1": dict(phase=-1),
           "kind": dict(kind=2), "n_at 9": dict(n_at=9), "max_pos < 0": dict(max_pos=-1), "dim 0": dict(dim=0),
           "total_items > 2^31 - 1": dict(g=(1, 0, 20, 1 << 31, 20, 1 << 31)),
           "Bu * P": dict(Bu=1 << 20, max_pos=4096), "null xrows": dict(xr=None),
           "phase 2 null xcnt": dict(phase=2, xc=None), "phase 3 null xcnt": dict(phase=3, xc=None),
           "null pos_off": dict(pos_off=None), "null neg_off": dict(neg_off=None),
           "null neg_off phase 2": dict(phase=2, neg_off=None)}
    for name, kw in bad.items():
        assert call(**kw) == -1, name   # ORX_ERR_INVALID
    torch.cuda.synchronize()
    assert (xrows == 7).all() and (xpred == 7).all() and (xcnt == 7).all() and (auc == 7.0).all()
    assert call(Bu=0) == 0 and call(Bu=0, neg_off=None) == 0


def _run_workers(world):
    outs = run_ranks(world, [os.path.join(ROOT, "tests", "_score_rank_listed_shard_worker.py")],
                     "gpu_score_rank_listed_shard", timeout=600)
    for rc, o in outs:
        assert rc == 0, o
    assert "evaluation ok" in outs[0][1], outs[0][1]


def test_end_to_end_world_one():
    """ShardedBPR / ShardedGMF in a single-rank NCCL group, three Adagrad steps, then CandidateEvaluator.evaluate
    equals evaluate on BPR / GMF holding the same tables."""
    _run_workers(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu():
    """One process per GPU over NCCL: train, evaluate on every rank (identical results), and on rank 0 compare with
    orx_score_rank_listed on the gathered tables."""
    _run_workers(min(torch.cuda.device_count(), 4))
