"""GPU, one H100: the censor of row-sharded tables (orx_censor_shard, csrc/orx_misc.cu) and UCML.censor_vec on
row-sharded models (openrec_b200.sharded.censor_vec_sharded, LoopbackGroup.censor_vec, ShardedUCML.censor_vec).

R virtual ranks on one device: each rank's shard holds rows r, r + R, ... of a global table and censors the ids it owns
among every rank's ids.  Reassembled, the shards must equal orx_censor on the global table bit for bit (torch.equal):
the kernel shares k_censor's row arithmetic.  A rank past the table's end keeps a 1-row dummy shard of sentinel values
that must stay untouched."""
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N
from openrec_b200.sharded import LoopbackGroup, censor_gathered
from _ranks import run_ranks
from test_gpu_shard_loopback import _oracle_state

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANKS = [1, 2, 3, 5, 8]
DIMS = [1, 7, 12, 50, 128, 132, 256, 512]
SENTINEL = 3.25


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def censor_vec_variant(D):
    return L.ORX_VARIANT_CENSOR_VEC if D % 4 == 0 and D <= 128 else L.ORX_VARIANT_CENSOR_SCALAR


def make_table(rng, rows, D):
    """Rows in +-0.4, with zero rows and rows of norm < 0.1 (those grow x10 and more per censor)."""
    t = rng.uniform(-0.4, 0.4, (rows, D)).astype(np.float32)
    t[::7] = 0.0
    t[3::11] *= np.float32(1e-3)
    return torch.from_numpy(t).cuda()


def shards_of(t, R):
    return [t[r::R].clone() if t[r::R].shape[0] else torch.full((1, t.shape[1]), SENTINEL, device=t.device)
            for r in range(R)]


def assemble(shards, total, R):
    full = torch.empty(total, shards[0].shape[1], device=shards[0].device)
    for r in range(R):
        full[r::R] = shards[r][:len(range(r, total, R))]
    return full


def check_dummies(shards, total, R):
    for r in range(total, R):        # ranks past the table's end
        assert torch.equal(shards[r], torch.full_like(shards[r], SENTINEL)), f"rank {r} wrote its dummy row"


def run_blocks(engines, shards, total, R, ids, n_per_block, block_stride, first=0):
    """Every rank's orx_censor_shard over the same [R] blocks; -> the dispatch records of each rank's call."""
    recs = []
    for r in range(R):
        engines[r].debug_dispatch_log()
        engines[r].censor_shard(shards[r], total, R, r, ids, n_per_block, block_stride, R, first=first)
        recs.append([x for x in engines[r].debug_dispatch_log() if x.op == L.ORX_OP_CENSOR_SHARD])
    return recs


def check_case(eng, R, D, total, per_rank, seed):
    """per_rank: R int32 arrays of one length, rank r's ids.  Shards vs orx_censor on the global table."""
    rng = np.random.default_rng(seed)
    tab = make_table(rng, total, D)
    ref = tab.clone()
    flat = torch.from_numpy(np.concatenate(per_rank).astype(np.int32)).cuda()
    if flat.numel():
        eng.censor(ref, flat)
    shards = shards_of(tab, R)
    n = len(per_rank[0])
    recs = run_blocks([eng] * R, shards, total, R, flat, n, n)
    assert torch.equal(assemble(shards, total, R), ref)
    check_dummies(shards, total, R)
    for r, rec in enumerate(recs):
        assert len(rec) == 1, rec
        x = rec[0]
        assert (x.variant, x.ta, x.m, x.n, x.k, x.s) == (censor_vec_variant(D), r, n * R, shards[r].shape[0], D, R), x
    return ref


def split(a, R):
    return [a[r * (len(a) // R):(r + 1) * (len(a) // R)] for r in range(R)]


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("R", RANKS)
def test_bit_equal_dims(eng, R, D):
    """Uniform ids with duplicates within and across ranks, both row variants."""
    rng = np.random.default_rng(1000 * R + D)
    check_case(eng, R, D, 1000, split(rng.integers(0, 1000, 400 * R).astype(np.int32), R), R * D)


CASES = ["dups", "bad_ids", "small_total", "empty", "one_owner", "grid_pass"]


@pytest.mark.parametrize("D", [12, 50])
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("R", RANKS)
def test_bit_equal_cases(eng, R, case, D):
    rng = np.random.default_rng(zlib.crc32(f"{R}-{case}-{D}".encode()))
    total = 997
    if case == "dups":                           # 20 rows, every one many times on every rank
        ids = rng.integers(0, 20, 64 * R).astype(np.int32)
    elif case == "bad_ids":
        ids = rng.integers(0, total, 64 * R).astype(np.int32)
        ids[::5], ids[1::5], ids[2::9] = -1, total, 2 ** 31 - 1
    elif case == "small_total":                  # total < R: ranks without rows keep an untouched dummy
        total = max(R - 2, 1)
        ids = rng.integers(-1, total + 1, 16 * R).astype(np.int32)
    elif case == "empty":
        ids = np.zeros(0, np.int32)
    elif case == "one_owner":                    # every id owned by rank R - 1
        ids = (rng.integers(0, total // R, 64 * R) * R + R - 1).astype(np.int32)
        ids = ids[ids < total][:32 * R]
    else:                                        # past one grid pass (8 blocks x 8 warps x up to 32 ids per SM)
        total = 100_000
        ids = rng.integers(0, total, 300_000 - 300_000 % R).astype(np.int32)
    check_case(eng, R, D, total, split(ids, R), R)


@pytest.mark.parametrize("D", [64, 50])
@pytest.mark.parametrize("R", RANKS)
def test_censor_vec_layout_and_order(eng, R, D):
    """The strided [R][3][B] block of censor_vec: user table over every u, then the item table over every p, then
    every n -- bit-equal to orx_censor(u), orx_censor(p), orx_censor(n) on the global tables.  Rows of norm 1e-3 sit in
    both p and n: censored twice (x100 in all), p first."""
    rng = np.random.default_rng(77 + R * D)
    U, I, B = 300, 400, 96
    user, item = make_table(rng, U, D), make_table(rng, I, D)
    tiny = np.arange(5, 45, dtype=np.int32) * 13 % I
    item[torch.from_numpy(tiny).long()] = torch.full((len(tiny), D), 1e-3 / np.sqrt(D), device="cuda")
    ids = [rng.integers(0, n, (R, B)).astype(np.int32) for n in (U, I, I)]
    ids[1][:, :4], ids[2][:, -4:] = tiny[:4 * R].reshape(-1, 4)[:R], tiny[:4 * R].reshape(-1, 4)[:R]
    ids[0][0, 0], ids[1][-1, 10], ids[2][0, 12] = -1, I, 2 ** 31 - 1
    ref_u, ref_i = user.clone(), item.clone()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda()
    eng.censor(ref_u, dev(ids[0])), eng.censor(ref_i, dev(ids[1])), eng.censor(ref_i, dev(ids[2]))
    block = dev(np.stack(ids, 1))                 # [R][3][B]
    su, si = shards_of(user, R), shards_of(item, R)
    engines = [N.Engine(0) for _ in range(R)]
    try:
        for r in range(R):
            censor_gathered(engines[r], su[r], si[r], U, I, R, r, block, B)
        torch.cuda.synchronize()
    finally:
        for e in engines:
            e.close()
    assert torch.equal(assemble(su, U, R), ref_u)
    got_i = assemble(si, I, R)
    assert torch.equal(got_i, ref_i)
    norms = got_i[torch.from_numpy(tiny[:4 * R].reshape(-1)).long()].norm(dim=1)
    assert torch.allclose(norms, torch.full_like(norms, 0.1), rtol=1e-3), norms     # x10, then x10 again


def _pairwise_tables(rng, U, I, D):
    init = [rng.uniform(-0.4, 0.4, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1))]
    return init, [torch.from_numpy(a).cuda() for a in init]


def test_scratch_isolation(eng):
    """orx_censor_shard between orx_pairwise_prefetch and the step that consumes it: the step still takes the
    prefetched set (S = 1 or 2 in its record) and equals the oracle.  The censor's 8x larger id count does not grow the
    handle's index workspace (growing it would drop the outstanding prefetch and the step would build set 0)."""
    rng = np.random.default_rng(5)
    U, I, D, B = 300, 500, 64, 512
    init, tabs = _pairwise_tables(rng, U, I, D)
    ref = [a.astype(np.float64) for a in init]
    tt = [N.table(t) for t in tabs]
    e = N.Engine(0)
    try:
        out4 = torch.zeros(4, device="cuda")
        warm = [torch.from_numpy(a).cuda() for a in _draw(rng, ref, U, I, B)]
        e.pairwise_step(N.ORX_PAIR_UCML, *tt, *warm, N.opt(L.ORX_OPT_SGD, 0.05, step=1), out4, margin=0.5)
        O.pairwise_train_step("ucml", *ref, *[w.cpu().numpy() for w in warm], O.OPT_SGD, {}, 1, 0.05, margin=0.5)
        ids = [torch.from_numpy(a).cuda() for a in _draw(rng, ref, U, I, B)]
        other = make_table(rng, 4000, D)
        other_ref = other.clone()
        cids = torch.from_numpy(rng.integers(0, 4000, 8 * B).astype(np.int32)).cuda()
        torch.cuda.synchronize()
        e.pairwise_prefetch(tt[0], tt[1], *ids, L.ORX_OPT_SGD, ids_ready=True)
        e.debug_dispatch_log()
        e.censor_shard(other, 4000, 1, 0, cids, 8 * B, 8 * B, 1)
        e.pairwise_step(N.ORX_PAIR_UCML, *tt, *ids, N.opt(L.ORX_OPT_SGD, 0.05, step=2), out4, margin=0.5)
        rec = e.debug_dispatch_log()
        assert [x.op for x in rec] == [L.ORX_OP_CENSOR_SHARD, L.ORX_OP_PAIRWISE_STEP], rec
        assert rec[1].s in (1, 2), rec
        O.pairwise_train_step("ucml", *ref, *[x.cpu().numpy() for x in ids], O.OPT_SGD, {}, 2, 0.05, margin=0.5)
        for t, r in zip(tabs, ref):
            np.testing.assert_allclose(t.cpu().numpy(), r, atol=1e-5, rtol=1e-5)
        eng.censor(other_ref, cids)
        assert torch.equal(other, other_ref)
    finally:
        e.close()


def test_epoch_wrap(eng):
    """The censor hash's 31-bit epoch wraps (orx_debug_set_epoch places it just below 2^31): the slots are emptied on
    the wrap and every call still censors each owned row exactly once."""
    rng = np.random.default_rng(9)
    R, D, total = 3, 32, 500
    e = [N.Engine(0) for _ in range(R)]
    try:
        tab = make_table(rng, total, D)
        ref = tab.clone()
        shards = shards_of(tab, R)
        for r in range(R):          # first call sizes the hash, then the epoch goes to the edge
            e[r].censor_shard(shards[r], total, R, r, torch.zeros(0, dtype=torch.int32, device="cuda"), 0, 0, R)
            e[r].debug_set_epoch(0x7fffffff - 3)
        for k in range(8):
            flat = torch.from_numpy(rng.integers(0, total, 150 * R).astype(np.int32)).cuda()
            eng.censor(ref, flat)
            run_blocks(e, shards, total, R, flat, 150, 150)
            assert torch.equal(assemble(shards, total, R), ref), f"call {k}"
    finally:
        for x in e:
            x.close()


def _draw(rng, ref, U, I, n):
    """n triplets away from the UCML hinge's kink on the float64 tables (|h| < 1e-3 can flip in float32)."""
    for _ in range(50):
        ids = tuple(rng.integers(0, m, n).astype(np.int32) for m in (U, I, I))
        u, p, q = ref[0][ids[0]], ref[1][ids[1]], ref[1][ids[2]]
        h = 0.5 - ((-((u - p) ** 2).sum(1) + ref[2][ids[1], 0]) - (-((u - q) ** 2).sum(1) + ref[2][ids[2], 0]))
        if not (np.abs(h) < 1e-3).any():
            return ids
    raise AssertionError("could not avoid hinge ties")


@pytest.mark.parametrize("announce", [False, True], ids=["plain", "announced"])
@pytest.mark.parametrize("opt_kind", [0, 1], ids=["sgd", "adagrad"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_ucml_loop_loopback(world, opt_kind, announce):
    """UCML's training loop on R virtual ranks: three steps, each followed by censor_vec of its batch (announced: the
    step before announced the batch, so its route / request ran before the censor) == the float64 oracle's step on the
    concatenated batch and its censor_vec, within 1e-5."""
    rng = np.random.default_rng(31 * world + 7 * opt_kind + announce)
    U, I, D, B = 301, 503, 64, 128
    init = [rng.uniform(-0.4, 0.4, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1))]
    ref = [a.astype(np.float64) for a in init]
    st = _oracle_state(*ref, opt_kind)
    oracle_opt = {0: O.OPT_SGD, 1: O.OPT_ADAGRAD}[opt_kind]
    g = LoopbackGroup(world, U, I, D, B, kind=1, opt_kind=opt_kind, lr=0.05, init=False)
    try:
        g.load_global(*init)
        # the oracle's tables at draw time are those the batch meets, so batches are drawn while the oracle runs
        ids = _draw(rng, ref, U, I, B * world)
        batches = [[tuple(torch.from_numpy(a[r * B:(r + 1) * B].copy()).cuda() for a in ids) for r in range(world)]]
        for step in range(3):
            O.pairwise_train_step("ucml", *ref, *ids, oracle_opt, st, step + 1, 0.05, margin=0.5)
            O.ucml_censor_vec(ref[0], ref[1], *ids)
            nxt_ids = _draw(rng, ref, U, I, B * world) if step < 2 else None
            if nxt_ids is not None:
                batches.append([tuple(torch.from_numpy(a[r * B:(r + 1) * B].copy()).cuda() for a in nxt_ids)
                                 for r in range(world)])
            g.step(batches[step], next_batches=batches[step + 1] if announce and nxt_ids is not None else None)
            g.censor_vec(batches[step])
            ids = nxt_ids
        g.check()
        for a, r in zip([t.cpu().numpy() for t in g.gather_global()], ref):
            np.testing.assert_allclose(a, r, atol=1e-5, rtol=1e-5)
    finally:
        g.close()


def _run_workers(world):
    outs = run_ranks(world, [os.path.join(ROOT, "tests", "_censor_shard_worker.py")], "gpu_censor_shard", timeout=600)
    for rc, o in outs:
        assert rc == 0, o
    assert "censor ok" in outs[0][1], outs[0][1]


def test_end_to_end_world_one():
    """ShardedUCML in a single-rank NCCL group: tape + Adagrad + censor_vec for three steps gives UCML's losses and
    tables from the same weights, and item_latent_factor.censor equals UCML's."""
    _run_workers(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu():
    """One process per GPU over NCCL: ShardedUCML trained with censor_vec against UCML on rank 0."""
    _run_workers(min(torch.cuda.device_count(), 4))
