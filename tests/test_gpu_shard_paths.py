"""GPU, ONE device: the home-routed sharded step (csrc/orx_shard.cu) on every path it takes, with R virtual ranks
(LoopbackGroup), against the float64 oracle on the global batch after EVERY step:

* at the bench's per-rank batch with its production capacities, where request, serve and compute take grid-stride
  second passes;
* exactly on, and one triplet past, each mailbox capacity (home_cap, the padded gradient inbox gin_cap, req_cap);
* at batch tails (plain and announced), loss / l2 scales other than 1, bad ids in a tail;
* over kind x optimizer x row width, at 16 and 64 ranks, across the index-epoch wrap with announced batches;
* beside the other entry points of a rank's handle while an announced batch is outstanding.

Each step compares the global (loss, l2) of every rank (bit-identical across ranks), all three tables, every optimizer
slot, and out4[2] (skipped triplets) / out4[3] (staged rows) of each rank against counts taken from the ids."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import device_samplers as S
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_kernels import avoid_hinge_ties  # noqa: E402
from test_gpu_misc_kernels import _pairwise_store  # noqa: E402
from test_gpu_shard_loopback import _oracle_state  # noqa: E402

pytestmark = pytest.mark.gpu

OPT = {0: O.OPT_SGD, 1: O.OPT_ADAGRAD, 2: O.OPT_ADAM_LAZY}
ERR_WORD = 4 * 64          # flags[4 * SH_MAX_R]: the sticky error word


# ---- path rules ------------------------------------------------------------------------------------------------------
# The branches of each kernel and how much one grid pass covers.  Persistent grids are at most 4 CTAs per SM (the
# launchers take min(occupancy, 4)); the pass sizes below use that bound, so a size chosen to need two passes needs them
# at any occupancy.
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def route_tail(B):                      # k_sh_route: thread i = block * 1024 + k * 256 + lane, i < B masks the last block
    return B % 256 != 0


def request_pass(home_cap):             # k_sh_request: min(ceil(home_cap / 512), SMs) blocks x 512 triplets; the owner
    return min((home_cap + 511) // 512, _sms()) * 512     # counters `cnt` restart at the top of every pass


def serve_pass():                       # k_sh_serve: 4 CTAs / SM x 8 warps x 8 inbox rows
    return _sms() * 4 * 8 * 8


def nq_class(D):                        # float4 slots per lane: D <= 128, <= 256, <= 512
    q = D // 4
    return 1 if q <= 32 else (2 if q <= 64 else 4)


def idle_lanes(D):                      # lanes of the top slot with e >= D / 4 (masked loads / stores)
    return D // 4 < 32 * nq_class(D)


def compute_pass(D):                    # k_sh_compute: 4 CTAs / SM x 8 warps x TPW triplets (TPW = 4, 2, 1 by class)
    return _sms() * 4 * 8 * {1: 4, 2: 2, 4: 1}[nq_class(D)]


def pad32(c):                           # a source's inbox rows start on a 32-row boundary
    return (c + 31) // 32 * 32


def stats(world, ids, U, I):
    """Counts a step's kernels see, from its global ids: triplets per home T[h], requests rc[owner, home], skipped
    triplets and staged rows per rank, and whether owned / staged user and item rows occur."""
    u, p, n = (np.asarray(a, np.int64) for a in ids)
    R = world
    b = len(u) // R
    ok = (u >= 0) & (u < U) & (p >= 0) & (p < I) & (n >= 0) & (n < I)
    u, p, n = u[ok], p[ok], n[ok]
    T = np.bincount(u % R, minlength=R)
    rc = np.zeros((R, R), np.int64)
    np.add.at(rc, (np.concatenate([p, n]) % R, np.concatenate([u, u]) % R), 1)
    uu, cu = np.unique(u, return_counts=True)
    ii, ci = np.unique(np.concatenate([p, n]), return_counts=True)
    staged = [int(((uu % R == r) & (cu > 1)).sum() + ((ii % R == r) & (ci > 1)).sum()) for r in range(R)]
    bad = [int((~ok[r * b:(r + 1) * b]).sum()) for r in range(R)]
    # item bias rows follow the item rows: an owned item's bias is applied in k_sh_apply, a staged one in k_sh_tail
    return dict(T=T, rc=rc, staged=staged, bad=bad, b=b, user_owned=bool((cu == 1).any()),
                user_staged=bool((cu > 1).any()), item_owned=bool((ci == 1).any()), item_staged=bool((ci > 1).any()))


def serve_rows(st):                     # inbox rows per owner: sum over homes of the padded request counts
    return np.array([sum(pad32(int(c)) for c in row) for row in st["rc"]])


def padding_warp(st):                   # a source with >= 8 padding rows: some warp's 8 rows are all padding
    return any(pad32(int(c)) - c >= 8 for c in st["rc"].ravel())


def partial_group(st):                  # a source whose last 8-row group is incomplete: vmask != 0xff
    return any(c % 8 for c in st["rc"].ravel())


# ---- cases -----------------------------------------------------------------------------------------------------------
U_BIG, I_BIG = 50021, 49999


def bench_world1_B():
    return _sms() * 512 + 1000          # production capacities (B > 65536), two request passes


BENCH = {"world1": 1, "world2_home0": 2}   # world 2: B = 40000, every user even: home 0 gets all 80000 = home_cap
BENCH_KINDS = [(0, 1), (1, 2)]          # BPR x Adagrad, UCML x lazy Adam

GRID_D = (4, 12, 128, 132, 260, 508)
GRID_KO = [(k, o) for k in (0, 1) for o in (0, 1, 2)]
LARGE_WORLDS = (16, 64)
TAIL_PLAN = [(512, True, 0.7, 1e-3), (300, False, 0.7, 1e-3), (77, True, 1.0, 1.0), (512, False, 0.7, 1e-3)]


def _spread(rng, n, R, total, shares):
    """n global ids of [0, total) whose residue mod R follows the counts `shares` (a list of R counts summing to n),
    in random order."""
    res = np.repeat(np.arange(R), shares)
    k = rng.integers(0, (total - R) // R, n)
    out = k * R + res
    rng.shuffle(out)
    return out


def _cap_ids(name, rng):
    """Global ids of the capacity cases (see CAPACITY) -> (uid, pid, nid) int32."""
    U, I = CAP_U, CAP_I
    if name.startswith("home"):          # world 3, 600 triplets: 350 (or 351) homed on rank 0
        t0 = 350 if name == "home_exact" else 351
        u = _spread(rng, 600, 3, U, [t0, 500 - t0, 100])
        p, n = rng.integers(0, I, 600), rng.integers(0, I, 600)
        return tuple(a.astype(np.int32) for a in (u, p, n))
    if name.startswith("gin"):           # world 2, 256 triplets, every item even: owner 0 takes every request
        # exact: homes 0 / 1 send 192 / 320 requests, 512 rows with no padding; over: one triplet moves to home 0,
        # 194 / 318 requests pad to 224 / 320 rows, 544 > 512
        t0 = 96 if name == "gin_exact" else 97
        home = np.array([0] * t0 + [1] * (256 - t0))
        u = rng.integers(0, U // 2 - 1, 256) * 2 + home
        p, n = rng.integers(0, I // 2 - 1, 256) * 2, rng.integers(0, I // 2 - 1, 256) * 2
        perm = rng.permutation(256)
        return tuple(a[perm].astype(np.int32) for a in (u, p, n))
    # req: world 2, 256 triplets; home 0 has 200, each with p even and n odd: 200 requests to each owner (= req_cap);
    # req_over turns one odd n even: 201 requests to owner 0
    home = np.array([0] * 200 + [1] * 56)
    u = rng.integers(0, U // 2 - 1, 256) * 2 + home
    p = rng.integers(0, I // 2 - 1, 256) * 2
    n = rng.integers(0, I // 2 - 1, 256) * 2 + 1
    if name == "req_over":
        n[0] -= 1
    perm = rng.permutation(256)
    return tuple(a[perm].astype(np.int32) for a in (u, p, n))


CAP_U, CAP_I = 1501, 2003
# name: (world, per-rank B, constructor capacities, req_cap forced on every rank, sticky code expected)
CAPACITY = {
    "home_exact": (3, 200, dict(home_cap=350), None, 0),
    "home_over": (3, 200, dict(home_cap=350), None, 2),
    "gin_exact": (2, 128, dict(gin_cap=512), None, 0),
    "gin_over": (2, 128, dict(gin_cap=512), None, 4),
    "req_exact": (2, 128, {}, 200, 0),
    "req_over": (2, 128, {}, 200, 3),
}


def test_shard_path_coverage():
    """The cases below reach both sides of every branch predicate of the six kernels, and a second grid pass of
    request, serve and compute."""
    # bench shapes: world 1 at B = SMs * 512 + 1000 (production: home_cap = 2B); world 2 at 40000 with home 0 full
    B1 = bench_world1_B()
    assert B1 > (1 << 16)                                                     # not "small": production capacities
    assert B1 > request_pass(2 * B1) and 80000 > request_pass(80000)        # two request passes (T = B1, 80000)
    assert B1 > compute_pass(128) and 80000 > compute_pass(128)
    assert 2 * B1 > serve_pass() and 80000 > serve_pass()                    # 2T lookups, ~T per owner at world 2
    # single-pass cases: the grid and the capacity cases
    assert 3 * 256 < min(request_pass(3 * 256), compute_pass(508)) and 2 * 3 * 256 < serve_pass()
    assert {route_tail(b) for b, *_ in TAIL_PLAN} == {True, False} and route_tail(B1)
    # row-width classes: each class with idle lanes, and full classes
    assert {nq_class(D) for D in GRID_D if idle_lanes(D)} == {1, 2, 4}
    assert any(not idle_lanes(D) for D in GRID_D)
    # inbox shapes, owned / staged rows and sticky codes, from the ids of the capacity cases and a grid step
    sts = []
    for name, (world, b, _, _, _) in CAPACITY.items():
        sts.append(stats(world, _cap_ids(name, np.random.default_rng(7)), CAP_U, CAP_I))
    rng = np.random.default_rng(11)
    sts.append(stats(3, [rng.integers(0, n, 3 * 256) for n in (301, 407, 407)], 301, 407))
    assert {padding_warp(s) for s in sts} == {True, False}
    assert {partial_group(s) for s in sts} == {True, False}
    for k in ("user_owned", "user_staged", "item_owned", "item_staged"):
        assert any(s[k] for s in sts), k
    assert {c[-1] for c in CAPACITY.values()} == {0, 2, 3, 4}
    gx = stats(2, _cap_ids("gin_exact", np.random.default_rng(7)), CAP_U, CAP_I)
    assert serve_rows(gx)[0] == 512                                          # exactly gin_cap
    go = stats(2, _cap_ids("gin_over", np.random.default_rng(7)), CAP_U, CAP_I)
    assert serve_rows(go)[0] == 544 and go["rc"].sum() == gx["rc"].sum()     # one triplet moved, 32 rows over
    hx = stats(3, _cap_ids("home_exact", np.random.default_rng(7)), CAP_U, CAP_I)
    assert hx["T"][0] == 350
    rx = stats(2, _cap_ids("req_exact", np.random.default_rng(7)), CAP_U, CAP_I)
    assert rx["rc"][0, 0] == rx["rc"][1, 0] == 200
    # prologue: fused (world 1) and stand-alone (world > 1); every case below announces some of its batches
    assert {w == 1 for w in BENCH.values()} == {True, False}


# ---- harness ---------------------------------------------------------------------------------------------------------
class Run:
    """A LoopbackGroup and the float64 oracle of the same global tables and optimizer slots."""

    def __init__(self, world, kind, opt_kind, U, I, D, B, seed=0, req_cap=None, **kw):
        from openrec_b200.sharded import LoopbackGroup
        self.world, self.kind, self.opt_kind, self.U, self.I, self.D = world, kind, opt_kind, U, I, D
        # Adam's step lr_t * m / (sqrt(v) + eps) is ~lr_t * sign(g) for any |g| >> eps: at eps = 1e-7 an element whose
        # summed gradient nearly cancels turns float32 rounding (and the order of the staging atomics) into a step of
        # up to 2 lr_t.  UCML x lazy Adam at the bench shape measured 6.4e-4 and 2.6e-4 table and 7.3e-4 slot errors
        # that way on an H100, on 1-7 of 6.4M elements.  eps = 1e-3 keeps the step Lipschitz in g at rounding scale.
        self.eps = 1e-3 if opt_kind == 2 else 1e-7
        self.rng = np.random.default_rng(seed)
        sc = 0.05 if kind == 0 else 0.4
        self.tabs = [self.rng.uniform(-sc, sc, s).astype(np.float32).astype(np.float64) for s in ((U, D), (I, D), (I, 1))]
        self.g = LoopbackGroup(world, U, I, D, B, kind=kind, opt_kind=opt_kind, lr=0.05, eps=self.eps, init=False, **kw)
        if req_cap is not None:          # below 2 * home_cap: the idboxes keep their size, every access stays in bounds
            for m in self.g.ranks:
                m._x.req_cap = req_cap
        self.g.load_global(*self.tabs)
        self.st = _oracle_state(*self.tabs, opt_kind)
        self.n = 0
        self.tol = 1e-5 if kind == 0 else 2e-4
        self.worst = {"table": 0.0, "slot": 0.0, "loss": 0.0}

    def close(self):
        self.g.close()

    def uniform(self, b):
        return [self.rng.integers(0, n, self.world * b).astype(np.int32) for n in (self.U, self.I, self.I)]

    def valid(self, ids):
        u, p, n = ids
        return (u >= 0) & (u < self.U) & (p >= 0) & (p < self.I) & (n >= 0) & (n < self.I)

    def prep(self, ids):
        """-> (global ids, per-rank device batches).  UCML: negatives of valid triplets resampled away from the hinge
        kink of the CURRENT oracle tables (call after the oracle took the previous step)."""
        ids = [np.asarray(a, np.int32).copy() for a in ids]
        if self.kind == 1:
            ok = self.valid(ids)
            ids[2][ok] = avoid_hinge_ties(self.rng, *self.tabs, ids[0][ok], ids[1][ok], ids[2][ok])
        b = len(ids[0]) // self.world
        dev = [tuple(torch.from_numpy(np.ascontiguousarray(a[r * b:(r + 1) * b])).cuda() for a in ids)
               for r in range(self.world)]
        return ids, dev

    def step(self, cur, nxt_fn=None, announce=False, c_loss=1.0, c_l2=1.0):
        """One step of the batch `cur` (from prep), compared with the oracle.  nxt_fn() -> global ids of the next step,
        drawn after the oracle step; announced in this step when `announce`.  -> the prepared next batch."""
        ids, dev = cur
        ok = self.valid(ids)
        self.n += 1
        frac = ok.sum() / len(ok) if self.kind == 0 else 1.0     # BPR's 1/B is over the submitted batch
        loss, l2 = O.pairwise_train_step("bpr" if self.kind == 0 else "ucml", *self.tabs, *[a[ok] for a in ids],
                                         OPT[self.opt_kind], self.st, self.n, 0.05, margin=0.5, c_loss=c_loss * frac,
                                         c_l2=c_l2, eps=self.eps)
        loss *= frac
        nxt = self.prep(nxt_fn()) if nxt_fn is not None else None
        outs = [o.cpu().numpy() for o in self.g.step(dev, c_loss, c_l2,
                                                     next_batches=nxt[1] if announce and nxt is not None else None)]
        self.g.check()
        for o in outs:
            np.testing.assert_allclose(o, [loss, l2], rtol=3e-5, atol=1e-6)
            assert np.array_equal(o, outs[0])                     # bit-identical on every rank
        self.worst["loss"] = max(self.worst["loss"], abs(outs[0][0] - loss) / max(abs(loss), 1e-30),
                                 abs(outs[0][1] - l2) / max(abs(l2), 1e-30))
        st = stats(self.world, ids, self.U, self.I)
        for r, m in enumerate(self.g.ranks):
            o4 = m._out[m.iterations % 16].cpu().numpy()
            assert o4[2] == st["bad"][r], (r, o4, st["bad"])
            assert o4[3] == st["staged"][r], (r, o4, st["staged"])
        self.compare()
        return nxt

    def compare(self):
        for a, ref, name in zip(self.g.gather_global(), self.tabs, ("user", "item", "bias")):
            a = a.cpu().numpy()
            self.worst["table"] = max(self.worst["table"], float(np.abs(a - ref).max()))
            np.testing.assert_allclose(a, ref, atol=self.tol, err_msg=name)
        for name, (got, ref) in self.slots().items():
            # slots are compared relative to their largest magnitude (Adam's v is ~1e-6 at these gradients)
            scale = max(float(np.abs(ref).max()), 1e-30)
            self.worst["slot"] = max(self.worst["slot"], float(np.abs(got - ref).max()) / scale)
            np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4 * scale, err_msg=name)

    def slots(self):
        """-> {name: (global slot gathered from the ranks with the r::R interleave, oracle slot)}"""
        R, out = self.world, {}
        for name, total in (("user", self.U), ("item", self.I), ("bias", self.I)):
            for k in range(2):
                shards = [getattr(m, name + "_slots")[k] for m in self.g.ranks]
                if shards[0] is None:
                    continue
                full = np.zeros((total, shards[0].shape[1]))
                for r, (m, s) in enumerate(zip(self.g.ranks, shards)):
                    full[r::R] = s[:(m.ru if name == "user" else m.ri)].cpu().numpy()
                out[f"{name}_s{k}"] = (full, self.st[name][k])
        return out

    def train(self, plan, gen=None):
        """plan: [(per-rank b, announce the next batch, c_loss, c_l2)]; gen(self, k, b) -> global ids of step k."""
        gen = gen or (lambda run, k, b: run.uniform(b))
        cur = self.prep(gen(self, 0, plan[0][0]))
        for k, (b, ann, cl, c2) in enumerate(plan):
            fn = (lambda k=k: gen(self, k + 1, plan[k + 1][0])) if k + 1 < len(plan) else None
            cur = self.step(cur, fn, ann, cl, c2)

    def snapshot(self):
        """float32 bits of every table and slot, global row order."""
        snap = {n: a.cpu().numpy().view(np.int32).copy() for a, n in zip(self.g.gather_global(), ("user", "item", "bias"))}
        for name, (got, _) in self.slots().items():
            snap[name] = got.astype(np.float32).view(np.int32)
        return snap


# ---- bench-scale passes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,opt_kind", BENCH_KINDS)
@pytest.mark.parametrize("shape", list(BENCH))
def test_bench_scale_passes(shape, kind, opt_kind):
    """Production capacities (home_cap = 2B, gin_cap = 4B + 32R) with second grid passes of request, serve and compute:
    the per-chunk owner counters of request, the loss accumulator carried across compute passes and serve's padding
    rows run more than once per block / warp.  Announced, announced-into and plain steps."""
    world = BENCH[shape]
    if world == 1:
        B = bench_world1_B()
        gen = None
    else:
        B = 40000
        gen = lambda run, k, b: [run.rng.integers(0, U_BIG // 2, 2 * b).astype(np.int32) * 2,
                                 run.rng.integers(0, I_BIG, 2 * b).astype(np.int32),
                                 run.rng.integers(0, I_BIG, 2 * b).astype(np.int32)]
    run = Run(world, kind, opt_kind, U_BIG, I_BIG, 128, B, seed=21 + world)
    try:
        assert run.g.ranks[0].home_cap == 2 * B                  # production sizes
        run.train([(B, True, 1.0, 1.0), (B, False, 1.0, 1.0), (B, False, 1.0, 1.0)], gen)
        print("worst", run.worst)
    finally:
        run.close()


# ---- capacity limits -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CAPACITY))
def test_capacity_limits(name):
    """One home / owner exactly on home_cap, on the padded gradient-inbox boundary, on req_cap: parity and a clean
    check().  One triplet past it: check() raises with the code of that mailbox, and every row, slot and bias that no
    triplet references keeps its bits.

    Why one past stays in bounds -- each clamp against the buffer it guards:
    * code 2: request clamps T to home_cap, and trip_u[t] / slot[2t + q] are [home_cap] / [2 home_cap] for t < T;
      tripbox reads stay at t - toff[s] < (clamped per-source count) <= batch_cap.
    * code 3: request stores only idx < req_cap (slot = -1 otherwise: compute skips the triplet); the published counts
      are clamped to req_cap, so serve reads idbox rows h * req_cap + idx < world * req_cap (lowering req_cap after
      construction only shrinks that).
    * code 4: serve serves acc = gin_cap & ~31 inbox rows (w.req and gin / ginb are [gin_cap]); compute stores a
      gradient row only where gbase + ip < gin_cap; serve drops a source whose got offset would pass got_rows
      (g + c <= got_rows)."""
    world, b, kw, req_cap, code = CAPACITY[name]
    run = Run(world, 0, 1, CAP_U, CAP_I, 64, b, seed=31, req_cap=req_cap, **kw)
    try:
        if code == 0:
            run.train([(b, True, 1.0, 1.0), (b, False, 1.0, 1.0)], lambda r, k, bb: _cap_ids(name, r.rng))
            return
        ids, dev = run.prep(_cap_ids(name, run.rng))
        before = run.snapshot()
        run.g.step(dev)
        torch.cuda.synchronize()
        codes = {int(m._flags()[ERR_WORD].item()) for m in run.g.ranks}
        assert codes - {0} == {code}, codes
        with pytest.raises(RuntimeError, match="sharded step"):
            run.g.check()
        after = run.snapshot()
        users = np.unique(ids[0])
        items = np.unique(np.concatenate([ids[1], ids[2]]))
        for key in before:
            rows = users if key.startswith("user") else items
            keep = np.ones(len(before[key]), bool)
            keep[rows] = False
            assert np.array_equal(after[key][keep], before[key][keep]), key
    finally:
        run.close()


# ---- tails and loss scales -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,opt_kind", [(0, 1), (1, 0)])
def test_tails_and_scales(kind, opt_kind):
    """Every rank passes B' < batch_cap as an announced next batch (300) and as a plain step (77), with bad ids in the
    tails; c_loss = 0.7 and c_l2 = 1e-3 on most steps."""
    def gen(run, k, b):
        ids = run.uniform(b)
        if b < 512:                      # bad ids in the tails: one per rank, of each kind
            for r in range(3):
                j = r * b + (k * 7 + r) % b
                ids[r % 3][j] = [-1, run.I, -5][r]
        return ids
    run = Run(3, kind, opt_kind, 701, 809, 64, 512, seed=41)
    try:
        run.train(TAIL_PLAN, gen)
    finally:
        run.close()


# ---- kind x optimizer x row width ------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", GRID_D)
@pytest.mark.parametrize("kind,opt_kind", GRID_KO)
def test_kind_opt_dim_grid(kind, opt_kind, D):
    """World 3, announced and plain steps alternating, every row-width class with and without idle lanes."""
    run = Run(3, kind, opt_kind, 301, 407, D, 256, seed=51 + D)
    try:
        run.train([(256, k % 2 == 0, 1.0, 1.0) for k in range(4)])
    finally:
        run.close()


# ---- large worlds ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", LARGE_WORLDS)
def test_large_worlds(world):
    """16 and 64 (= SH_MAX_R) virtual ranks at 64 triplets each; half of the users live on home 0 and half of the item
    lookups on owner 1, the rest spread over every rank."""
    U, I = 40 * world + 3, 50 * world + 7

    def gen(run, k, b):
        n = world * b
        skew = lambda total, hot: np.where(run.rng.random(n) < 0.5,
                                           run.rng.integers(0, (total - hot - 1) // world, n) * world + hot,
                                           run.rng.integers(0, total, n))
        return [skew(U, 0).astype(np.int32), skew(I, 1).astype(np.int32), skew(I, 1).astype(np.int32)]
    run = Run(world, 0, 1, U, I, 16, 64, seed=61 + world)
    try:
        run.train([(64, True, 1.0, 1.0), (64, False, 1.0, 1.0), (64, False, 1.0, 1.0)], gen)
    finally:
        run.close()


# ---- epoch wrap ------------------------------------------------------------------------------------------------------
def test_epoch_wrap_announced_world3():
    """The epoch counters of every rank's index sets start 4 below 2^31 - 1; announced steps cross the wrap of the item
    set (one epoch a step, at the 5th step) and of both user sets (one epoch every other step, at the 9th / 10th)."""
    run = Run(3, 0, 1, 97, 131, 32, 256, seed=71)
    try:
        cur = run.prep(run.uniform(256))
        cur = run.step(cur, lambda: run.uniform(256))
        for m in run.g.ranks:
            m.eng.debug_set_epoch(0x7fffffff - 4)
        for k in range(12):
            cur = run.step(cur, lambda: run.uniform(256), announce=True)
        run.step(cur)
    finally:
        run.close()


# ---- a shared handle -------------------------------------------------------------------------------------------------
def _shared_run():
    return Run(2, 0, 1, 301, 407, 64, 256, seed=81)


def _cap_B(run):
    m = run.g.ranks[0]
    return max(m.home_cap, (m.gin_cap + 1) // 2)      # lookups the sharded step's user index sets are sized for


class _SmallPairwise:
    """A BPR x Adagrad pairwise_step on tables of its own on `eng`, compared with the oracle.  prefetch() builds its
    batch index ahead on the handle's side stream; step() then checks in the dispatch record that it consumed it."""

    def __init__(self, eng, rng, B):
        U, I, D = 50, 60, 64
        self.eng, self.prefetched = eng, False
        self.host = [rng.uniform(-0.05, 0.05, s).astype(np.float32) for s in ((U, D), (I, D), (I, 1))]
        self.ids = [rng.integers(0, n, B).astype(np.int32) for n in (U, I, I)]
        self.t = [torch.from_numpy(a).cuda() for a in self.host]
        self.acc = [torch.full_like(x, 0.1) for x in self.t]
        self.tabs = [N.table(x, s) for x, s in zip(self.t, self.acc)]
        self.dids = [torch.from_numpy(a).cuda() for a in self.ids]

    def prefetch(self):
        self.eng.pairwise_prefetch(self.tabs[0], self.tabs[1], *self.dids, N.ORX_OPT_ADAGRAD)
        self.prefetched = True

    def step(self):
        self.eng.debug_dispatch_log()
        out4 = torch.zeros(4, device="cuda")
        self.eng.pairwise_step(N.ORX_PAIR_BPR, *self.tabs, *self.dids, N.opt(N.ORX_OPT_ADAGRAD, 0.05), out4)
        rec = self.eng.debug_dispatch_log()
        assert len(rec) == 1 and (rec[0].s != 0) == self.prefetched, rec
        ref = [a.astype(np.float64) for a in self.host]
        st = {k: (np.full_like(v, 0.1), None) for k, v in zip(("user", "item", "bias"), ref)}
        loss, l2 = O.pairwise_train_step("bpr", *ref, *self.ids, O.OPT_ADAGRAD, st, 1, 0.05)
        np.testing.assert_allclose(out4[:2].cpu().numpy(), [loss, l2], rtol=3e-5, atol=1e-6)
        for x, r in zip(self.t, ref):
            np.testing.assert_allclose(x.cpu().numpy(), r, atol=1e-5)


def _censor(eng, rng, n):
    """A censor of n ids on a table of its own on `eng` (it grows the handle's workspace to n lookups), compared with
    the oracle."""
    tab = rng.uniform(-1, 1, (5000, 64)).astype(np.float32)
    ids = rng.integers(0, 5000, n).astype(np.int32)
    t = torch.from_numpy(tab).cuda()
    eng.censor(t, torch.from_numpy(ids).cuda())
    ref = tab.astype(np.float64)
    O.censor(ref, ids)
    np.testing.assert_allclose(t.cpu().numpy(), ref, atol=1e-6)


ACCEPTED = ["pairwise_step", "score_topk", "score_rank", "sample_pairwise", "censor_grow", "prefetch", "epoch_wrap",
            "prefetch_across_step"]


@pytest.mark.parametrize("call", ACCEPTED)
def test_shared_handle_accepts_while_announced(call):
    """Calls on a rank's handle between an announced step and its successor -- a workspace growth, a pairwise prefetch
    consumed by its step, a wrap of the handle's index epoch included -- match their own reference, and the announced
    step and a plain one after it match the oracle.  prefetch_across_step: the announced step runs while a pairwise
    prefetch is outstanding, and the pairwise step consumes it after."""
    run = _shared_run()
    try:
        a = run.prep(run.uniform(256))
        b = run.step(a, lambda: run.uniform(256), announce=True)
        eng = run.g.ranks[0].eng
        rng = np.random.default_rng(6)
        after = None
        if call == "pairwise_step":
            _SmallPairwise(eng, rng, 200).step()
        elif call == "censor_grow":
            _censor(eng, rng, _cap_B(run) + 100)
        elif call in ("prefetch", "prefetch_across_step"):
            sp = _SmallPairwise(eng, rng, 64)
            sp.prefetch()
            if call == "prefetch":
                sp.step()
            else:
                after = sp
        elif call == "epoch_wrap":
            # the small step wraps the handle's epoch; then the announced step wraps its item set, the plain one a user set
            eng.debug_set_epoch(0x7fffffff)
            _SmallPairwise(eng, rng, 64).step()
        elif call in ("score_topk", "score_rank"):
            # same call on a fresh handle: bit-identical (the evaluation suites hold it to the oracle)
            Uq, I, D = 40, 300, 64
            ut, it = (torch.from_numpy(rng.uniform(-1, 1, s).astype(np.float32)).cuda() for s in ((Uq, D), (I, D)))
            bt = torch.from_numpy(rng.uniform(-1, 1, I).astype(np.float32)).cuda()
            uid = torch.arange(Uq, dtype=torch.int32, device="cuda")
            pos = [np.sort(rng.choice(I, 3, replace=False)) for _ in range(Uq)]
            off = torch.tensor(np.concatenate([[0], np.cumsum([len(p) for p in pos])]), dtype=torch.int64, device="cuda")
            items = torch.from_numpy(np.concatenate(pos).astype(np.int32)).cuda()
            fresh = N.Engine(0)
            try:
                if call == "score_topk":
                    f = lambda e: e.score_topk(N.ORX_SCORE_DOT, ut, uid, it, bt, off, items, 10)
                else:
                    f = lambda e: e.score_rank(N.ORX_SCORE_DOT, ut, uid, it, bt, off, items, None, None, 3, at=(5, 20))
                got, want = f(eng), f(fresh)
                for x, y in zip(got, want):
                    assert torch.equal(x.view(torch.int32), y.view(torch.int32))
            finally:
                fresh.close()
        else:
            st = _pairwise_store()
            sd = st.struct(0)
            out = [torch.full((500,), -7, dtype=torch.int32, device="cuda") for _ in range(3)]
            L.check(eng.lib.orx_sample_pairwise(eng.h, C.byref(sd), 99, 12345, 500,
                                                *(C.c_void_p(t.data_ptr()) for t in out), eng.stream()))
            for g, w in zip(out, S.sample_pairwise(st.sd, 99, 12345, 500)):
                assert np.array_equal(g.cpu().numpy(), w)
        c = run.step(b, lambda: run.uniform(256))
        if after is not None:
            after.step()
        run.step(c)
    finally:
        run.close()


def test_shared_handle_grows_after_plain_step():
    """With nothing announced, a workspace-growing call between two steps is accepted, and the steps after it match
    the oracle."""
    run = _shared_run()
    try:
        run.step(run.prep(run.uniform(256)))
        eng = run.g.ranks[0].eng
        _censor(eng, np.random.default_rng(7), _cap_B(run) + 100)
        run.step(run.prep(run.uniform(256)), lambda: run.uniform(256))
        run.step(run.prep(run.uniform(256)))
    finally:
        run.close()
