"""GPU, ONE device: the row-sharded "home-routed" step (csrc/orx_shard.cu) with R virtual ranks on one GPU equals the
single-process oracle step on the same global batch -- cross-rank duplicates, skewed homes, out-of-range ids and padded
inbox tails included.  The virtual ranks run the very kernels and peer-pointer tables of the multi-GPU step; only the
order of the launches differs (phase by phase on one stream instead of one stream per GPU)."""
import numpy as np
import pytest
import torch

import step_bar as S
from oracle import openrec_oracle as O

pytestmark = pytest.mark.gpu


def _oracle_state(user, item, bias, opt_kind):
    if opt_kind == 0:
        return {k: (None, None) for k in ("user", "item", "bias")}
    if opt_kind == 1:
        return {k: (np.full_like(v, 0.1), None) for k, v in zip(("user", "item", "bias"), (user, item, bias))}
    return {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in zip(("user", "item", "bias"), (user, item, bias))}


def _run(world, kind, opt_kind, U, I, D, B, steps=3, bad=False, seed=5, announce=False, c_l2=1.0, margin=0.5, eps=1e-7,
         beta1=0.9, beta2=0.999):
    from openrec_b200.sharded import LoopbackGroup
    rng = np.random.default_rng(seed)
    sc = 0.05 if kind == 0 else 0.4
    user, item, bias = (rng.uniform(-sc, sc, s).astype(np.float32).astype(np.float64) for s in ((U, D), (I, D), (I, 1)))
    consts = dict(eps=eps, beta1=beta1, beta2=beta2)
    g = LoopbackGroup(world, U, I, D, B, kind=kind, opt_kind=opt_kind, lr=0.05, margin=margin, init=False, **consts)
    try:
        g.load_global(user, item, bias)
        st = _oracle_state(user, item, bias, opt_kind)
        oracle_opt = {0: O.OPT_SGD, 1: O.OPT_ADAGRAD, 2: O.OPT_ADAM_LAZY}[opt_kind]
        all_ids, all_batches = [], []
        for step in range(steps):
            ids = [rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
            if bad:                                  # a few triplets carry an id out of range: skipped as a whole
                ids[0][3] = -1
                ids[1][(B + 1) % (B * world)] = I
                ids[2][2 * B - 1 if world > 1 else 5] = -7
            all_ids.append(ids)
            all_batches.append([tuple(torch.from_numpy(a[r * B:(r + 1) * B].copy()).cuda() for a in ids) for r in range(world)])
        for step in range(steps):
            ids, batches = all_ids[step], all_batches[step]
            ok = (ids[0] >= 0) & (ids[0] < U) & (ids[1] >= 0) & (ids[1] < I) & (ids[2] >= 0) & (ids[2] < I)
            # announce: the next step's route / request are issued inside this step (every second time, so that announced
            # and plain steps alternate)
            nxt = all_batches[step + 1] if announce and step + 1 < steps and step % 3 != 2 else None
            outs = [o.cpu().numpy() for o in g.step(batches, c_l2=c_l2, next_batches=nxt)]
            g.check()
            good = [a[ok] for a in ids]
            # BPR's 1/B is over the SUBMITTED batch (skipped triplets still count, as in the single-GPU step)
            frac = ok.sum() / (B * world) if kind == 0 else 1.0
            loss, l2 = O.pairwise_train_step("bpr" if kind == 0 else "ucml", user, item, bias, *good, oracle_opt, st,
                                             step + 1, 0.05, margin=margin, c_loss=frac, c_l2=c_l2, **consts)
            loss = loss * frac
            for o in outs:
                np.testing.assert_allclose(o, [loss, l2], rtol=3e-5, atol=1e-6)
                assert np.array_equal(o, outs[0])    # bit-identical on every rank
        got = [t.cpu().numpy() for t in g.gather_global()]
        tol = 1e-5 if kind == 0 else 2e-4
        for a, ref in zip(got, (user, item, bias)):
            np.testing.assert_allclose(a, ref, atol=tol)
    finally:
        g.close()


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("kind,opt_kind", [(0, 1), (0, 0), (1, 1), (0, 2)])
def test_loopback_matches_oracle(world, kind, opt_kind):
    _run(world, kind, opt_kind, U=1501, I=2003, D=128, B=1024)


def test_loopback_constants():
    """Non-default c_l2, margin, eps and betas reach the sharded step (three steps, value bar)."""
    _run(2, 1, 2, U=301, I=407, D=64, B=256, c_l2=0.25, margin=1.25, eps=1e-2, beta1=0.5, beta2=0.75)


def _step_bar(world, arm, kind, opt, D=128, B=256):
    """One step of `world` loopback ranks on the global batch of a step_bar arm (a) / (d) case, every table and slot
    judged by step_bar.Bar: the global inv_B, the cross-rank duplicate reduction and the apply of orx_shard_step."""
    from openrec_b200.sharded import LoopbackGroup
    c = S.loopback_case(world, arm, kind, opt, D, B)
    P = c.P
    g = LoopbackGroup(world, len(c.tabs["user"]), len(c.tabs["item"]), D, B, kind=S.PAIR_KINDS.index(kind),
                      opt_kind=opt, lr=c.lr, eps=P["eps"], beta1=P["beta1"], beta2=P["beta2"], margin=P["margin"],
                      init=False)
    try:
        g.load_global(*(c.tabs[n] for n in c.names))
        for m in g.ranks:
            m.iterations = c.step - 1                # the step below runs at Adam step c.step
            for name, slots in zip(c.names, (m.user_slots, m.item_slots, m.bias_slots)):
                for k, s in enumerate(c.slots[name]):
                    if s is not None:
                        local = s[m.rank::world]
                        slots[k][:len(local)] = torch.as_tensor(local, dtype=torch.float32).reshape(-1, s.shape[1])
        batches = [tuple(torch.from_numpy(a[r * B:(r + 1) * B].copy()).cuda() for a in c.ids) for r in range(world)]
        g.step(batches, c_loss=P["c_loss"], c_l2=P["c_l2"])
        g.check()
        torch.cuda.synchronize()
        got = {}
        for j, name in enumerate(c.names):
            arrs = [c.tabs[name].copy()] + [None if s is None else s.copy() for s in c.slots[name]]
            for m in g.ranks:
                n_loc = len(arrs[0][m.rank::world])
                shard = (m.local_shards()[j], *((m.user_slots, m.item_slots, m.bias_slots)[j]))
                for a, t in zip(arrs, shard):
                    if a is not None:
                        a[m.rank::world] = t[:n_loc].cpu().numpy().reshape(n_loc, -1)
            got[name] = tuple(arrs)
        S.Bar(c).check(got, f"loopback world {world}")
    finally:
        g.close()


@pytest.mark.parametrize("world,arm,kind,opt", S.loopback_specs())
def test_loopback_step_updates(world, arm, kind, opt):
    """Two ranks, arm (a) (loss only, Keras slots) and arm (d) (beta1 0.5, beta2 0.75, eps 1e-2, margin 1.25 at step 3)
    under the per-element update bar of tests/step_bar.py; the batch has users and items shared across the ranks."""
    _step_bar(world, arm, kind, opt)


@pytest.mark.parametrize("D", [8, 64, 192, 256, 512])
def test_loopback_dims(D):
    _run(3, 0, 1, U=301, I=407, D=D, B=256)


def test_loopback_heavy_duplicates_and_skew():
    # 7 users / 11 items: every row is shared across ranks, homes and owners are badly unbalanced
    _run(4, 0, 1, U=7, I=11, D=64, B=200)
    _run(2, 1, 1, U=5, I=3, D=32, B=96)


def test_loopback_bad_ids():
    _run(2, 0, 1, U=801, I=1201, D=128, B=512, bad=True)


def test_loopback_eight_ranks():
    _run(8, 0, 1, U=4001, I=9001, D=128, B=2048, steps=2)


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind,opt_kind", [(0, 1), (1, 2)])
def test_loopback_announced_batches(world, kind, opt_kind):
    """The next batch announced a step ahead (its route / request run before this step's apply; world 1 = the fused
    launch of the multi-GPU step): same results, duplicates across the two steps in flight included."""
    _run(world, kind, opt_kind, U=151, I=203, D=128, B=512, steps=7, announce=True)
    _run(world, kind, opt_kind, U=1501, I=2003, D=64, B=1024, steps=5, announce=True, bad=True)


@pytest.mark.parametrize("D", [8, 64, 192, 256, 512])
def test_loopback_announced_dims(D):
    # D <= 256: the asynchronous (shared-memory ring) form of the early serve; above: the register form
    _run(2, 0, 1, U=301, I=407, D=D, B=256, steps=4, announce=True)


def test_announced_batch_must_match():
    from openrec_b200.sharded import LoopbackGroup
    g = LoopbackGroup(1, 50, 60, 32, 64, kind=0, opt_kind=1)
    mk = lambda: [tuple(torch.randint(0, n, (64,), dtype=torch.int32, device="cuda") for n in (50, 60, 60))]
    try:
        a, b, c = mk(), mk(), mk()
        g.step(a, next_batches=b)
        with pytest.raises(ValueError):
            g.step(c)
        g.step(b)
        g.check()
    finally:
        g.close()


def test_loopback_index_epoch_wrap():
    """The epochs of the sharded step's index sets wrap at 2^31 (the item set takes one a step, each user set one every
    other step): a set is emptied on the step's stream when its epoch wraps, also while an announced batch is in
    flight."""
    from openrec_b200.sharded import LoopbackGroup
    rng = np.random.default_rng(3)
    U, I, D, B = 97, 131, 32, 256
    user, item, bias = (rng.uniform(-0.05, 0.05, s).astype(np.float32).astype(np.float64) for s in ((U, D), (I, D), (I, 1)))
    g = LoopbackGroup(1, U, I, D, B, kind=0, opt_kind=1, lr=0.05, init=False)
    try:
        g.load_global(user, item, bias)
        st = _oracle_state(user, item, bias, 1)
        batches = [[tuple(torch.from_numpy(rng.integers(0, n, B).astype(np.int32)).cuda() for n in (U, I, I))] for _ in range(14)]
        g.step(batches[0])      # builds the workspace
        O.pairwise_train_step("bpr", user, item, bias, *[t.cpu().numpy() for t in batches[0][0]], O.OPT_ADAGRAD, st, 1, 0.05)
        m = g.ranks[0]
        m.eng.debug_set_epoch(0x7fffffff - 4)      # the item set wraps at the 5th step, the user sets at the 9th / 10th
        for k in range(1, 13):
            g.step(batches[k], next_batches=batches[k + 1])
            O.pairwise_train_step("bpr", user, item, bias, *[t.cpu().numpy() for t in batches[k][0]], O.OPT_ADAGRAD, st, k + 1, 0.05)
        g.step(batches[13])
        O.pairwise_train_step("bpr", user, item, bias, *[t.cpu().numpy() for t in batches[13][0]], O.OPT_ADAGRAD, st, 14, 0.05)
        g.check()
        for a, ref in zip([t.cpu().numpy() for t in g.gather_global()], (user, item, bias)):
            np.testing.assert_allclose(a, ref, atol=1e-5)
    finally:
        g.close()


def test_shard_checkpoint_roundtrip(tmp_path):
    from openrec_b200.sharded import LoopbackGroup
    rng = np.random.default_rng(1)
    U, I, D, B, R = 301, 407, 64, 128, 2
    g = LoopbackGroup(R, U, I, D, B, kind=0, opt_kind=1, lr=0.05, seed=3)
    ids = lambda: [tuple(torch.from_numpy(rng.integers(0, n, B).astype(np.int32)).cuda() for n in (U, I, I)) for _ in range(R)]
    try:
        g.step(ids())
        for m in g.ranks:
            m.save_shard(str(tmp_path / f"shard{m.rank}.npz"))
        nxt = ids()
        ref = [o.cpu().numpy() for o in g.step(nxt)]
        ref_tabs = [t.cpu().numpy() for t in g.gather_global()]
        g2 = LoopbackGroup(R, U, I, D, B, kind=0, opt_kind=1, lr=0.05, seed=99)
        try:
            for m in g2.ranks:
                m.load_shard(str(tmp_path / f"shard{m.rank}.npz"))
            out = [o.cpu().numpy() for o in g2.step(nxt)]
            for a, b in zip(out, ref):
                np.testing.assert_allclose(a, b, rtol=1e-6)
            for a, b in zip([t.cpu().numpy() for t in g2.gather_global()], ref_tabs):
                np.testing.assert_allclose(a, b, atol=1e-7)
            with pytest.raises(ValueError):
                g2.ranks[0].load_shard(str(tmp_path / "shard1.npz"))
        finally:
            g2.close()
    finally:
        g.close()
