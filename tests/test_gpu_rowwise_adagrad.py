"""Row-wise Adagrad (ORX_OPT_ROWWISE_ADAGRAD) on the GPU: every fused step, un-fused apply and Keras model that takes it,
judged against the float64 row-wise step under tests/rowwise_bar.py's bar, plus the cases that must be exact.

Fused steps run step_bar's arms at every specialised D and one generic D (50), on mixed, all-owned and all-staged
batches and batch tails, through orx_pairwise_step, _step_host, prefetched steps and orx_pointwise_step; each asserts the
kernel variant its dispatch record shows.  Exact: untouched rows and rows whose contributions are all exact zeros are
bit-identical (value and accumulator), item-bias rows referenced once update as under ADAGRAD, a dim-1 table updates as
under ADAGRAD, and rows referenced once give the same bits on every run."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import rowwise_bar as RB
import step_bar as S
from _ranks import run_ranks
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N
from test_gpu_kernels import PAIR_OP, POINT_OP, SPECIAL_D, _check_step_dispatch, _pair_rule, _point_rule, dev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RW = N.ORX_OPT_ROWWISE_ADAGRAD
ORX_ERR_INVALID = -1          # orx.h, orx_status
KINDS = {"bpr": N.ORX_PAIR_BPR, "ucml": N.ORX_PAIR_UCML, "gmf": N.ORX_POINT_GMF, "wrmf": N.ORX_POINT_WRMF}


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def _opt(c, kind=None):
    return N.opt(c.opt if kind is None else kind, c.lr, eps=c.P["eps"], beta1=c.P["beta1"], beta2=c.P["beta2"],
                 step=c.step)


class Dev:
    """A case's tables and slots on the device (row-wise: [rows] accumulators on user / item; slots / kind given: those
    slots, checked for that optimizer)."""

    def __init__(self, c, slots=None, kind=RW):
        self.c = c
        sl = slots or c.slots
        self.t = {n: [None if x is None else dev(x) for x in (c.tabs[n], *sl[n])] for n in c.names}
        self.tt = {n: N.table(*v, kind=kind if n in RB.TABLES else None) for n, v in self.t.items()}

    def got(self):
        torch.cuda.synchronize()
        return {n: tuple(None if x is None else x.cpu().numpy().astype(np.float64) for x in v)
                for n, v in self.t.items()}


def _pair_launch(eng, c, d, entry, dids=None, kind=None):
    P = dict(margin=c.P["margin"], c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    out = torch.zeros(4, device="cuda")
    if entry == "host":
        ids = [torch.from_numpy(x).pin_memory() for x in c.ids]
        out = torch.zeros(4).pin_memory()
        eng.pairwise_step_host(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c, kind), out, **P)
        torch.cuda.synchronize()
    else:
        eng.pairwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"],
                          *(dids or [dev(x, torch.int32) for x in c.ids]), _opt(c, kind), out, **P)
    return out


def _point_launch(eng, c, d, kind=None):
    out = torch.zeros(4, device="cuda")
    eng.pointwise_step(KINDS[c.kind], d.tt["user"], d.tt["item"], d.tt["bias"], d.tt.get("w"),
                       *(dev(x, torch.int32) for x in c.ids), dev(c.label), _opt(c, kind), out,
                       c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False),
                       c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    return out


def _sid(s):
    return "-".join(map(str, s))


@pytest.mark.parametrize("spec", RB.pair_specs(), ids=_sid)
def test_rowwise_pairwise_step(eng, spec):
    entry = spec[5]
    eng.debug_dispatch_log()
    if entry == "prefetch":
        sets = []
        for k in (0, 1):
            c = RB.build(spec, k)
            d = Dev(c)
            dids = [dev(x, torch.int32) for x in c.ids]
            torch.cuda.synchronize()
            eng.pairwise_prefetch(d.tt["user"], d.tt["item"], *dids, RW, ids_ready=True)
            _pair_launch(eng, c, d, "step", dids)
            sets.append(_check_step_dispatch(eng, PAIR_OP, KINDS[c.kind], RW, c.B, c.D, "prefetch"))
            RB.RowBar(c).check(d.got(), f"prefetched step {k}")
        assert sorted(sets) == [1, 2], sets
        return
    c = RB.build(spec)
    d = Dev(c)
    _pair_launch(eng, c, d, entry)
    _check_step_dispatch(eng, PAIR_OP, KINDS[c.kind], RW, c.B, c.D, "prefetch" if entry == "host" else 0)
    RB.RowBar(c).check(d.got(), entry)


@pytest.mark.parametrize("spec", RB.point_specs(), ids=_sid)
def test_rowwise_pointwise_step(eng, spec):
    c = RB.build(spec)
    d = Dev(c)
    eng.debug_dispatch_log()
    _point_launch(eng, c, d)
    _check_step_dispatch(eng, POINT_OP, KINDS[c.kind], RW, c.B, c.D)
    RB.RowBar(c).check(d.got(), "pointwise step")


def test_rowwise_dispatch_coverage():
    """The specs above reach every (op, variant, kind, ROWWISE, specialised D or generic, index set) combination, and
    batch tails at every specialised D and the generic one."""
    dcls = lambda D: D if D in SPECIAL_D else "generic"
    kinds = dict(KINDS, wrmf_sig=N.ORX_POINT_WRMF)
    seen = set()
    for arm, kind, D, B, ids, entry in RB.pair_specs():
        for s in ((0,) if entry == "step" else (1, 2) if entry == "prefetch" else ()):
            seen.add((PAIR_OP, _pair_rule(D, RW)[0], kinds[kind], dcls(D), s))
    for arm, kind, D, B, ids, entry in RB.point_specs():
        seen.add((POINT_OP, _point_rule(D)[0], kinds[kind], dcls(D), 0))
    want = {(PAIR_OP, _pair_rule(D, RW)[0], k, dcls(D), s) for D in SPECIAL_D + (50,)
            for k in (N.ORX_PAIR_BPR, N.ORX_PAIR_UCML) for s in (0, 1, 2)}
    want |= {(POINT_OP, _point_rule(D)[0], k, dcls(D), 0) for D in SPECIAL_D + (50,)
             for k in (N.ORX_POINT_GMF, N.ORX_POINT_WRMF)}
    assert seen == want, (sorted(want - seen), sorted(seen - want))
    assert {D for _, _, D, B, _, _ in RB.pair_specs() if B % 8} >= set(SPECIAL_D + (50,)), "batch tails"
    assert {i for *_, i, _ in RB.pair_specs()} == {"mixed", "owned", "staged"}


# ---- exact cases --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", S.PAIR_KINDS)
@pytest.mark.parametrize("D", (64, 50))
def test_rowwise_zero_and_untouched_rows(eng, kind, D):
    """Arm (c): users 0 and 1 meet only clamped / inactive triplets at c_l2 = 0 (every contribution an exact zero):
    value and accumulator bit-identical, as every row the batch does not touch."""
    c = RB.to_rowwise(S.pair_case("c", kind, O.OPT_ADAGRAD, D, 203, S.spec_seed("rw_zero", kind, D)), 5)
    U = c.tabs["user"].shape[0]
    c.tabs["user"] = np.concatenate([c.tabs["user"], S.f32(np.full((9, D), 0.25))])   # rows U.. untouched
    c.slots["user"] = (np.concatenate([c.slots["user"][0], np.full(9, 0.5)]), None)
    d = Dev(c)
    _pair_launch(eng, c, d, "step")
    got = d.got()
    RB.RowBar(c).check(got, "zero rows")
    for sl in (slice(0, 2), slice(U, U + 9)):
        assert np.array_equal(got["user"][0][sl], c.tabs["user"][sl])
        assert np.array_equal(got["user"][1][sl], c.slots["user"][0][sl])
    assert (got["user"][1][2:U] != c.slots["user"][0][2:U]).any()


def _once(ids):
    u, n = np.unique(ids, return_counts=True)
    return u[n == 1]


@pytest.mark.parametrize("kind", ("bpr", "gmf"))
def test_rowwise_bias_equals_adagrad(eng, kind):
    """Item-bias rows referenced once, from the same start, update bit for bit as under ADAGRAD (element-wise, the same
    FMA); so do the accumulators of those bias rows."""
    spec = ("b", kind, 128, 237, "mixed", "step")
    runs = []
    for opt in (O.OPT_ADAGRAD, RW):
        c = RB.build(spec)
        slots = dict(c.slots)
        if opt == O.OPT_ADAGRAD:
            slots.update({n: S.init_slots(O.OPT_ADAGRAD, c.tabs[n]) for n in RB.TABLES})
        d = Dev(c, slots, opt)
        if kind == "bpr":
            _pair_launch(eng, c, d, "step", kind=opt)
        else:
            _point_launch(eng, c, d, kind=opt)
        runs.append(d.got()["bias"])
    items = c.ids[1] if kind == "gmf" else np.concatenate(c.ids[1:])
    once = _once(items)
    assert len(once) > 20
    for j in (0, 1):
        assert np.array_equal(runs[0][j][once], runs[1][j][once])


@pytest.mark.parametrize("entry", ("sparse", "bag"))
def test_rowwise_dim1_equals_adagrad(eng, entry):
    """A dim-1 table with unique ids: orx_sparse_apply / orx_bag_sparse_apply under ROWWISE is ADAGRAD bit for bit."""
    rng = np.random.default_rng(11)
    R, n = 500, 300
    var = S.f32(rng.uniform(-0.3, 0.3, (R, 1)))
    acc = S.f32(rng.uniform(0.05, 0.3, (R, 1)))
    ids = rng.permutation(R)[:n].astype(np.int32)
    vals = S.f32(rng.standard_normal((n, 1)) * 0.1)
    out = []
    for kind in (O.OPT_ADAGRAD, RW):
        t = [dev(var), dev(acc)]
        tab = N.table(t[0], t[1], kind=kind)
        o = N.opt(kind, 0.05)
        if entry == "sparse":
            eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
        else:
            eng.bag_sparse_apply(tab, dev(ids.reshape(n, 1), torch.int32), 0, 1, dev(vals), 0, o)
        torch.cuda.synchronize()
        out.append([x.cpu().numpy() for x in t])
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    assert not np.array_equal(out[1][0], var)


@pytest.mark.parametrize("spec", [("a", "bpr", 128, 4096, "mixed", "step"), ("d", "ucml", 256, 203, "mixed", "step"),
                                  ("b", "bpr", 50, 203, "mixed", "step"), ("b", "gmf", 64, 237, "mixed", "step")],
                         ids=_sid)
def test_rowwise_runs_repeat(eng, spec):
    """The same inputs twice: rows referenced once (and their accumulators) get the same bits both times."""
    runs = []
    for _ in range(2):
        c = RB.build(spec)
        d = Dev(c)
        _pair_launch(eng, c, d, "step") if c.kind in S.PAIR_KINDS else _point_launch(eng, c, d)
        runs.append(d.got())
    users = _once(c.ids[0])
    items = _once(np.concatenate(c.ids[1:]))
    for name, rows in (("user", users), ("item", items)):
        for j in (0, 1):
            assert np.array_equal(runs[0][name][j][rows], runs[1][name][j][rows]), (name, j)


# ---- un-fused applies -----------------------------------------------------------------------------------------------
def _bags(rng, B, Lmax, R):
    """Ragged bags: [B, Lmax] ids with -1 padding (some bags empty), the lookups' (id, bag) pairs."""
    sp = np.full((B, Lmax), -1, np.int32)
    for b in range(B):
        n = rng.integers(0, Lmax + 1)
        sp[b, :n] = rng.integers(0, R - 7, n)
    return sp


@pytest.mark.parametrize("D", (128, 256, 50))
@pytest.mark.parametrize("entry", ("sparse", "strided", "bag_sum", "bag_mean"))
@pytest.mark.parametrize("offset", (0, 1, 4), ids=("aligned", "table_off16", "acc_off16"))
def test_rowwise_unfused_apply(eng, D, entry, offset):
    """orx_sparse_apply / _strided / orx_bag_sparse_apply (sum and mean over ragged bags) on duplicated ids, rows R-7..
    untouched.  offset 1: the table starts 4 bytes off a 16-byte boundary (the scalar path); offset 4: only the
    accumulator does (the float4 path still runs: the accumulator is read as scalars)."""
    rng = np.random.default_rng(S.spec_seed("rw_apply", D, entry, offset))
    R, n = 97, 300
    lr, eps = float(np.float32(0.05)), float(np.float32(1e-7))
    var = S.f32(rng.uniform(-0.3, 0.3, (R, D)))
    acc = S.f32(rng.uniform(0.05, 0.3, R))
    vt = torch.zeros(R * D + 4, device="cuda")
    at = torch.zeros(R + 4, device="cuda")
    tv = vt[(1 if offset == 1 else 0):][:R * D].view(R, D)
    ta = at[(1 if offset == 4 else 0):][:R]
    tv.copy_(dev(var))
    ta.copy_(dev(acc))
    tab = N.OrxTable(tv.data_ptr(), ta.data_ptr(), None, R, D)
    o = N.opt(RW, lr, eps=eps)
    if entry in ("sparse", "strided"):
        ids = rng.integers(0, R - 7, n).astype(np.int32)
        vals = S.f32(rng.standard_normal((n, D)) * 0.1)
        if entry == "sparse":
            eng.sparse_apply(tab, dev(ids, torch.int32), dev(vals), o)
        else:
            eng.sparse_apply_strided(tab, dev(np.stack([ids[::-1], ids], 1), torch.int32), 1,
                                     dev(np.stack([np.zeros_like(vals), vals], 1)), o)
        lk_ids, lk_vals = ids, vals
    else:
        B, Lmax = 120, 5
        sp = _bags(rng, B, Lmax, R)
        dz = S.f32(rng.standard_normal((B, D)) * 0.1)
        mean = entry == "bag_mean"
        eng.bag_sparse_apply(tab, dev(sp, torch.int32), 0, Lmax, dev(dz), 1 if mean else 0, o)
        b_of, l_of = np.nonzero(sp >= 0)
        lk_ids = sp[b_of, l_of]
        cnt = (sp >= 0).sum(1).astype(np.float32)
        lk_vals = (dz[b_of] / cnt[b_of, None]).astype(np.float32).astype(np.float64) if mean else dz[b_of]
    idx, G, E = S.dedup(lk_ids, lk_vals, np.zeros_like(lk_vals), np.abs(lk_vals))
    ref, tol = RB.row_update_bar(lr, eps, (var, acc, None), idx, G, E)
    torch.cuda.synchronize()
    q = S.ratios(ref, tol, [tv.cpu().numpy(), ta.cpu().numpy(), None])
    assert max(x for x in q if x is not None) <= 1.0, (entry, D, offset, q)


def test_rowwise_step_acc_off16_keeps_float4_kernel(eng):
    """A 16-byte-aligned table whose accumulator starts off a 16-byte boundary still runs k_pair_step / k_point_step
    (the float4 kernels), and updates correctly; a table off the boundary takes the generic kernel."""
    for spec, op in ((("a", "bpr", 128, 203, "mixed", "step"), PAIR_OP), (("a", "gmf", 64, 237, "mixed", "step"), POINT_OP)):
        for off_table in (False, True):
            c = RB.build(spec)
            d = Dev(c)
            for n in RB.TABLES:
                if off_table:
                    buf = torch.zeros(d.t[n][0].numel() + 4, device="cuda")
                    d.t[n][0] = buf[1:1 + d.t[n][0].numel()].view_as(d.t[n][0]).copy_(d.t[n][0])
                else:
                    buf = torch.zeros(d.t[n][1].numel() + 4, device="cuda")
                    d.t[n][1] = buf[1:1 + d.t[n][1].numel()].copy_(d.t[n][1])
                d.tt[n] = N.OrxTable(d.t[n][0].data_ptr(), d.t[n][1].data_ptr(), None, *d.t[n][0].shape)
            eng.debug_dispatch_log()
            _pair_launch(eng, c, d, "step") if op == PAIR_OP else _point_launch(eng, c, d)
            rec = eng.debug_dispatch_log()[0]
            assert rec.variant == (L.ORX_VARIANT_STEP_GENERIC if off_table else _pair_rule(c.D, RW)[0] if op == PAIR_OP
                                   else L.ORX_VARIANT_STEP), (spec, off_table, rec)
            RB.RowBar(c).check(d.got(), f"off16 table={off_table}")


def test_rowwise_dense_apply_equals_adagrad(eng):
    """orx_dense_apply under ROWWISE is element-wise ADAGRAD, bit for bit."""
    rng = np.random.default_rng(5)
    var, acc = S.f32(rng.uniform(-1, 1, (33, 17))), S.f32(rng.uniform(0.05, 0.3, (33, 17)))
    g = S.f32(rng.standard_normal((33, 17)))
    out = []
    for kind in (O.OPT_ADAGRAD, RW):
        t = [dev(var), dev(acc)]
        eng.dense_apply(t[0], t[1], None, dev(g), N.opt(kind, 0.05))
        torch.cuda.synchronize()
        out.append([x.cpu().numpy() for x in t])
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_rowwise_refusals(eng):
    """A missing accumulator is ORX_ERR_INVALID before any device work; a [rows, D] accumulator is refused by
    native.table; orx_shard_step (the home-routed step) refuses the kind."""
    lib = L.lib()
    var = torch.zeros(10, 8, device="cuda")
    tab = N.OrxTable(var.data_ptr(), None, None, 10, 8)
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    vals = torch.zeros(4, 8, device="cuda")
    o = N.opt(RW, 0.05)
    rc = lib.orx_sparse_apply(eng.h, C.byref(tab), C.c_void_p(ids.data_ptr()), C.c_void_p(vals.data_ptr()), 4,
                              C.byref(o), None)
    assert rc == ORX_ERR_INVALID
    b = torch.zeros(10, 1, device="cuda")
    out4 = torch.zeros(4, device="cuda")
    bt = N.OrxTable(b.data_ptr(), None, None, 10, 1)
    rc = lib.orx_pairwise_step(eng.h, 0, C.byref(tab), C.byref(tab), C.byref(bt), C.c_void_p(ids.data_ptr()),
                               C.c_void_p(ids.data_ptr()), C.c_void_p(ids.data_ptr()), 4, C.c_float(0.5),
                               C.c_float(1.0), C.c_float(1.0), C.byref(o), C.c_void_p(out4.data_ptr()), None)
    assert rc == ORX_ERR_INVALID
    with pytest.raises(ValueError):
        N.table(var, torch.zeros(10, 8, device="cuda"), kind=RW)
    N.table(var, torch.zeros(10, device="cuda"), kind=RW)
    N.table(var, torch.zeros(10, 1, device="cuda"), kind=RW)


_SHARD = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "compat"), os.path.join({root!r}, "tests")]
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(0)
dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
import tensorflow as tf
from openrec.tf2.recommenders import DLRM, GMF, ShardedBPR, ShardedDLRM, ShardedGMF
from openrec_b200.tfshim.keras.optimizers import RowwiseAdagrad
from openrec_b200 import native as N
from openrec_b200 import _lib as L

# the home-routed step refuses the kind: ShardedBPR before any device work, orx_shard_step with ORX_ERR_INVALID
m = ShardedBPR(16, 16, 50, 80)
try:
    with tf.GradientTape() as tape:
        loss, l2 = m(np.zeros(8, np.int32), np.zeros(8, np.int32), np.ones(8, np.int32))
    RowwiseAdagrad().apply_gradients(zip(tape.gradient((loss, l2), m.trainable_variables), m.trainable_variables))
    raise SystemExit("ShardedBPR took RowwiseAdagrad")
except NotImplementedError:
    pass
from openrec_b200.sharded import HomeRoutedPairwise
hr = HomeRoutedPairwise(N.engine(), 0, 1, 50, 80, 16, 8, opt_kind=N.ORX_OPT_ADAGRAD)
hr.opt_kind = N.ORX_OPT_ROWWISE_ADAGRAD
ids = torch.zeros(8, dtype=torch.int32, device="cuda")
try:
    hr._call(ids, ids, ids, 1.0, 1.0, 0, 5, epoch=1)
    raise SystemExit("orx_shard_step took ROWWISE_ADAGRAD")
except RuntimeError as e:
    assert "supports SGD, Adagrad and row-sparse Adam" in str(e), e
hr.close()

def run(models, data, shard_slots):
    losses, opts = [], []
    for model in models:
        optimizer = RowwiseAdagrad(learning_rate=0.05)

        @tf.function
        def train_step(*b):
            with tf.GradientTape() as tape:
                out = model(*b)
            gradients = tape.gradient(out, model.trainable_variables)
            optimizer.apply_gradients(zip(gradients, model.trainable_variables))
            return out

        losses.append([])
        for b in data:
            out = train_step(*b)
            out = out if isinstance(out, tuple) else (out,)
            losses[-1].append([float(x.numpy()) for x in out])
        opts.append(optimizer)
    np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5, atol=1e-6)
    for s in shard_slots(opts[0]):
        assert s.dim() == 1, s.shape           # one accumulator per row on the shards
    return opts

# ShardedGMF against GMF
U, I, D = 300, 2000, 64
rng = np.random.default_rng(0)
models = [ShardedGMF(D, D, U, I, seed=3), GMF(D, D, U, I)]
for a_, b_ in zip(models[1].trainable_variables, models[0].trainable_variables):
    a_.t.copy_(b_.t)
data = [(rng.integers(0, U, 256).astype(np.int32), rng.integers(0, I, 256).astype(np.int32),
         (rng.random(256) < 0.3).astype(np.float32)) for _ in range(3)]
opts = run(models, data, lambda o: [o.slots(v)[0] for v in models[0].trainable_variables[:2]])
for a_, b_ in zip(models[0].trainable_variables, models[1].trainable_variables):
    torch.testing.assert_close(a_.t, b_.t, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(opts[0].slots(a_)[0], opts[1].slots(b_)[0], atol=1e-5, rtol=1e-5)

# ShardedDLRM against DLRM, one-hot and multi-hot
vocab, D = [3, 1, 500, 2, 90], 16
for bags in (None, [2, 1, 3, 1, 2]):
    kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[32, D], ln_top=[64, 1], interaction_mode="dlrm")
    if bags:
        kw.update(bag_sizes=bags, pooling="mean")
    models = [ShardedDLRM(**kw), DLRM(**kw)]
    models[0]._build(13); models[1]._graph(13)
    for lf, k in zip(models[1]._latent_factors, np.cumsum([0] + vocab[:-1])):
        lf.embeddings.t.copy_(models[0].embedding_shard.t[k:k + lf.embeddings.t.shape[0]])
    for a, b in zip(models[0].trainable_variables[1:], models[1].trainable_variables[len(vocab):]):
        b.t.copy_(a.t)
    cols = bags or [1] * len(vocab)
    data = [(rng.random((64, 13)).astype(np.float32),
             np.concatenate([rng.integers(0, v, (64, c)) for v, c in zip(vocab, cols)], 1).astype(np.int32),
             (rng.random(64) < 0.3).astype(np.float32)) for _ in range(3)]
    opts = run(models, data, lambda o: [o.slots(models[0].embedding_shard)[0]])
    table = torch.cat([lf.embeddings.t for lf in models[1]._latent_factors])
    torch.testing.assert_close(models[0].embedding_shard.t[:table.shape[0]], table, atol=1e-5, rtol=1e-5)
    acc = torch.cat([opts[1].slots(lf.embeddings)[0] for lf in models[1]._latent_factors])
    torch.testing.assert_close(opts[0].slots(models[0].embedding_shard)[0][:acc.shape[0]], acc, atol=1e-5, rtol=1e-5)
dist.destroy_process_group()
print("sharded ok")
"""


def test_rowwise_sharded_models_one_rank():
    """ShardedGMF and ShardedDLRM (one-hot and bag_sizes) in a one-rank NCCL group under RowwiseAdagrad match GMF and
    DLRM; ShardedBPR and orx_shard_step refuse the kind."""
    [(rc, out)] = run_ranks(1, _SHARD.format(root=ROOT), "gpu_rowwise sharded", timeout=600)
    assert rc == 0 and "sharded ok" in out, out


# ---- whole models ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    import tensorflow
    return tensorflow


def test_rowwise_bpr_model(tf):
    """BPR through tape + RowwiseAdagrad.apply_gradients: [rows] accumulators on user / item, element-wise on the item
    bias, two steps against the float64 row-wise step."""
    from openrec.tf2.recommenders import BPR
    from openrec_b200.tfshim.keras.optimizers import RowwiseAdagrad
    rng = np.random.default_rng(1)
    U, I, D, B = 60, 90, 32, 128
    model, opt = BPR(D, D, U, I), RowwiseAdagrad(learning_rate=0.05)
    tabs = [v.numpy().astype(np.float64) for v in model.trainable_variables]
    for it in range(2):
        ids = tuple(rng.integers(0, n, B).astype(np.int32) for n in (U, I, I))
        c = S.Case("bpr", O.OPT_ADAGRAD, tabs, ids, init="keras", lr=0.05, c_loss=1.0, c_l2=1.0)
        c = RB.to_rowwise(c)
        if it:
            c.slots = slots
        ref = RB.step(c)
        with tf.GradientTape() as tape:
            loss, l2 = model(*ids)
        opt.apply_gradients(zip(tape.gradient((loss, l2), model.trainable_variables), model.trainable_variables))
        for v, n in zip(model.trainable_variables, ("user", "item", "bias")):
            s0 = opt.slots(v)[0]
            assert tuple(s0.shape) == (v.shape[0],)
            np.testing.assert_allclose(v.numpy(), ref[n][0], atol=2e-6, rtol=1e-5)
            np.testing.assert_allclose(s0.cpu().numpy().reshape(-1), ref[n][1].reshape(-1), rtol=1e-5)
        tabs = [v.numpy().astype(np.float64) for v in model.trainable_variables]
        slots = {n: (S.f32(opt.slots(v)[0].cpu().numpy().reshape(ref[n][1].shape)), None)
                 for v, n in zip(model.trainable_variables, ("user", "item", "bias"))}


@pytest.mark.parametrize("bags", (False, True))
def test_rowwise_dlrm_model(tf, bags):
    """DLRM (one-hot and bag_sizes) through tape + RowwiseAdagrad: each embedding table against the float64 row-wise
    apply of its summed gradients (the un-fused DLRM backward, read from an SGD twin at lr = 1), the Dense layers as
    element-wise Adagrad."""
    from openrec.tf2.recommenders import DLRM
    from openrec_b200.tfshim.keras.optimizers import RowwiseAdagrad
    rng = np.random.default_rng(2)
    vocab, D, B = [30, 1, 200, 2], 16, 128
    sizes = [2, 1, 3, 1] if bags else None
    kw = dict(m_spa=D, ln_emb=vocab, ln_bot=[16, D], ln_top=[32, 1], interaction_mode="dlrm")
    if bags:
        kw.update(bag_sizes=sizes, pooling="sum")
    models = [DLRM(**kw), DLRM(**kw)]
    for m in models:
        m._graph(13)
    for a, b in zip(models[0].trainable_variables, models[1].trainable_variables):
        b.t.copy_(a.t)
    T = len(vocab)
    cols = sizes or [1] * T
    dense = rng.random((B, 13)).astype(np.float32)
    sparse = np.concatenate([rng.integers(0, v, (B, c)) for v, c in zip(vocab, cols)], 1).astype(np.int32)
    label = (rng.random(B) < 0.3).astype(np.float32)
    old = [v.numpy().astype(np.float64) for v in models[0].trainable_variables]
    # gradients: an SGD step at lr 1 moves each variable by minus its (deduplicated) gradient
    sgd = tf.keras.optimizers.SGD(learning_rate=1.0)
    rw = RowwiseAdagrad(learning_rate=0.05)
    for m, o in zip(models, (sgd, rw)):
        with tf.GradientTape() as tape:
            loss = m(dense, sparse, label)
        o.apply_gradients(zip(tape.gradient(loss, m.trainable_variables), m.trainable_variables))
    lr, eps = float(np.float32(0.05)), float(np.float32(1e-7))
    for j, (v1, v2) in enumerate(zip(models[0].trainable_variables, models[1].trainable_variables)):
        G = old[j] - v1.numpy().astype(np.float64)
        s0 = rw.slots(v2)[0].cpu().numpy()
        if j < T:
            assert s0.shape == (vocab[j],)
            rows = np.nonzero(np.abs(G).sum(1))[0]
            acc = np.full(vocab[j], 0.1)
            acc[rows] += (G[rows] ** 2).mean(1)
            want = old[j].copy()
            want[rows] -= lr * G[rows] / (np.sqrt(acc[rows])[:, None] + eps)
        else:
            assert s0.shape == old[j].shape
            acc = 0.1 + G * G
            want = old[j] - lr * G / (np.sqrt(acc) + eps)
        np.testing.assert_allclose(s0.reshape(acc.shape), acc, rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(v2.numpy(), want, rtol=1e-4, atol=1e-6)
