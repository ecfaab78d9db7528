"""bf16 user / item tables in the fused BPR / UCML step (orx_pairwise_step_bf16 and friends).

The rounding is pinned first: orx_debug_round_bf16 against the numpy restatement of H in tests/bf16_np.py.  A step
is then judged element by element from a bf16-exact start: the float64 oracle's value x64 and its float32 bar tol
(step_bar / rowwise_bar / momentum_bar) bound the kernel's float32 result, and the stochastic rounding is monotone in
that result for fixed random bits, so the stored bf16 value must lie in [sr(x64 - tol), sr(x64 + tol)], with the bits
H gives that element.  When both ends round alike only the neighbour H selects passes: random bits keyed on the wrong
step, row, column or table fail.  Untouched rows have tol = 0 and must keep their bits (under dense Adam every row
moves and is judged the same way).  Slots, the item bias, the loss and l2 meet the fp32 bars."""
import numpy as np
import pytest
import torch

import bf16_np as H
import momentum_bar as M
import rowwise_bar as R
import step_bar as S
from oracle import openrec_oracle as O
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

SGD, ADAGRAD, LAZY, DENSE = O.OPT_SGD, O.OPT_ADAGRAD, O.OPT_ADAM_LAZY, O.OPT_ADAM_DENSE
ROWWISE, MOM, NEST = N.ORX_OPT_ROWWISE_ADAGRAD, N.ORX_OPT_MOMENTUM, N.ORX_OPT_NESTEROV
OPTS = (SGD, ADAGRAD, LAZY, DENSE, ROWWISE, MOM, NEST)
DIMS = (32, 64, 128, 256, 50)
SEED = 0x5eed_b16


@pytest.fixture(scope="module")
def eng():
    """A handle of this module's own, destroyed when the module ends.  A handle's index workspace grows to the largest
    batch times the widest row it has stepped and is never shrunk; this module steps D = 256, so on the process-wide
    handle the large batches of later modules would size it at D = 256 too, gigabytes more than they need."""
    e = N.Engine(torch.cuda.current_device())
    yield e
    torch.cuda.synchronize()
    e.close()


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def bits_dev(a64):
    """bf16 CUDA tensor holding the bf16-exact float64 values a64"""
    b = H.rne(np.asarray(a64, np.float32)).view(np.int16)
    return torch.from_numpy(b.copy()).cuda().view(torch.bfloat16)


def bits_of(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


# ---- the rounding ---------------------------------------------------------------------------------------------------
def _specials(rng, n):
    x = rng.standard_normal(n).astype(np.float32) * np.float32(0.05)
    x[:8] = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, np.float32(3.4e38)]
    x[8:16] = np.frombuffer(np.array([0x7f800001, 0xff812345, 0x7fc00000, 0x00000001, 0x80000001, 0x007fffff,
                                      0x7f7fffff, 0xff7fffff], np.uint32).tobytes(), np.float32)
    x[16:40] = rng.uniform(-1e-38, 1e-38, 24).astype(np.float32)                  # subnormals and tiny normals
    return x


@pytest.mark.parametrize("table,seed,step,row0,dim", [(0, 0, 1, 0, 128), (1, 0, 1, 0, 128), (0, 7, 3, 999, 50),
                                                      (1, 2 ** 63 + 5, 2 ** 40, 2 ** 31 - 9, 4)])
def test_round_hook_matches_restatement(eng, table, seed, step, row0, dim):
    rng = np.random.default_rng(table + 2 * dim)
    x = _specials(rng, 1 << 15)
    got = bits_of(eng.debug_round_bf16(dev(x), row0, dim, table, seed, step))
    i = np.arange(x.size)
    want = H.sr(x, seed, step, table, row0 + i // dim, i % dim)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    ex = H.up(H.rne(x)).astype(np.float32)                    # bf16-exact inputs come back unchanged
    ex = ex[np.isfinite(ex)]
    back = bits_of(eng.debug_round_bf16(dev(ex), row0, dim, table, seed, step))
    assert np.array_equal(H.up(back), ex.astype(np.float64))


def test_round_is_unbiased(eng):
    """One value rounded with the bits of 4096 steps: the mean lies within 4 sigma of the value (fixed seed, so the
    outcome is deterministic); the kernel's bits equal the restatement's."""
    x = np.float32(0.05 + 1e-5)
    steps = np.arange(1, 4097)
    got = np.array([H.up(bits_of(eng.debug_round_bf16(dev(np.full(1, x)), 17, 128, 1, 11, int(s))))[0]
                    for s in steps[:64]])
    vals = np.array([H.up(H.sr(np.array([x]), 11, int(s), 1, 17, 0))[0] for s in steps])
    assert np.array_equal(got, vals[:64])
    ulp = 2.0 ** (np.floor(np.log2(float(x))) - 7)
    p = float(x) / ulp - np.floor(float(x) / ulp)
    sigma = ulp * np.sqrt(p * (1 - p) / len(steps))
    assert len(set(vals)) == 2
    assert abs(vals.mean() - float(x)) < 4 * sigma, (vals.mean(), float(x), sigma)


# ---- one step under the bars ----------------------------------------------------------------------------------------
def make_case(kind, opt, D, B, seed, U=None, I=None):
    base = SGD if opt in (MOM, NEST) else ADAGRAD if opt == ROWWISE else opt
    c = S.pair_case("b", kind, base, D, B, seed, U, I)
    for n in ("user", "item"):
        c.tabs[n] = H.round_table(c.tabs[n])
    if opt == ROWWISE:
        return R.to_rowwise(c, seed), R.RowBar
    if opt in (MOM, NEST):
        return M.to_momentum(c, opt, seed), M.MomBar
    return c, S.Bar


class Dev:
    def __init__(self, c, off=0):
        self.c = c
        self.t = {}
        for n in c.names:
            var = c.tabs[n]
            if n == "bias":
                v = dev(var)
            elif off:   # a table whose base sits `off` bf16 elements into its allocation (off the 8-byte boundary)
                buf = bits_dev(np.concatenate([np.zeros(off), var.reshape(-1)]))
                v = buf[off:].view(var.shape)
            else:
                v = bits_dev(var)
            self.t[n] = [v] + [None if x is None else dev(x) for x in c.slots[n]]
        self.tt = {n: (N.table if n == "bias" else N.table_bf16)(*v, kind=c.opt) for n, v in self.t.items()}

    def got(self):
        torch.cuda.synchronize()
        out = {}
        for n, v in self.t.items():
            var = v[0].float() if v[0].dtype == torch.bfloat16 else v[0]
            out[n] = tuple(None if x is None else x.cpu().numpy().astype(np.float64) for x in [var] + v[1:])
        return out


def _opt(c):
    return N.opt(c.opt, c.lr, eps=c.P["eps"], beta1=c.P["beta1"], beta2=c.P["beta2"], step=c.step)


def _kind(c):
    return N.ORX_PAIR_BPR if c.kind == "bpr" else N.ORX_PAIR_UCML


def launch(eng, c, d, entry="step", sr_seed=SEED):
    P = dict(margin=c.P["margin"], c_loss=c.P["c_loss"], c_l2=c.P["c_l2"])
    if entry == "host":
        ids = [torch.from_numpy(x).pin_memory() for x in c.ids]
        out = torch.zeros(4).pin_memory()
        eng.pairwise_step_host_bf16(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c), sr_seed, out,
                                    **P)
        torch.cuda.synchronize()
        return out.numpy().copy()
    out = torch.zeros(4, device="cuda")
    ids = [dev(x, torch.int32) for x in c.ids]
    if entry == "prefetch":
        eng.pairwise_prefetch(d.tt["user"], d.tt["item"], *ids, c.opt, ids_ready=True)
    eng.pairwise_step_bf16(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], *ids, _opt(c), sr_seed, out, **P)
    return out.cpu().numpy()


def judge(c, bar_cls, got, out4, what, sr_seed=SEED):
    bar = bar_cls(c)
    for t, n in enumerate(("user", "item")):
        ref, tol = bar.ref[n][0], bar.tol[n][0]
        rows, cols = np.indices(ref.shape)
        lo, hi = H.sr_interval(ref, tol, sr_seed, c.step, t, rows, cols)
        g = got[n][0]
        bad = (g < lo) | (g > hi)
        assert not bad.any(), f"{what} {n}: {bad.sum()} elements off, first {np.argwhere(bad)[:4].tolist()}"
        for j in (1, 2):
            if bar.tol[n][j] is not None:
                q = S.ratios((bar.ref[n][j],), (bar.tol[n][j],), (got[n][j],))[0]
                assert q <= 1.0, f"{what} {n}/s{j - 1}: err/tol {q:.3g}"
    q = S.ratios(bar.ref["bias"], bar.tol["bias"], got["bias"])
    assert all(x is None or x <= 1.0 for x in q), f"{what} bias: {q}"
    st = c.state()
    fwd = O.bpr_forward if c.kind == "bpr" else O.ucml_forward
    args = (st["user"][0], st["item"][0], st["bias"][0], *c.ids)
    loss, l2 = fwd(*args) if c.kind == "bpr" else fwd(*args, margin=c.P["margin"])
    assert abs(out4[0] - loss) <= 1e-5 * max(1.0, abs(loss)), (out4, loss)
    assert abs(out4[1] - l2) <= 1e-5 * max(1.0, abs(l2)), (out4, l2)


def _record(eng, c, B, D):
    rec = eng.debug_dispatch_log()
    assert len(rec) == 1 and rec[0].op == N.ORX_OP_PAIRWISE_STEP_BF16, rec
    assert (rec[0].ta, rec[0].tb, rec[0].m, rec[0].n) == (_kind(c), c.opt, B, D), rec
    return rec[0]


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("kind", ("bpr", "ucml"))
def test_step_bar(eng, kind, opt, D):
    c, bar = make_case(kind, opt, D, 203, S.spec_seed("bf16", kind, opt, D))
    d = Dev(c)
    eng.debug_dispatch_log()
    out4 = launch(eng, c, d)
    r = _record(eng, c, c.B, D)
    assert (r.variant == N.ORX_VARIANT_STEP_GENERIC) == (D == 50), r
    judge(c, bar, d.got(), out4, f"{kind} opt{opt} D{D}")


@pytest.mark.parametrize("opt", (SGD, ADAGRAD, ROWWISE, DENSE))
@pytest.mark.parametrize("kind", ("bpr", "ucml"))
def test_step_bar_big_batch(eng, kind, opt):
    """B = 4096 over small tables: most rows staged (the tail's rounding), the rest owned."""
    c, bar = make_case(kind, opt, 128, 4096, S.spec_seed("bf16big", kind, opt))
    d = Dev(c)
    out4 = launch(eng, c, d)
    assert out4[3] > 0
    judge(c, bar, d.got(), out4, f"{kind} opt{opt} B4096")


@pytest.mark.parametrize("opt", (SGD, ADAGRAD, ROWWISE))
def test_unaligned_tables_take_generic(eng, opt):
    c, bar = make_case("bpr", opt, 128, 203, S.spec_seed("bf16una", opt))
    d = Dev(c, off=1)
    eng.debug_dispatch_log()
    out4 = launch(eng, c, d)
    assert _record(eng, c, c.B, 128).variant == N.ORX_VARIANT_STEP_GENERIC
    judge(c, bar, d.got(), out4, f"unaligned opt{opt}")


# ---- path independence ----------------------------------------------------------------------------------------------
def _owned_with_bad_ids(c, seed):
    """Every row referenced once (owned by its triplet), plus three bad ids.  A staged row's summed gradient is a float
    atomic sum in no fixed order, so only owned rows have one float32 result, and so one rounding, on every path."""
    rng = np.random.default_rng(seed)
    B, I = c.B, c.tabs["item"].shape[0]
    uid = rng.permutation(c.tabs["user"].shape[0])[:B].astype(np.int32)
    it = rng.permutation(I)[:2 * B].astype(np.int32)
    pid, nid = it[:B].copy(), it[B:].copy()
    uid[5], pid[7], nid[9] = -1, I, -3
    c.ids = (uid, pid, nid)
    return c


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("kind", ("bpr", "ucml"))
def test_paths_bit_identical(eng, kind, opt):
    """The same batch (with bad ids) through the plain, prefetched and host entries, and twice with one seed, gives
    the same bits; another rounding seed does not.  (Under ADAM_DENSE every row is staged: its rows are rounded by the
    sweep, which sums nothing, and staged rows with a single contribution are exact too.)"""
    res = []
    for entry, seed in (("step", SEED), ("prefetch", SEED), ("host", SEED), ("step", SEED), ("step", SEED + 1)):
        c, _ = make_case(kind, opt, 128, 1000, S.spec_seed("bf16paths", kind, opt), U=3000, I=5000)
        c = _owned_with_bad_ids(c, 4)
        d = Dev(c)
        out4 = launch(eng, c, d, entry, seed)
        assert out4[2] == 3
        torch.cuda.synchronize()
        res.append([bits_of(d.t[n][0]) for n in ("user", "item")] +
                   [x.cpu().numpy() for n in ("user", "item", "bias") for x in d.t[n][1:] if x is not None] +
                   [d.t["bias"][0].cpu().numpy()])
    for r in res[1:4]:
        for a, b in zip(res[0], r):
            assert np.array_equal(a, b)
    assert not all(np.array_equal(a, b) for a, b in zip(res[0][:2], res[4][:2]))


# ---- forward, un-fused gradients, censor ----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ("bpr", "ucml"))
def test_fwd_grad_match_fp32_on_upcast(eng, kind):
    """The bf16 forward / gradient entries equal the fp32 ones on the upcast tables, bit for bit."""
    c, _ = make_case(kind, SGD, 64, 203, S.spec_seed("bf16fg", kind))
    d = Dev(c)
    f = {n: [dev(c.tabs[n])] for n in c.names}
    ft = {n: N.table(*v) for n, v in f.items()}
    ids = [dev(x, torch.int32) for x in c.ids]
    k, B, D = _kind(c), c.B, c.D
    o1, o2 = torch.zeros(4, device="cuda"), torch.zeros(4, device="cuda")
    eng.pairwise_fwd_bf16(k, d.tt["user"], d.tt["item"], d.tt["bias"], *ids, o1, margin=c.P["margin"])
    eng.pairwise_fwd(k, ft["user"], ft["item"], ft["bias"], *ids, o2, margin=c.P["margin"])
    assert torch.equal(o1, o2)
    g1 = {n: torch.empty(B, D, device="cuda") for n in ("d_user", "d_pos", "d_neg")}
    g2 = {n: torch.empty(B, D, device="cuda") for n in ("d_user", "d_pos", "d_neg")}
    eng.pairwise_grad_bf16(k, d.tt["user"], d.tt["item"], d.tt["bias"], *ids, c.P["margin"], 2.0, 0.5, **g1)
    eng.pairwise_grad(k, ft["user"], ft["item"], ft["bias"], *ids, c.P["margin"], 2.0, 0.5, **g2)
    for n in g1:
        assert torch.equal(g1[n], g2[n]), n


def test_censor_bf16(eng):
    rng = np.random.default_rng(3)
    tab = H.round_table(rng.uniform(-0.4, 0.4, (300, 50)))
    ids = rng.integers(0, 300, 500).astype(np.int32)
    t = bits_dev(tab)
    eng.censor_bf16(t, dev(ids, torch.int32), 0.1)
    ref = O.censor(tab.astype(np.float32), ids, 0.1).astype(np.float32)
    want = H.rne(ref)
    got = bits_of(t)
    # the kernel's fp32 norm and division may differ from numpy's in the last float32 bit: compare in bf16 ulps
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert diff.max() <= 1, diff.max()
    untouched = np.setdiff1d(np.arange(300), ids)
    assert np.array_equal(got[untouched], H.rne(tab[untouched].astype(np.float32)))


# ---- the model classes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt_name", ("SGD", "Adagrad", "Adam", "LazyAdam", "RowwiseAdagrad", "Momentum", "Nesterov"))
@pytest.mark.parametrize("cls_name", ("BPR", "UCML"))
def test_model_trains_through_tape(eng, cls_name, opt_name):
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tfshim import GradientTape
    from openrec_b200.tfshim.keras import optimizers as Op
    mk = {"SGD": lambda: Op.SGD(0.05), "Adagrad": lambda: Op.Adagrad(0.05), "Adam": lambda: Op.Adam(),
          "LazyAdam": lambda: Op.LazyAdam(), "RowwiseAdagrad": lambda: Op.RowwiseAdagrad(0.05),
          "Momentum": lambda: Op.SGD(0.05, momentum=0.9), "Nesterov": lambda: Op.SGD(0.05, momentum=0.9, nesterov=True)}
    model = getattr(Rm, cls_name)(32, 32, 200, 300, embedding_dtype="bfloat16", rounding_seed=4)
    opt = mk[opt_name]()
    rng = np.random.default_rng(1)
    N.engine().debug_dispatch_log()   # the models step on the process-wide handle
    for _ in range(3):
        u, p, n = (torch.from_numpy(rng.integers(0, m, 256).astype(np.int32)).cuda() for m in (200, 300, 300))
        with GradientTape() as tape:
            loss, l2 = model(u, p, n)
        grads = tape.gradient((loss, l2), model.trainable_variables)
        opt.apply_gradients(zip(grads, model.trainable_variables))
        assert np.isfinite(float(loss.numpy()))
        if cls_name == "UCML":
            model.censor_vec(u, p, n)
    rec = [r for r in N.engine().debug_dispatch_log() if r.op == N.ORX_OP_PAIRWISE_STEP_BF16]
    assert len(rec) == 3
    for v in model.trainable_variables:
        for s in opt.slots_if_any(v):
            assert s is None or s.dtype == torch.float32
    assert model.user_latent_factor.embeddings.t.dtype == torch.bfloat16
    assert model.item_bias.embeddings.t.dtype == torch.float32


@pytest.mark.parametrize("cls_name", ("BPR", "UCML"))
def test_model_early_loss_and_slices(eng, cls_name):
    """Reading the loss before apply_gradients and reading IndexedSlices values run the bf16 forward / gradients,
    which equal the fp32 entries on the upcast tables."""
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tfshim import GradientTape
    model = getattr(Rm, cls_name)(32, 32, 200, 300, embedding_dtype="bfloat16")
    ref = getattr(Rm, cls_name)(32, 32, 200, 300)
    for a, b in zip(ref.variables, model.variables):
        a.assign(b.numpy())
    rng = np.random.default_rng(2)
    u, p, n = (torch.from_numpy(rng.integers(0, m, 128).astype(np.int32)).cuda() for m in (200, 300, 300))
    with GradientTape() as tape:
        loss, l2 = model(u, p, n)
    with GradientTape() as tape2:
        loss2, l22 = ref(u, p, n)
    assert float(loss.numpy()) == float(loss2.numpy()) and float(l2.numpy()) == float(l22.numpy())
    g = tape.gradient((loss, l2), model.trainable_variables)
    g2 = tape2.gradient((loss2, l22), ref.trainable_variables)
    for a, b in zip(g, g2):
        assert np.array_equal(np.asarray(a.values.numpy()), np.asarray(b.values.numpy()))


@pytest.mark.parametrize("cls_name", ("BPR", "UCML"))
def test_scoring_equals_fp32_model_of_upcast(eng, cls_name):
    from openrec_b200.tf2 import recommenders as Rm
    model = getattr(Rm, cls_name)(32, 32, 200, 300, embedding_dtype="bfloat16")
    ref = getattr(Rm, cls_name)(32, 32, 200, 300)
    for a, b in zip(ref.variables, model.variables):
        a.assign(b.numpy())
    users = np.arange(0, 200, 3, dtype=np.int32)
    a = model.inference(users).numpy()
    b = ref.inference(users).numpy()
    assert np.array_equal(a, b)
    x, y = Rm.Retriever(k=10).recommend(model, users), Rm.Retriever(k=10).recommend(ref, users)
    for s, t in zip(x, y):
        assert np.array_equal(s.numpy(), t.numpy())
    from openrec_b200.tf2.data.dataset import Dataset
    from openrec_b200.tf2.metrics.evaluator import RankingEvaluator
    rng = np.random.default_rng(8)

    def mk(n):
        raw = np.empty(n, dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = rng.integers(0, 200, n), rng.integers(0, 300, n)
        return Dataset(raw_data=raw, total_users=200, total_items=300)
    train, val = mk(2000), mk(300)
    ra = RankingEvaluator(val, excl_datasets=[train], at=[10, 50]).evaluate(model)
    rb = RankingEvaluator(val, excl_datasets=[train], at=[10, 50]).evaluate(ref)
    for k in ("AUC", "NDCG", "Recall"):
        assert np.array_equal(ra[k].numpy(), rb[k].numpy(), equal_nan=True), k


def test_checkpoint_round_trip_and_dtype_refusal(eng, tmp_path):
    from openrec_b200.tf2 import checkpoint
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tfshim.keras import optimizers as Op
    from openrec_b200.tfshim import GradientTape
    model = Rm.BPR(32, 32, 200, 300, embedding_dtype="bfloat16", rounding_seed=9)
    opt = Op.Adagrad(0.05)
    rng = np.random.default_rng(5)
    u, p, n = (torch.from_numpy(rng.integers(0, m, 256).astype(np.int32)).cuda() for m in (200, 300, 300))
    with GradientTape() as tape:
        loss, l2 = model(u, p, n)
    opt.apply_gradients(zip(tape.gradient((loss, l2), model.trainable_variables), model.trainable_variables))
    path = str(tmp_path / "ck.npz")
    checkpoint.save(path, model, opt)
    other = Rm.BPR(32, 32, 200, 300, embedding_dtype="bfloat16")
    opt2 = Op.Adagrad(0.05)
    checkpoint.load(path, other, opt2)
    for a, b in zip(model.variables, other.variables):
        assert torch.equal(a.t.view(torch.int16) if a.t.dtype == torch.bfloat16 else a.t,
                           b.t.view(torch.int16) if b.t.dtype == torch.bfloat16 else b.t)
    for v, w in zip(model.variables, other.variables):
        for s, t in zip(opt.slots_if_any(v), opt2.slots_if_any(w)):
            assert (s is None and t is None) or torch.equal(s, t)
    with pytest.raises(ValueError, match="bfloat16"):
        checkpoint.load(path, Rm.BPR(32, 32, 200, 300))


def test_latent_factor_lookup_numpy_assign(eng):
    """A bf16 LatentFactor looks up fp32 rows equal to its upcast table; numpy() is that upcast; assign rounds to
    nearest even; optimizer slots of the table are fp32."""
    from openrec_b200.tf2.modules import LatentFactor
    from openrec_b200.tfshim.keras import optimizers as Op
    lf = LatentFactor(500, 64, name="lf", dtype="bfloat16")
    v = lf.embeddings
    assert v.t.dtype == torch.bfloat16 and v.numpy().dtype == np.float32
    ids = torch.tensor([3, 0, 499, 3, 17], dtype=torch.int32, device="cuda")
    rows = lf(ids).numpy()
    assert rows.dtype == np.float32 and np.array_equal(rows, v.numpy()[[3, 0, 499, 3, 17]])
    x = np.random.default_rng(0).standard_normal((500, 64)).astype(np.float32)
    v.assign(x)
    assert np.array_equal(bits_of(v.t), H.rne(x))
    for opt in (Op.Adagrad(0.1), Op.RowwiseAdagrad(0.1), Op.SGD(0.1, momentum=0.9), Op.LazyAdam()):
        assert all(s is None or s.dtype == torch.float32 for s in opt.slots(v))
    with pytest.raises(ValueError):
        LatentFactor(10, 4, dtype="float16")
