"""bf16 user / item tables in the fused GMF / WRMF step (orx_pointwise_step_bf16 and friends).

A step is judged element by element from a bf16-exact start, as tests/test_gpu_bf16_tables.py judges the pairwise
step: the float64 oracle's value x64 and its float32 bar tol (step_bar / rowwise_bar / momentum_bar) bound the kernel's
float32 result, and the stochastic rounding is monotone in that result for fixed random bits, so the stored bf16 value
must lie in [sr(x64 - tol), sr(x64 + tol)] with the bits H gives that element (table 0 = user, 1 = item).  Untouched
rows have tol = 0 and must keep their bits (under dense Adam every row moves and is judged the same way).  Slots, the
item bias, GMF's w and its slots, the loss and l2 meet the fp32 bars."""
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
KINDS = ("gmf", "wrmf", "wrmf_sig")
SEED = 0x5eed_b16f


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


# ---- one step under the bars ----------------------------------------------------------------------------------------
def make_case(kind, opt, D, B, seed, U=None, I=None):
    base = SGD if opt in (MOM, NEST) else ADAGRAD if opt == ROWWISE else opt
    c = S.point_case("b", kind[:4], base, D, B, seed, U, I, sig=kind == "wrmf_sig")
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
            if n in ("bias", "w"):
                v = dev(var)
            elif off:   # a table whose base sits `off` bf16 elements into its allocation (off the 8-byte boundary)
                buf = bits_dev(np.concatenate([np.zeros(off), var.reshape(-1)]))
                v = buf[off:].view(var.shape)
            else:
                v = bits_dev(var)
            self.t[n] = [v] + [None if x is None else dev(x) for x in c.slots[n]]
        # the item bias and GMF's w keep element-wise slots under every optimizer
        self.tt = {n: N.table(*v) if n in ("bias", "w") else N.table_bf16(*v, kind=c.opt) for n, v in self.t.items()}

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
    return N.ORX_POINT_GMF if c.kind == "gmf" else N.ORX_POINT_WRMF


def _point_args(c):
    return c.P.get("a", 1.0), c.P.get("b", 1.0), c.P.get("sig", False)


def launch(eng, c, d, sr_seed=SEED):
    out = torch.zeros(4, device="cuda")
    uid, iid = (dev(x, torch.int32) for x in c.ids)
    eng.pointwise_step_bf16(_kind(c), d.tt["user"], d.tt["item"], d.tt["bias"], d.tt.get("w"), uid, iid,
                            dev(c.label), _opt(c), sr_seed, out, *_point_args(c), c_loss=c.P["c_loss"],
                            c_l2=c.P["c_l2"])
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
    for n in c.names[2:]:   # the item bias and GMF's w, with their slots: float32 bars
        q = S.ratios(bar.ref[n], bar.tol[n], got[n])
        assert all(x is None or x <= 1.0 for x in q), f"{what} {n}: {q}"
    st = c.state()
    if c.kind == "gmf":
        loss, l2 = O.gmf_forward(st["user"][0], st["item"][0], st["bias"][0], st["w"][0], *c.ids, c.label)
    else:
        a, b, sig = _point_args(c)
        loss, l2 = O.wrmf_forward(st["user"][0], st["item"][0], st["bias"][0], *c.ids, c.label, a, b, sig)
    assert abs(out4[0] - loss) <= 1e-5 * max(1.0, abs(loss)), (out4, loss)
    assert abs(out4[1] - l2) <= 1e-5 * max(1.0, abs(l2)), (out4, l2)


def _record(eng, c, B, D):
    rec = eng.debug_dispatch_log()
    assert len(rec) == 1 and rec[0].op == N.ORX_OP_POINTWISE_STEP_BF16, rec
    assert (rec[0].ta, rec[0].tb, rec[0].m, rec[0].n) == (_kind(c), c.opt, B, D), rec
    return rec[0]


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("kind", KINDS)
def test_step_bar(eng, kind, opt, D):
    c, bar = make_case(kind, opt, D, 203, S.spec_seed("bf16pt", kind, opt, D))
    d = Dev(c)
    eng.debug_dispatch_log()
    out4 = launch(eng, c, d)
    r = _record(eng, c, c.B, D)
    assert (r.variant == N.ORX_VARIANT_STEP_GENERIC) == (D == 50), r
    judge(c, bar, d.got(), out4, f"{kind} opt{opt} D{D}")


@pytest.mark.parametrize("opt", (SGD, ADAGRAD, ROWWISE, DENSE))
@pytest.mark.parametrize("kind", KINDS)
def test_step_bar_big_batch(eng, kind, opt):
    """B = 4096 over small tables: most rows staged (the tail's rounding), the rest owned."""
    c, bar = make_case(kind, opt, 128, 4096, S.spec_seed("bf16ptbig", kind, opt))
    d = Dev(c)
    out4 = launch(eng, c, d)
    assert out4[3] > 0
    judge(c, bar, d.got(), out4, f"{kind} opt{opt} B4096")


@pytest.mark.parametrize("opt", (SGD, ADAGRAD, ROWWISE))
@pytest.mark.parametrize("kind", ("gmf", "wrmf"))
def test_unaligned_tables_take_generic(eng, kind, opt):
    c, bar = make_case(kind, opt, 128, 203, S.spec_seed("bf16ptuna", kind, opt))
    d = Dev(c, off=1)
    eng.debug_dispatch_log()
    out4 = launch(eng, c, d)
    assert _record(eng, c, c.B, 128).variant == N.ORX_VARIANT_STEP_GENERIC
    judge(c, bar, d.got(), out4, f"unaligned {kind} opt{opt}")


# ---- repeatability --------------------------------------------------------------------------------------------------
def _owned_with_bad_ids(c, seed):
    """Every row referenced once (owned by its sample), plus three bad ids.  A staged row's summed gradient is a float
    atomic sum in no fixed order, so only owned rows have one float32 result, and so one rounding, on every run."""
    rng = np.random.default_rng(seed)
    B = c.B
    uid = rng.permutation(c.tabs["user"].shape[0])[:B].astype(np.int32)
    iid = rng.permutation(c.tabs["item"].shape[0])[:B].astype(np.int32)
    uid[5], iid[7], uid[9] = -1, c.tabs["item"].shape[0] + 3, c.tabs["user"].shape[0]
    c.ids = (uid, iid)
    return c


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("kind", ("gmf", "wrmf"))
def test_repeat_bit_identical(eng, kind, opt):
    """The same batch (with bad ids) stepped twice with one seed gives the same table, slot and bias bits; another
    rounding seed changes the table bits.  (Under ADAM_DENSE every row is staged: its rows are rounded by the sweep,
    which sums nothing, and staged rows with a single contribution are exact too.)  GMF's w reads the same in both
    runs' table updates, which use its pre-step value; its own gradient is a float atomic sum over the batch in no
    fixed order, so w and its slots are held to float32 rounding of that sum instead of to their bits."""
    res, ws = [], []
    for seed in (SEED, SEED, SEED + 1):
        c, _ = make_case(kind, opt, 128, 1000, S.spec_seed("bf16ptrep", kind, opt), U=3000, I=5000)
        c = _owned_with_bad_ids(c, 4)
        d = Dev(c)
        out4 = launch(eng, c, d, seed)
        assert out4[2] == 3
        torch.cuda.synchronize()
        res.append([bits_of(d.t[n][0]) for n in ("user", "item")] +
                   [x.cpu().numpy() for n in ("user", "item", "bias") for x in d.t[n][1:] if x is not None] +
                   [d.t["bias"][0].cpu().numpy()])
        ws.append([x.cpu().numpy() for x in d.t.get("w", []) if x is not None])
    for a, b in zip(res[0], res[1]):
        assert np.array_equal(a, b)
    for a, b in zip(ws[0], ws[1]):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-7)
    assert not all(np.array_equal(a, b) for a, b in zip(res[0][:2], res[2][:2]))


# ---- forward and un-fused gradients ---------------------------------------------------------------------------------
def contraction_ok(got, want, own, c_l2):
    """A lookup's gradient element g w x + c_l2 y (y the lookup's own row) with its two products fused into the sum in
    either order: nvcc picks one per instance, and even per unrolled iteration of the fp32 kernel, so the bf16 and fp32
    entries may differ by the rounding of one product.  |g w x| <= |d| + |c_l2 y| bounds it."""
    got, want, own = (np.asarray(x, np.float64) for x in (got, want, own))
    return np.all(np.abs(got - want) <= 2.0 ** -23 * (np.abs(want) + 2 * abs(c_l2) * np.abs(own)))


@pytest.mark.parametrize("D", (64, 50))
@pytest.mark.parametrize("kind", KINDS)
def test_fwd_grad_match_fp32_on_upcast(eng, kind, D):
    """The bf16 forward entry equals the fp32 one on the upcast tables bit for bit, as do the gradient entry's per-sample
    scalars (d_bias, g_out); its gradient rows and GMF's d_w meet the fp32 entry's up to the FMA contraction
    (contraction_ok) and the float atomic order of d_w's batch sum."""
    c, _ = make_case(kind, SGD, D, 203, S.spec_seed("bf16ptfg", kind, D))
    d = Dev(c)
    fp = {n: dev(c.tabs[n]) for n in c.names}   # kept alive: a table struct holds only the raw pointer
    ft = {n: N.table(v) for n, v in fp.items()}
    ids = [dev(x, torch.int32) for x in c.ids]
    lab = dev(c.label)
    k, B, a, b, sig = _kind(c), c.B, *_point_args(c)
    w_bf, w_fp = d.tt.get("w"), ft.get("w")
    o1, o2 = torch.zeros(4, device="cuda"), torch.zeros(4, device="cuda")
    eng.pointwise_fwd_bf16(k, d.tt["user"], d.tt["item"], d.tt["bias"], w_bf, *ids, lab, o1, a, b, sig)
    eng.pointwise_fwd(k, ft["user"], ft["item"], ft["bias"], w_fp, *ids, lab, o2, a, b, sig)
    assert torch.equal(o1, o2)
    shapes = {"d_user": (B, D), "d_item": (B, D), "d_bias": (B,), "g_out": (B,)}
    if c.kind == "gmf":
        shapes["d_w"] = (D,)
    g1 = {n: torch.full(s, float("nan"), device="cuda") for n, s in shapes.items()}
    g2 = {n: torch.full(s, float("nan"), device="cuda") for n, s in shapes.items()}
    eng.pointwise_grad_bf16(k, d.tt["user"], d.tt["item"], d.tt["bias"], w_bf, *ids, lab, a, b, sig, 2.0, 0.5, **g1)
    eng.pointwise_grad(k, ft["user"], ft["item"], ft["bias"], w_fp, *ids, lab, a, b, sig, 2.0, 0.5, **g2)
    for n in ("d_bias", "g_out"):
        assert torch.equal(g1[n], g2[n]), n
    assert contraction_ok(g1["d_user"].cpu(), g2["d_user"].cpu(), c.tabs["user"][c.ids[0]], 0.5)
    assert contraction_ok(g1["d_item"].cpu(), g2["d_item"].cpu(), c.tabs["item"][c.ids[1]], 0.5)
    if "d_w" in g1:   # summed over the batch by float atomics: the same terms in another order
        torch.testing.assert_close(g1["d_w"], g2["d_w"], rtol=1e-5, atol=1e-6)


# ---- the model classes ----------------------------------------------------------------------------------------------
def _batch(rng, n, U=200, I=300):
    u, i = (torch.from_numpy(rng.integers(0, m, n).astype(np.int32)).cuda() for m in (U, I))
    return u, i, torch.from_numpy((rng.random(n) < 0.4).astype(np.float32)).cuda()


def _pair(cls_name, **kw):
    """A bf16 model and an fp32 model holding its upcast values."""
    from openrec_b200.tf2 import recommenders as Rm
    model = getattr(Rm, cls_name)(32, 32, 200, 300, embedding_dtype="bfloat16", **kw)
    ref = getattr(Rm, cls_name)(32, 32, 200, 300)
    for a, b in zip(ref.variables, model.variables):
        a.assign(b.numpy())
    return model, ref


@pytest.mark.parametrize("opt_name", ("SGD", "Adagrad", "Adam", "LazyAdam", "RowwiseAdagrad", "Momentum", "Nesterov"))
@pytest.mark.parametrize("cls_name", ("GMF", "WRMF"))
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
    before = model.user_latent_factor.embeddings.t.clone()
    N.engine().debug_dispatch_log()   # the models step on the process-wide handle
    for _ in range(3):
        u, i, lab = _batch(rng, 256)
        with GradientTape() as tape:
            loss, l2 = model(u, i, lab)
        grads = tape.gradient((loss, l2), model.trainable_variables)
        opt.apply_gradients(zip(grads, model.trainable_variables))
        assert np.isfinite(float(loss.numpy()))
    rec = [r for r in N.engine().debug_dispatch_log() if r.op in (N.ORX_OP_POINTWISE_STEP_BF16, N.ORX_OP_POINTWISE_STEP)]
    assert len(rec) == 3 and all(r.op == N.ORX_OP_POINTWISE_STEP_BF16 for r in rec), rec
    for v in model.trainable_variables:
        for s in opt.slots_if_any(v):
            assert s is None or s.dtype == torch.float32
    assert model.user_latent_factor.embeddings.t.dtype == torch.bfloat16
    assert model.item_latent_factor.embeddings.t.dtype == torch.bfloat16
    assert model.item_bias.embeddings.t.dtype == torch.float32
    if cls_name == "GMF":
        assert model.mlp.layers[0].kernel.t.dtype == torch.float32
    assert not torch.equal(before, model.user_latent_factor.embeddings.t)


@pytest.mark.parametrize("cls_name", ("GMF", "WRMF"))
def test_model_early_loss_and_slices(eng, cls_name):
    """Reading the loss before apply_gradients and reading IndexedSlices values run the bf16 forward / gradients: the
    loss equals the fp32 model's bit for bit, the slices' indices too, their values up to the FMA contraction."""
    from openrec_b200.tfshim import GradientTape
    model, ref = _pair(cls_name)
    u, i, lab = _batch(np.random.default_rng(2), 128)
    with GradientTape() as tape:
        loss, l2 = model(u, i, lab)
    with GradientTape() as tape2:
        loss2, l22 = ref(u, i, lab)
    assert float(loss.numpy()) == float(loss2.numpy()) and float(l2.numpy()) == float(l22.numpy())
    g = tape.gradient((loss, l2), model.trainable_variables)
    g2 = tape2.gradient((loss2, l22), ref.trainable_variables)
    for a, b, v in zip(g, g2, ref.trainable_variables):
        if getattr(a, "indices", None) is not None:
            idx = np.asarray(a.indices.numpy())
            assert np.array_equal(idx, np.asarray(b.indices.numpy()))
            own = v.numpy()[idx].reshape(len(idx), -1)
            assert contraction_ok(np.asarray(a.values.numpy()).reshape(own.shape),
                                  np.asarray(b.values.numpy()).reshape(own.shape), own, 1.0), v.name
        else:   # GMF's w: a dense gradient summed over the batch by float atomics
            np.testing.assert_allclose(np.asarray(a.values.numpy()), np.asarray(b.values.numpy()), rtol=1e-5,
                                       atol=1e-6)


@pytest.mark.parametrize("cls_name", ("GMF", "WRMF"))
def test_scoring_equals_fp32_model_of_upcast(eng, cls_name):
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tf2.data.dataset import Dataset
    from openrec_b200.tf2.metrics.evaluator import CandidateEvaluator, RankingEvaluator
    model, ref = _pair(cls_name)
    users = np.arange(0, 200, 3, dtype=np.int32)
    assert np.array_equal(model.inference(users).numpy(), ref.inference(users).numpy())
    x, y = Rm.Retriever(k=10).recommend(model, users), Rm.Retriever(k=10).recommend(ref, users)
    for s, t in zip(x, y):
        assert np.array_equal(s.numpy(), t.numpy())
    rng = np.random.default_rng(8)

    def mk(n, **kw):
        raw = np.empty(n, dtype=[("user_id", np.int32), ("item_id", np.int32)])
        raw["user_id"], raw["item_id"] = rng.integers(0, 200, n), rng.integers(0, 300, n)
        return Dataset(raw_data=raw, total_users=200, total_items=300, **kw)
    train, val = mk(2000), mk(300)
    ra = RankingEvaluator(val, excl_datasets=[train], at=[10, 50]).evaluate(model)
    rb = RankingEvaluator(val, excl_datasets=[train], at=[10, 50]).evaluate(ref)
    for k in ("AUC", "NDCG", "Recall"):
        assert np.array_equal(ra[k].numpy(), rb[k].numpy(), equal_nan=True), k
    np.random.seed(11)
    listed = mk(300, num_negatives=20)
    ca = CandidateEvaluator(listed, excl_datasets=[train], at=[10], batch_size=64).evaluate(model)
    cb = CandidateEvaluator(listed, excl_datasets=[train], at=[10], batch_size=64).evaluate(ref)
    for k in ("AUC", "NDCG", "Recall"):
        assert np.array_equal(ca[k].numpy(), cb[k].numpy(), equal_nan=True), k


@pytest.mark.parametrize("cls_name", ("GMF", "WRMF"))
def test_checkpoint_round_trip_and_dtype_refusal(eng, tmp_path, cls_name):
    from openrec_b200.tf2 import checkpoint
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tfshim import GradientTape
    from openrec_b200.tfshim.keras import optimizers as Op
    cls = getattr(Rm, cls_name)
    model = cls(32, 32, 200, 300, embedding_dtype="bfloat16", rounding_seed=9)
    opt = Op.Adagrad(0.05)
    u, i, lab = _batch(np.random.default_rng(5), 256)
    with GradientTape() as tape:
        loss, l2 = model(u, i, lab)
    opt.apply_gradients(zip(tape.gradient((loss, l2), model.trainable_variables), model.trainable_variables))
    path = str(tmp_path / "ck.npz")
    checkpoint.save(path, model, opt)
    other = cls(32, 32, 200, 300, embedding_dtype="bfloat16")
    opt2 = Op.Adagrad(0.05)
    checkpoint.load(path, other, opt2)
    for a, b in zip(model.variables, other.variables):
        assert a.t.dtype == b.t.dtype
        assert torch.equal(a.t.view(torch.int16) if a.t.dtype == torch.bfloat16 else a.t,
                           b.t.view(torch.int16) if b.t.dtype == torch.bfloat16 else b.t)
    for v, w in zip(model.variables, other.variables):
        for s, t in zip(opt.slots_if_any(v), opt2.slots_if_any(w)):
            assert (s is None and t is None) or torch.equal(s, t)
    with pytest.raises(ValueError, match="bfloat16"):
        checkpoint.load(path, cls(32, 32, 200, 300))
    fp = str(tmp_path / "fp.npz")
    checkpoint.save(fp, cls(32, 32, 200, 300))
    with pytest.raises(ValueError, match="bfloat16|float32"):
        checkpoint.load(fp, cls(32, 32, 200, 300, embedding_dtype="bfloat16"))
