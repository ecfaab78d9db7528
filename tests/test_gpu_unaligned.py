"""GPU: every entry point that takes a caller's table, on tables that start off a 16-byte boundary.

orx.h allows a table, its slot rows, GMF's w and a gather's output to start at any 4-byte-aligned address (a view into
one flat parameter buffer is contiguous and may start 4 bytes past a boundary).  Each buffer below is placed in a
sentinel buffer (the NaN payload no kernel writes) at a float offset of 0, 1, 2 or 3; after the call the floats around
it must still hold the sentinel bit for bit, and the result must equal the aligned call (bit for bit where the
arithmetic is the same per element) or the float64 oracle at the bound the other suites use for that entry point.
Every entry point runs the aligned control, every caller pointer misaligned at once, and each pointer misaligned on its
own (the offset rotating through 4, 8 and 12 bytes), so a gate that forgets one pointer is caught by its own case.

Audit of the 128-bit accesses in csrc/ (float4, orx_ld4*, orx_st4*, __ldcs, __ldcg(reinterpret_cast, red.global.add.v4)
and the caller pointer each one goes through:
  gated by orx_aligned16 (orx_common.cuh), else the scalar / generic path:
    orx_gather (k_gather: tab, out), orx_gather_strided (k_gather_strided: tab, out),
    orx_censor / orx_censor_shard (orx_censor_rows8: tab; orx_censor_shard records CENSOR_SCALAR),
    orx_sparse_apply / _strided (k_sparse_apply: values, var, s0, s1), orx_bag_sparse_apply (k_bag_apply: dZ, var,
    s0, s1), the staged-row tail of every sparse step and sparse apply (orx_tail_rows: user / item var, s0, s1),
    orx_pairwise_step / _host / prefetched steps (k_pair_step: user / item var, s0, s1 -> k_pair_generic),
    orx_pointwise_step (k_point_step: user / item var, s0, s1, w -> k_point_generic),
    orx_bag_gather (tabs, out), orx_rows_segment_sum (src, out), orx_bag_segment_sum (dZ, out),
    orx_pointwise_serve (rows; the table reads are scalar), orx_pointwise_grad_rows (rows, d_rows, w),
    orx_interact_fwd / _bwd (emb, dense, demb, ddense), the Dense-layer GEMM (A, B -> SIMT);
  refused with ORX_ERR_INVALID before any device work: orx_shard_step (user / item var, s0, s1: local shards);
  scalar on caller memory: orx_pairwise_fwd / _grad / _grad_rows (k_pair_generic MODE 1), orx_pointwise_fwd / _grad,
    k_adam_sweep, orx_dense_apply, orx_fill_uniform, orx_rows_scale, orx_score_all, orx_score_* (float4 only from
    shared memory), orx_pred_loss;
  library-owned (carved 256-byte aligned): staging rows, hash slots, partials, mailboxes and orx_shard_step's got /
    gin rows."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import test_gpu_kernels as TK
from oracle import openrec_oracle as O
from openrec_b200 import _lib as L
from openrec_b200 import native as N
from test_gpu_kernels import OPTS, PairProb, PointProb, _ids, _point_ids

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD          # a quiet NaN whose payload no kernel writes
PAD = 64                       # floats of sentinel on each side of a view
STEP_D = (12, 32, 64, 128, 256)   # the specialised step kernels, and D = 12: generic step, 128-bit tail when aligned
GENERIC = L.ORX_VARIANT_STEP_GENERIC


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def vp(t):
    return C.c_void_p(t.data_ptr())


def bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


class Arena:
    """Places tensors in sentinel buffers at a float offset and checks that nothing was written around them."""

    def __init__(self):
        self.bufs = []

    def place(self, a, off):
        t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a, np.float32))
        n = t.numel()
        buf = torch.full((n + 2 * PAD,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
        v = buf[PAD + off:PAD + off + n].view(t.shape)
        v.copy_(t.to("cuda", torch.float32))
        assert v.data_ptr() % 16 == 4 * off
        self.bufs.append((buf, PAD + off, n))
        return v

    def check(self, what=""):
        for buf, s, n in self.bufs:
            b = bits(buf)
            assert (b[:s] == SENTINEL).all() and (b[s + n:] == SENTINEL).all(), f"wrote outside a view: {what}"


def layouts(ptrs, salt=0, passive=()):
    """-> [(label, {pointer: float offset})]: the aligned control; every pointer misaligned at once (passive pointers,
    read only by scalar code, too); each of `ptrs` misaligned on its own, at an offset rotating with `salt`."""
    out = [("aligned", {}), ("all", {p: 1 + (i + salt) % 3 for i, p in enumerate(tuple(ptrs) + tuple(passive))})]
    out += [(f"only {p}", {p: 1 + (i + salt) % 3}) for i, p in enumerate(ptrs)]
    return out


def every_offset(ptrs, passive=()):
    """layouts() at the three rotations: every pointer misaligned alone at 4, 8 and 12 bytes (one aligned control)."""
    return layouts(ptrs, 0, passive) + [x for salt in (1, 2) for x in layouts(ptrs, salt, passive)[1:]]


def slot_ptrs(name, opt):
    """The pointers of table `name` that optimizer opt reads: var, s0 (all but SGD), s1 (Adam)."""
    return (name,) + ((f"{name}.s0",) if opt >= 1 else ()) + ((f"{name}.s1",) if opt >= 2 else ())


def relocate(p, names, offs, arena):
    """Moves a PairProb / PointProb's tables and slots into the arena at offs[pointer] (default 0)."""
    p.tabs = [arena.place(t, offs.get(n, 0)) for t, n in zip(p.tabs, names)]
    p.dv = {n: tuple(None if s is None else arena.place(s, offs.get(f"{n}.s{j}", 0)) for j, s in enumerate(p.dv[n]))
            for n in names}
    p.tt = [N.table(t, *p.dv[n]) for t, n in zip(p.tabs, names)]


@pytest.fixture(scope="module")
def eng():
    return N.engine()


@pytest.fixture
def rules(monkeypatch):
    """The dispatch rule of test_gpu_kernels with the alignment gate: rules["vec"] = False expects STEP_GENERIC."""
    state = {"vec": True}
    pair, point = TK._pair_rule, TK._point_rule
    monkeypatch.setattr(TK, "_pair_rule", lambda D, opt: pair(D, opt) if state["vec"] else (GENERIC, 0))
    monkeypatch.setattr(TK, "_point_rule", lambda D: point(D) if state["vec"] else (GENERIC, 0))
    return state


# ---- what the parametrisation reaches --------------------------------------------------------------------------------
GATED = {   # entry point -> its gated caller pointers, as the tests below name them
    "gather": ("tab", "out"),
    "gather_strided": ("tab", "out"),
    "censor": ("tab",),
    "censor_shard": ("tab",),
    "sparse_apply": slot_ptrs("var", 2) + ("values",),
    "sparse_apply_strided": slot_ptrs("var", 2) + ("values",),
    "bag_sparse_apply": slot_ptrs("var", 2) + ("dz",),
    "pairwise_step": slot_ptrs("user", 2) + slot_ptrs("item", 2),
    "pairwise_prefetched": slot_ptrs("user", 2) + slot_ptrs("item", 2),
    "pairwise_step_host": slot_ptrs("user", 2) + slot_ptrs("item", 2),
    "pointwise_step": slot_ptrs("user", 2) + slot_ptrs("item", 2) + ("w",),
    "shard_step": slot_ptrs("user", 2) + slot_ptrs("item", 2),
}
CENSOR_OFFS = (0, 1, 2, 3)
SHARD_REFUSE = [(p, 1 + i % 3) for i, p in enumerate(GATED["shard_step"])]


def _point_ptrs(kind, opt):
    return slot_ptrs("user", opt) + slot_ptrs("item", opt) + (("w",) if kind == "gmf" else ())


# The parametrisation of the tests below, shared with test_unaligned_path_coverage: each test takes its layouts from the
# function of its entry point, over these lists.
GATHER_D = CENSOR_D = APPLY_D = FLAT_D = (12, 128)
PAIR_KINDS, POINT_KINDS = ("bpr", "ucml"), ("gmf", "wrmf")
PIPE_OPTS, PIPE_D = ("adagrad", "adam_lazy"), (64, 128)
BIAS_PTRS = ("bias", "bias.s0", "bias.s1")


def gather_layouts(entry):
    return every_offset(GATED[entry])


def censor_layouts():
    return [(f"offset {o}", {"tab": o}) for o in CENSOR_OFFS]


def apply_layouts(entry, opt, D):
    return layouts(slot_ptrs("var", opt) + GATED[entry][-1:], salt=opt + D)


def pair_layouts(opt, D):
    return layouts(slot_ptrs("user", opt) + slot_ptrs("item", opt), salt=D + opt, passive=BIAS_PTRS)


def pipe_layouts(opt):
    return every_offset(slot_ptrs("user", opt) + slot_ptrs("item", opt), BIAS_PTRS)


def point_layouts(kind, opt, D):
    passive = BIAS_PTRS + (("w.s0", "w.s1") if kind == "gmf" else ())
    return layouts(_point_ptrs(kind, opt), salt=D + opt, passive=passive)


def shard_layouts():
    return [("aligned", {})] + [(f"only {p}", {p: o}) for p, o in SHARD_REFUSE]


def _reached():
    """entry -> {pointer: set of offsets the tests below run it at}."""
    seen = {e: {p: set() for p in ps} for e, ps in GATED.items()}

    def add(entry, lays):
        for _, offs in lays:
            for p in GATED[entry]:
                seen[entry][p].add(offs.get(p, 0))

    for e in ("gather", "gather_strided"):
        add(e, gather_layouts(e))
    for e in ("censor", "censor_shard"):
        add(e, censor_layouts())
    for e in ("sparse_apply", "sparse_apply_strided", "bag_sparse_apply"):
        for opt, _ in OPTS.values():
            for D in APPLY_D:
                add(e, apply_layouts(e, opt, D))
    for opt, _ in OPTS.values():
        for D in STEP_D:
            add("pairwise_step", pair_layouts(opt, D))
            for kind in POINT_KINDS:
                add("pointwise_step", point_layouts(kind, opt, D))
    for optname in PIPE_OPTS:
        for e in ("pairwise_prefetched", "pairwise_step_host"):
            add(e, pipe_layouts(OPTS[optname][0]))
    add("shard_step", shard_layouts())
    return seen


def test_unaligned_path_coverage():
    """Every gated pointer of every entry point runs aligned and misaligned, at each of the 4-, 8- and 12-byte offsets
    somewhere in the parametrisation, and misaligned alone."""
    for entry, per in _reached().items():
        for p, offs in per.items():
            assert offs >= {0, 1, 2, 3} or (entry == "shard_step" and 0 in offs and len(offs) > 1), (entry, p, offs)
    for opt, _ in OPTS.values():      # the aligned control, all at once, and each gated pointer alone
        want = lambda ps: {"aligned", "all"} | {f"only {p}" for p in ps}
        for e in ("sparse_apply", "bag_sparse_apply"):
            assert want(slot_ptrs("var", opt) + GATED[e][-1:]) <= {lab for lab, _ in apply_layouts(e, opt, 12)}, e
        assert want(slot_ptrs("user", opt) + slot_ptrs("item", opt)) <= {lab for lab, _ in pair_layouts(opt, 12)}
        for kind in POINT_KINDS:
            assert want(_point_ptrs(kind, opt)) <= {lab for lab, _ in point_layouts(kind, opt, 12)}
    for e in ("gather", "gather_strided"):
        assert {"aligned", "all"} | {f"only {p}" for p in GATED[e]} <= {lab for lab, _ in gather_layouts(e)}


# ---- gathers ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", GATHER_D)
def test_gather_unaligned(eng, D):
    """orx_gather and orx_gather_strided bit-equal to the aligned gather (bad ids give zero rows and are counted);
    nothing around the table or the output is written."""
    rng = np.random.default_rng(seed_of("gather", D))
    rows, n = 500, 777
    tab_h = rng.standard_normal((rows, D)).astype(np.float32)
    ids = rng.integers(0, rows, n).astype(np.int32)
    ids[[3, 400]] = [-1, rows]
    did = torch.from_numpy(ids).cuda()
    want = eng.gather(torch.from_numpy(tab_h).cuda(), did)
    for label, offs in gather_layouts("gather"):
        arena = Arena()
        tab = arena.place(tab_h, offs.get("tab", 0))
        out = arena.place(np.zeros((n, D), np.float32), offs.get("out", 0))
        n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        L.check(eng.lib.orx_gather(eng.h, vp(tab), rows, D, vp(did), 0, n, vp(out), vp(n_bad), eng.stream()),
                "orx_gather")
        assert np.array_equal(bits(out), bits(want)), label
        assert n_bad.item() == 2, label
        arena.check(f"gather D={D} {label}")
    ld = 2 * D
    for label, offs in gather_layouts("gather_strided"):
        arena = Arena()
        tab = arena.place(tab_h, offs.get("tab", 0))
        out = arena.place(np.full((n, ld), 7.0, np.float32), offs.get("out", 0))
        L.check(eng.lib.orx_gather_strided(eng.h, vp(tab), rows, D, vp(did), 1, n, vp(out), ld, None, eng.stream()),
                "orx_gather_strided")
        assert np.array_equal(bits(out[:, :D]), bits(want)), label
        assert (out[:, D:] == 7.0).all(), label
        arena.check(f"gather_strided D={D} {label}")


# ---- censor ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", CENSOR_D)
def test_censor_unaligned(eng, D):
    """orx_censor and orx_censor_shard (world 1) on a table at every float offset against O.censor (bound 1e-7 +
    1e-5 |ref|, as test_gpu_misc_kernels); untouched rows keep their bits.  orx_censor_shard records CENSOR_VEC when the
    table is 16-byte aligned (D % 4 == 0, D <= 128) and CENSOR_SCALAR otherwise."""
    rng = np.random.default_rng(seed_of("censor", D))
    rows, n = 600, 1500
    tab_h = (rng.standard_normal((rows, D)) * np.where(rng.random(rows) < 0.5, 1e-3, 1.0)[:, None]).astype(np.float32)
    ids = rng.integers(0, 400, n).astype(np.int32)
    ids[:8] = [7, 7, 9, 7, 11, 11, 7, 9]
    ids[[3, 20]] = [-1, rows]
    valid = ids[(ids >= 0) & (ids < rows)]
    ref = tab_h.astype(np.float64)
    O.censor(ref, valid, 0.1)
    untouched = np.setdiff1d(np.arange(rows), valid)
    did = torch.from_numpy(ids).cuda()
    for _, offs in censor_layouts():
        off = offs["tab"]
        for shard in (False, True):
            arena = Arena()
            t = arena.place(tab_h, off)
            eng.debug_dispatch_log()
            if shard:
                eng.censor_shard(t, rows, 1, 0, did, n, n, 1)
                rec = eng.debug_dispatch_log()
                want = L.ORX_VARIANT_CENSOR_VEC if off == 0 else L.ORX_VARIANT_CENSOR_SCALAR
                assert len(rec) == 1 and rec[0].op == L.ORX_OP_CENSOR_SHARD and rec[0].variant == want, (off, rec)
            else:
                eng.censor(t, did, 0.1)
            what = f"D={D} offset={off} shard={shard}"
            np.testing.assert_allclose(t.cpu().numpy().astype(np.float64), ref, atol=1e-7, rtol=1e-5, err_msg=what)
            assert np.array_equal(bits(t)[untouched], tab_h.view(np.int32)[untouched]), what
            arena.check(what)


# ---- un-fused sparse applies -----------------------------------------------------------------------------------------
def _slot_arrays(rng, opt, shape):
    return [np.full(shape, 0.1, np.float32) if opt == 1 else (rng.random(shape) * 0.01).astype(np.float32)
            for _ in range({0: 0, 1: 1}.get(opt, 2))]


def _place_table(arena, var, slots, offs):
    t = arena.place(var, offs.get("var", 0))
    s = [arena.place(x, offs.get(f"var.s{j}", 0)) for j, x in enumerate(slots)]
    return t, s, N.table(t, *s)


@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D", APPLY_D)
def test_sparse_apply_unaligned(eng, optname, D):
    """orx_sparse_apply and orx_sparse_apply_strided on all-owned ids bit-equal to the aligned call (orx_update1 and
    orx_apply4 do the same arithmetic per element); with duplicate ids (staged rows: atomics reorder the sums) against
    O.apply_sparse within 2e-5, as test_gpu_kernels.test_sparse_apply."""
    opt, lr = OPTS[optname]
    rng = np.random.default_rng(seed_of("sparse-un", optname, D))
    rows, n, F, col = 400, 200, 3, 1
    var = rng.uniform(-0.3, 0.3, (rows, D)).astype(np.float32)
    slots = _slot_arrays(rng, opt, (rows, D))
    uniq = rng.permutation(rows)[:n].astype(np.int32)
    dup = rng.integers(0, 150, n).astype(np.int32)
    vals = rng.standard_normal((n, D)).astype(np.float32)
    vals3 = rng.standard_normal((n, F, D)).astype(np.float32)
    ids2d = rng.integers(0, rows, (n, F)).astype(np.int32)
    ids2d[:, col] = uniq

    def run(offs):
        arena, out = Arena(), []
        for how in ("plain", "strided", "dup"):
            t, s, tt = _place_table(arena, var, slots, offs)
            o = N.opt(opt, lr, step=3)
            if how == "strided":
                v = arena.place(vals3, offs.get("values", 0))
                eng.sparse_apply_strided(tt, torch.from_numpy(ids2d).cuda(), col, v, o)
            else:
                v = arena.place(vals, offs.get("values", 0))
                eng.sparse_apply(tt, torch.from_numpy(uniq if how == "plain" else dup).cuda(), v, o)
            out.append([t] + s)
        arena.check(f"sparse_apply {optname} D={D} {offs}")
        return out

    want = run({})
    ref = [var.astype(np.float64)] + [x.astype(np.float64) for x in slots] + [None] * (2 - len(slots))
    O.apply_sparse(opt, ref[0], ref[1], ref[2], dup, vals.astype(np.float64), 3, lr)
    assert apply_layouts("sparse_apply", opt, D) == apply_layouts("sparse_apply_strided", opt, D)
    for label, offs in apply_layouts("sparse_apply", opt, D):
        got = run(offs)
        for k in (0, 1):
            for g, w in zip(got[k], want[k]):
                assert np.array_equal(bits(g), bits(w)), (label, ("plain", "strided")[k])
        for j, g in enumerate(got[2]):
            np.testing.assert_allclose(g.cpu().numpy(), ref[j], atol=2e-5, rtol=1e-5, err_msg=f"{label} dup {j}")


@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D", APPLY_D)
def test_bag_sparse_apply_unaligned(eng, optname, D):
    """orx_bag_sparse_apply (sum and mean bags, every id once in the batch: all rows owned) bit-equal to the aligned
    call."""
    opt, lr = OPTS[optname]
    rng = np.random.default_rng(seed_of("bag-un", optname, D))
    rows, B, Lb, Cn, col_lo = 500, 60, 3, 5, 1
    var = rng.uniform(-0.3, 0.3, (rows, D)).astype(np.float32)
    slots = _slot_arrays(rng, opt, (rows, D))
    sparse = rng.integers(0, rows, (B, Cn)).astype(np.int32)
    sparse[:, col_lo:col_lo + Lb] = rng.permutation(rows)[:B * Lb].reshape(B, Lb)
    sparse[4, col_lo] = -1                                 # a bag with a missing id (the mean counts valid ids)
    dz = rng.standard_normal((B, D)).astype(np.float32)
    sp = torch.from_numpy(sparse).cuda()

    def run(offs):
        arena, out = Arena(), []
        for mode in (0, 1):
            t, s, tt = _place_table(arena, var, slots, offs)
            eng.bag_sparse_apply(tt, sp, col_lo, Lb, arena.place(dz, offs.get("dz", 0)), mode, N.opt(opt, lr, step=2))
            out.append([t] + s)
        arena.check(f"bag_sparse_apply {optname} D={D} {offs}")
        return out

    want = run({})
    for label, offs in apply_layouts("bag_sparse_apply", opt, D):
        for mode, (g_all, w_all) in enumerate(zip(run(offs), want)):
            for g, w in zip(g_all, w_all):
                assert np.array_equal(bits(g), bits(w)), (label, mode)


# ---- fused sparse steps ----------------------------------------------------------------------------------------------
PAIR_NAMES, POINT_NAMES = ("user", "item", "bias"), ("user", "item", "bias", "w")


def _gated(offs, ptrs):
    return any(offs.get(p, 0) for p in ptrs)


@pytest.mark.parametrize("kind", PAIR_KINDS)
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D", STEP_D)
def test_pairwise_step_unaligned(eng, rules, kind, optname, D):
    """orx_pairwise_step with "owned" batches (every row once: k_pair_step's in-register update) and "staged" batches
    (every row at least twice: the tail) on misaligned tables and slots, against O.pairwise_train_step within 1e-5
    (test_pairwise_step's bound); the step records STEP_GENERIC when a table or slot base is misaligned and its usual
    variant for the aligned control and for a misaligned bias (read by scalar code only)."""
    opt = OPTS[optname][0]
    ptrs = slot_ptrs("user", opt) + slot_ptrs("item", opt)
    B = 96
    for mode in ("owned", "staged"):
        U, I = (B + 7, 2 * B + 9) if mode == "owned" else (3 * B, 5 * B)
        rng = np.random.default_rng(seed_of("pair-un", kind, optname, D, mode))
        for label, offs in pair_layouts(opt, D):
            p = PairProb(kind, optname, D, U, I, seed_of("pair-un-tabs", kind, optname, D, mode))
            arena = Arena()
            relocate(p, PAIR_NAMES, offs, arena)
            rules["vec"] = not _gated(offs, ptrs)
            p.optname = f"{optname} {mode} {label}"
            p.step(eng, p.draw(rng, lambda r: _ids(r, mode, U, I, B)))
            arena.check(f"{kind} {p.optname} D={D}")


@pytest.mark.parametrize("kind", PAIR_KINDS)
@pytest.mark.parametrize("optname", PIPE_OPTS)
@pytest.mark.parametrize("D", PIPE_D)
def test_pairwise_pipelined_unaligned(eng, rules, kind, optname, D):
    """A prefetched step (orx_pairwise_prefetch, then the step that consumes it) and orx_pairwise_step_host on
    misaligned tables: the consumed prefetch set in the record, the gate's variant, the oracle within 1e-5."""
    opt = OPTS[optname][0]
    ptrs = slot_ptrs("user", opt) + slot_ptrs("item", opt)
    U, I, B = 150, 260, 300
    rng = np.random.default_rng(seed_of("pipe-un", kind, optname, D))
    for label, offs in pipe_layouts(opt):
        p = PairProb(kind, optname, D, U, I, seed_of("pipe-un-tabs", kind, optname, D), scale=0.05)
        arena = Arena()
        relocate(p, PAIR_NAMES, offs, arena)
        rules["vec"] = not _gated(offs, ptrs)
        p.optname = f"{optname} {label}"
        ids = p.draw(rng, lambda r: _ids(r, "mixed", U, I, B))
        dids = [torch.from_numpy(x).cuda() for x in ids]
        torch.cuda.synchronize()                         # the id tensors are complete: ids_ready=True is honest
        eng.pairwise_prefetch(p.tt[0], p.tt[1], *dids, p.opt, ids_ready=True)
        p.step(eng, ids, dids=dids, index_set="prefetch")
        ids = p.draw(rng, lambda r: _ids(r, "mixed", U, I, B))
        out, n, _ = p.run(eng, ids, host=True, index_set="prefetch")
        p.verify(out, ids, n)
        arena.check(f"{kind} {p.optname} D={D}")


@pytest.mark.parametrize("kind", POINT_KINDS)
@pytest.mark.parametrize("optname", list(OPTS))
@pytest.mark.parametrize("D", STEP_D)
def test_pointwise_step_unaligned(eng, rules, kind, optname, D):
    """orx_pointwise_step, owned and staged batches, with misaligned tables, slots and GMF's w, against
    O.pointwise_train_step within 1e-5 (test_pointwise_step's bound) and the gate's variant."""
    opt = OPTS[optname][0]
    ptrs = _point_ptrs(kind, opt)
    B = 96
    for mode in ("owned", "staged"):
        U, I = (B + 5, B + 11) if mode == "owned" else (3 * B, 3 * B)
        rng = np.random.default_rng(seed_of("point-un", kind, optname, D, mode))
        for label, offs in point_layouts(kind, opt, D):
            p = PointProb(kind, optname, D, U, I, seed_of("point-un-tabs", kind, optname, D, mode))
            arena = Arena()
            relocate(p, POINT_NAMES, offs, arena)
            rules["vec"] = not _gated(offs, ptrs)
            p.optname = f"{optname} {mode} {label}"
            p.step(eng, _point_ids(rng, mode, U, I, B), (rng.random(B) < 0.4).astype(np.float32))
            arena.check(f"{kind} {p.optname} D={D}")


# ---- the row-sharded step --------------------------------------------------------------------------------------------
def test_shard_step_refuses_unaligned():
    """orx_shard_step has no scalar path: a local shard or slot row off a 16-byte boundary returns ORX_ERR_INVALID
    naming the pointer, before any device work; the next aligned steps on the same handle match the oracle."""
    from openrec_b200.sharded import LoopbackGroup
    rng = np.random.default_rng(17)
    U, I, D, B = 301, 407, 64, 256
    user, item, bias = (rng.uniform(-0.05, 0.05, s).astype(np.float32).astype(np.float64)
                        for s in ((U, D), (I, D), (I, 1)))
    g = LoopbackGroup(1, U, I, D, B, kind=0, opt_kind=2, lr=0.05, init=False)
    try:
        g.load_global(user, item, bias)
        m = g.ranks[0]
        batches = [[tuple(torch.from_numpy(rng.integers(0, n, B).astype(np.int32)).cuda() for n in (U, I, I))]
                   for _ in range(2)]
        good = m._tabs
        for _, lay in shard_layouts()[1:]:
            (ptr, off), = lay.items()
            arena = Arena()
            name, _, slot = ptr.partition(".s")
            k = 0 if name == "user" else 1
            var, slots = (m.user, m.user_slots) if k == 0 else (m.item, m.item_slots)
            moved = [arena.place(var, off if not slot else 0)] + \
                    [arena.place(s, off if slot == str(j) else 0) for j, s in enumerate(slots[:2])]
            tabs = list(good)
            tabs[k] = N.table(*moved)
            m._tabs = tuple(tabs)
            try:
                with pytest.raises(RuntimeError, match=rf"status -1\).*{name}->{'var' if not slot else 's' + slot}"):
                    m._call(*batches[0][0], 1.0, 1.0, 0, 5, epoch=1)
            finally:
                m._tabs = good
            arena.check(ptr)
        st = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in zip(PAIR_NAMES, (user, item, bias))}
        for step, b in enumerate(batches):
            out = g.step(b)[0].cpu().numpy()
            g.check()
            ids = [t.cpu().numpy() for t in b[0]]
            loss, l2 = O.pairwise_train_step("bpr", user, item, bias, *ids, O.OPT_ADAM_LAZY, st, step + 1, 0.05,
                                             margin=0.5, c_loss=1.0)
            np.testing.assert_allclose(out[:2], [loss, l2], rtol=3e-5, atol=1e-6)
        for a, ref in zip([t.cpu().numpy() for t in g.gather_global()], (user, item, bias)):
            np.testing.assert_allclose(a, ref, atol=1e-5)
    finally:
        g.close()


# ---- the Python surface: tables as views into one flat parameter buffer ---------------------------------------------
def _flat_views(arrs, start):
    """One flat float32 tensor holding every array back to back from float `start` (odd), and a view of each."""
    total = start + sum(a.size for a in arrs)
    flat = torch.zeros(total + 8, device="cuda")
    views, o = [], start
    for a in arrs:
        v = flat[o:o + a.size].view(a.shape)
        v.copy_(torch.from_numpy(np.ascontiguousarray(a, np.float32)))
        views.append(v)
        o += a.size
    return flat, views


@pytest.mark.parametrize("D", FLAT_D)
def test_flat_parameter_buffer_step(eng, D):
    """BPR (user, item, bias + Adagrad slots) and GMF (the same + w and its slots) as views into one flat tensor, each
    at an odd float offset, through native.table(): one step equals the same model in separately allocated tensors --
    bit for bit at D = 12 (both take the generic kernel; all-owned rows: no staging sums to reorder), within 1e-5 at
    D = 128 (k_pair_step / k_point_step against the generic kernels)."""
    rng = np.random.default_rng(seed_of("flat", D))
    U, I, B = 120, 260, 100
    uid, pid, nid = (x.copy() for x in _ids(rng, "owned", U, I, B))
    iid = pid.copy()
    label = (rng.random(B) < 0.4).astype(np.float32)
    o = N.opt(L.ORX_OPT_ADAGRAD, 0.05, step=1)
    for model in ("bpr", "gmf"):
        shapes = [(U, D), (I, D), (I, 1)] + ([(1, D)] if model == "gmf" else [])
        vals = [rng.uniform(-0.3, 0.3, s).astype(np.float32) for s in shapes]
        accs = [np.full(s, 0.1, np.float32) for s in shapes]
        arrs = [x for pair in zip(vals, accs) for x in pair]
        flat, views = _flat_views(arrs, 3)
        assert all(v.data_ptr() % 16 == 12 for v in views)   # every table and slot 12 bytes past a boundary
        sep = [torch.from_numpy(a).cuda() for a in arrs]
        outs = []
        for ts in (views, sep):
            tt = [N.table(ts[2 * k], ts[2 * k + 1]) for k in range(len(shapes))]
            out = torch.zeros(4, device="cuda")
            if model == "bpr":
                eng.pairwise_step(N.ORX_PAIR_BPR, *tt, *(torch.from_numpy(x).cuda() for x in (uid, pid, nid)), o, out)
            else:
                eng.pointwise_step(N.ORX_POINT_GMF, *tt, torch.from_numpy(uid).cuda(), torch.from_numpy(iid).cuda(),
                                   torch.from_numpy(label).cuda(), o, out)
            outs.append(out)
        for a, b in zip(views + [outs[0]], sep + [outs[1]]):
            if D == 12:
                assert np.array_equal(bits(a), bits(b)), model
            else:
                np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), atol=1e-5, rtol=1e-5, err_msg=model)
