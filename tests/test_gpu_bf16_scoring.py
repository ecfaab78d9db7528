"""Scoring bf16 tables in place: orx_score_all_bf16, orx_score_rank_bf16, orx_score_rank_listed_bf16 and
orx_score_topk_bf16, and the models that reach them through native.Engine.

The bf16 entries widen each element exactly and keep the fp32 arithmetic and its order, so the oracle is the fp32 entry
point called on the float32 upcast of the same tables, and every output is compared as bits (int32 views: NaN
positions and payloads, -0.0 and +-inf included)."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import far_tables as F
from openrec_b200 import _lib
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

DOT, SQ = N.ORX_SCORE_DOT, N.ORX_SCORE_NEG_SQDIST
KINDS = [pytest.param(DOT, id="dot"), pytest.param(SQ, id="neg_sqdist")]
INT32_MAX = 2 ** 31 - 1
GB = 1 << 30
ORX_ERR_INVALID = -1   # include/orx.h
AT = (1, 5, 50)
# bf16 bit patterns: +-0, +-inf, NaNs with payloads, subnormals, +-max finite
SPECIALS = np.array([0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC1, 0xFFA5, 0x7F81, 0x0001, 0x807F, 0x7F7F, 0xFF7F],
                    np.uint16)


@pytest.fixture(scope="module")
def eng():
    return N.engine()


def dev(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dtype)


def bf16_tab(rng, rows, D, specials=0, offset=0, lo=-1.0, hi=1.0):
    """A bf16 [rows, D] CUDA table of uniform values, with `specials` rows holding SPECIALS; offset > 0: a view whose
    base sits `offset` bf16 elements into its allocation."""
    bits = torch.from_numpy(rng.uniform(lo, hi, (rows, D)).astype(np.float32)).to(torch.bfloat16).view(torch.int16)
    bits = bits.numpy().view(np.uint16).copy()
    for r in rng.choice(rows, min(specials, rows), replace=False):
        bits[r] = rng.choice(SPECIALS, D)
    flat = np.concatenate([np.zeros(offset, np.uint16), bits.reshape(-1)])
    t = torch.from_numpy(flat.view(np.int16)).cuda().view(torch.bfloat16)
    return t[offset:].view(rows, D)


def same_bits(got, want, what):
    g = [got] if isinstance(got, torch.Tensor) else list(got)
    w = [want] if isinstance(want, torch.Tensor) else list(want)
    for j, (a, b) in enumerate(zip(g, w)):
        a, b = a.contiguous(), b.contiguous()
        assert a.shape == b.shape and a.dtype == b.dtype, (what, j)
        if a.dtype == torch.float32:
            a, b = a.view(torch.int32), b.view(torch.int32)
        assert torch.equal(a, b), (what, j, int((a != b).sum()))


def csr(rng, U, I, lo, hi, stray=False):
    """One sorted, unique row of [lo, hi] items per user id (entries outside [0, I) added when stray)."""
    rows = []
    for _ in range(U):
        n = int(rng.integers(lo, hi + 1))
        r = set(rng.choice(I, min(n, I), replace=False).tolist())
        if stray and rng.random() < 0.3:
            r |= {-3, I, I + 7}
        rows.append(sorted(r))
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    items = np.array([x for r in rows for x in r], np.int32)
    return dev(off, torch.int64), dev(items, torch.int32), max(len(r) for r in rows)


def uids(rng, U, Bu):
    u = rng.integers(0, U, Bu).astype(np.int64)
    for j, bad in enumerate((-1, U, INT32_MAX)):
        if Bu > 3 * j + 2:
            u[3 * j + 2] = bad
    return dev(u.astype(np.int32), torch.int32)


class Case:
    """Tables, lists and ids of one shape; up() gives the fp32 upcast the oracle scores."""

    def __init__(self, kind, D, I, Bu, seed, offset=0, specials=True):
        rng = np.random.default_rng(seed)
        self.kind, self.D, self.I, self.Bu = kind, D, I, Bu
        self.U = 67
        self.user = bf16_tab(rng, self.U, D, 2 if specials else 0, offset)
        self.item = bf16_tab(rng, I, D, 3 if specials and I > 8 else 0, offset)
        self.bias = dev(rng.uniform(-1, 1, I).astype(np.float32), torch.float32)
        self.scale = dev(rng.uniform(0.5, 1.5, D).astype(np.float32), torch.float32)
        self.uid = uids(rng, self.U, Bu)
        self.pos = csr(rng, self.U, I, 1, 6, stray=True)
        self.excl = csr(rng, self.U, I, 0, 9)
        self.neg = csr(rng, self.U, I, 0, 40, stray=True)

    def up(self):
        return self.user.float(), self.item.float()

    def variants(self):
        """(bias, scale) pairs: none, bias only, and (DOT) the scale with the bias."""
        out = [(None, None), (self.bias, None)]
        if self.kind == DOT:
            out.append((self.bias, self.scale))
        return out


def run_all(eng, c, user, item, bias, scale):
    return eng.score_all(c.kind, user, c.uid, item, bias, scale=scale)


def run_rank(eng, c, user, item, bias, scale, excl=True, max_pos=None):
    po, pi, mp = c.pos
    eo, ei, _ = c.excl if excl else (None, None, 0)
    return eng.score_rank(c.kind, user, c.uid, item, bias, po, pi, eo, ei, mp if max_pos is None else max_pos, at=AT,
                          scale=scale)


def run_listed(eng, c, user, item, bias, scale, excl=True, max_pos=None):
    po, pi, mp = c.pos
    no, ni, _ = c.neg
    eo, ei, _ = c.excl if excl else (None, None, 0)
    return eng.score_rank_listed(c.kind, user, c.uid, item, bias, po, pi, no, ni, eo, ei,
                                 mp if max_pos is None else max_pos, at=AT, scale=scale)


def run_topk(eng, c, user, item, bias, scale, k, excl=True):
    eo, ei, _ = c.excl if excl else (None, None, 0)
    return eng.score_topk(c.kind, user, c.uid, item, bias, eo, ei, k, scale=scale)


def check_case(eng, c, what):
    uf, itf = c.up()
    for bias, scale in c.variants():
        tag = f"{what} bias={bias is not None} scale={scale is not None}"
        same_bits(run_all(eng, c, c.user, c.item, bias, scale), run_all(eng, c, uf, itf, bias, scale), "all " + tag)
        for excl in (True, False):
            t = f"{tag} excl={excl}"
            # max_pos one short of the longest positive row: that row's outputs are NaN
            for mp in (None, max(c.pos[2] - 1, 0)):
                same_bits(run_rank(eng, c, c.user, c.item, bias, scale, excl, mp),
                          run_rank(eng, c, uf, itf, bias, scale, excl, mp), f"rank {t} max_pos={mp}")
                same_bits(run_listed(eng, c, c.user, c.item, bias, scale, excl, mp),
                          run_listed(eng, c, uf, itf, bias, scale, excl, mp), f"listed {t} max_pos={mp}")
            for k in sorted({1, 10, min(c.I + 3, 1024), 1024}):
                same_bits(run_topk(eng, c, c.user, c.item, bias, scale, k, excl),
                          run_topk(eng, c, uf, itf, bias, scale, k, excl), f"topk {t} k={k}")


SHAPES = [(1, 1), (127, 127), (128, 128), (129, 129), (5000, 300)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", [1, 7, 8, 12, 50, 64, 128, 256])
@pytest.mark.parametrize("I,Bu", SHAPES, ids=[f"I{i}-Bu{b}" for i, b in SHAPES])
def test_entry_points_equal_fp32_on_upcast(eng, kind, D, I, Bu):
    """All four bf16 entries equal their fp32 forms on the upcast tables, bit for bit: every D chunk tail (D % 4 == 0
    takes the 8-byte tile loader, the others the scalar one), user and item tile tail, bias / scale, excl_off NULL,
    bad uids, rows past max_pos, k up to ORX_MAX_TOPK, bf16 specials."""
    check_case(eng, Case(kind, D, I, Bu, seed=hash((kind, D, I, Bu)) % 2 ** 32), f"kind={kind} D={D} I={I} Bu={Bu}")


@pytest.mark.parametrize("kind", KINDS)
def test_rank_global_variant(eng, kind):
    """A max_pos large enough that the thresholds leave shared memory (RANK_GLOBAL): still bit-equal, same variant."""
    c = Case(kind, 64, 3000, 200, seed=5)
    uf, itf = c.up()
    mp = 40000
    eng.debug_dispatch_log()
    same_bits(run_rank(eng, c, c.user, c.item, c.bias, None, max_pos=mp),
              run_rank(eng, c, uf, itf, c.bias, None, max_pos=mp), "rank global")
    log = eng.debug_dispatch_log()
    assert [r.op for r in log] == [N.ORX_OP_SCORE_RANK_BF16, N.ORX_OP_SCORE_RANK]
    assert log[0].variant == N.ORX_VARIANT_RANK_GLOBAL and log[0][1:] == log[1][1:]
    same_bits(run_listed(eng, c, c.user, c.item, c.bias, None, max_pos=mp),
              run_listed(eng, c, uf, itf, c.bias, None, max_pos=mp), "listed global")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", [50, 64])
@pytest.mark.parametrize("offset", [1, 2, 3, 4])
def test_unaligned_tables(eng, kind, D, offset):
    """Tables starting `offset` bf16 elements into their allocation (2-, 4-, 2- and 8-byte aligned) give the bits of
    the aligned upcast: at D = 64 the tile loop takes 4 columns per 8-byte load on the 8-byte-aligned tables and the
    scalar loader on the others."""
    c = Case(kind, D, 700, 140, seed=11 + offset, offset=offset)
    assert c.user.data_ptr() % 8 == c.item.data_ptr() % 8 == 2 * offset % 8
    check_case(eng, c, f"D={D} offset={offset}")


@pytest.mark.parametrize("kind", KINDS)
def test_dispatch_records(eng, kind):
    """orx_score_rank_bf16 / orx_score_topk_bf16 log ops 14 / 15 with the fields of the fp32 call on the same shapes;
    orx_score_all_bf16 and orx_score_rank_listed_bf16 log nothing."""
    for I, Bu in ((129, 1), (5000, 300), (100000, 1024)):
        c = Case(kind, 128, I, Bu, seed=I, specials=False)
        uf, itf = c.up()
        eng.debug_dispatch_log()
        run_rank(eng, c, c.user, c.item, c.bias, None)
        run_rank(eng, c, uf, itf, c.bias, None)
        run_topk(eng, c, c.user, c.item, c.bias, None, 100)
        run_topk(eng, c, uf, itf, c.bias, None, 100)
        run_all(eng, c, c.user, c.item, c.bias, None)
        run_listed(eng, c, c.user, c.item, c.bias, None)
        log = eng.debug_dispatch_log()
        assert [r.op for r in log] == [N.ORX_OP_SCORE_RANK_BF16, N.ORX_OP_SCORE_RANK, N.ORX_OP_SCORE_TOPK_BF16,
                                       N.ORX_OP_SCORE_TOPK], log
        assert log[0][1:] == log[1][1:] and log[2][1:] == log[3][1:], log
        assert log[0].ta == kind and log[0].m == Bu and log[0].n == I and log[0].k == 128 and log[2].tb == 100


# ---- refusals ---------------------------------------------------------------------------------------------------
def test_refusals_match_fp32(eng):
    """Each bf16 entry returns ORX_ERR_INVALID exactly where its fp32 form does; the Engine refuses mixed dtypes."""
    lib, h = _lib.lib(), eng.h
    c = Case(DOT, 8, 50, 4, seed=3, specials=False)
    uf, itf = c.up()
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    po, pi, _ = c.pos
    no, ni, _ = c.neg
    out = torch.empty(4, 1024, device="cuda")
    top = torch.empty(4, 1024, dtype=torch.int32, device="cuda")
    at = (C.c_int32 * 9)(*range(1, 10))
    base = dict(kind=DOT, U=c.U, Bu=4, I=50, dim=8, max_pos=6, n_at=3, k=10, null_user=False, neg=True)
    # (change, the calls it applies to): each is a refusal of those calls' fp32 forms; the others would run
    bad = [(dict(kind=7), "all rank listed topk"), (dict(U=0), "all rank listed topk"),
           (dict(I=0), "all rank listed topk"), (dict(I=2 ** 31), "rank listed topk"),
           (dict(dim=0), "all rank listed topk"), (dict(Bu=-1), "all rank listed topk"),
           (dict(max_pos=-1), "rank listed"), (dict(n_at=9), "rank listed"), (dict(k=0), "topk"),
           (dict(k=1025), "topk"), (dict(null_user=True), "all rank listed topk"), (dict(neg=False), "listed"),
           (dict(Bu=2 ** 20, max_pos=2 ** 11), "rank listed")]

    def calls(a, user, item):
        u = None if a["null_user"] else p(user)
        args = (a["kind"], u, a["U"], p(c.uid), a["Bu"], None, p(item), p(c.bias), a["I"], a["dim"])
        return {
            "all": lambda f: getattr(lib, "orx_score_all" + f)(h, *args, p(out), None),
            "rank": lambda f: getattr(lib, "orx_score_rank" + f)(h, *args, p(po), p(pi), None, None, a["max_pos"], at,
                                                                 a["n_at"], p(out), p(out), p(out), None),
            "listed": lambda f: getattr(lib, "orx_score_rank_listed" + f)(
                h, *args, p(po), p(pi), p(no) if a["neg"] else None, p(ni), None, None, a["max_pos"], at, a["n_at"],
                p(out), p(out), p(out), None),
            "topk": lambda f: getattr(lib, "orx_score_topk" + f)(h, *args, None, None, a["k"], p(top), p(out), None),
        }
    for change, names in bad:
        a = {**base, **change}
        f32, b16 = calls(a, uf, itf), calls(a, c.user, c.item)
        for name in names.split():
            rc32, rc16 = f32[name](""), b16[name]("_bf16")
            assert rc32 == ORX_ERR_INVALID and rc16 == ORX_ERR_INVALID, (name, change, rc32, rc16)
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="bfloat16"):
        eng.score_all(DOT, c.user, c.uid, itf, None)
    with pytest.raises(ValueError, match="float32"):
        eng.score_topk(DOT, uf, c.uid, c.item, None, None, None, 5)
    with pytest.raises(ValueError, match="torch.float16"):
        eng.score_rank(DOT, c.user.half(), c.uid, c.item.half(), None, po, pi, None, None, 6)


# ---- far rows ---------------------------------------------------------------------------------------------------
def need(nbytes, what):
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes + 2 * GB:
        pytest.skip(f"{what} needs {(nbytes + 2 * GB) / GB:.1f} GB free on the device, {free / GB:.1f} GB are")


@pytest.mark.parametrize("kind", KINDS)
def test_far_rows(eng, kind):
    """A bf16 item table past 2^32 elements (D = 128, far_rows(D) rows, zero except planted rows): rows beyond element
    2^32 score near the users and their 32-bit aliases far from them, so orx_score_topk_bf16 must return the far rows,
    and orx_score_rank_bf16 / orx_score_rank_listed_bf16 must count them, with the scores of orx_score_all on the
    fp32 upcast of the gathered rows."""
    D = 128
    I = F.far_rows(D)
    need(I * D * 2 + I * 4, "a far bf16 item table and its bias")
    rng = np.random.default_rng(kind + 40)
    item = torch.zeros(I, D, dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(I, device="cuda")
    try:
        first_far = -(-F.MID_END // D)
        far = np.sort(rng.choice(np.arange(first_far, I), 40, replace=False))
        alias = np.array(sorted({a for r in far for a in F.alias_rows(r, D)}))
        planted = np.concatenate([far, alias])
        item[dev(far, torch.int64)] = bf16_tab(rng, len(far), D, lo=0.25, hi=0.5)
        item[dev(alias, torch.int64)] = bf16_tab(rng, len(alias), D, lo=-0.5, hi=-0.25)
        Bu = 8
        user = bf16_tab(rng, Bu, D, lo=0.25, hi=0.5)
        uid = dev(np.arange(Bu), torch.int32)
        # expected scores: the planted rows and one zero row (the bulk), gathered and upcast
        zero = next(i for i in range(I) if i not in set(planted.tolist()))
        rows = np.concatenate([planted, [zero]])
        sc = eng.score_all(kind, user.float(), uid, item[dev(rows, torch.int64)].float(), bias[dev(rows, torch.int64)])
        sc = sc.cpu().numpy()
        s_of = [dict(zip(rows.tolist(), sc[b].tolist())) for b in range(Bu)]
        bulk = sc[:, -1]

        # top-K: the far rows outrank the bulk, which ties at the lowest ids, the aliases rank last
        K = 64
        items, scores = eng.score_topk(kind, user, uid, item, bias, None, None, K)
        items, scores = items.cpu().numpy(), scores.cpu().numpy()
        pl = set(planted.tolist())
        for b in range(Bu):
            cand = [(s_of[b][i], i) for i in planted.tolist()]
            cand += [(float(bulk[b]), i) for i in range(K + len(pl)) if i not in pl]
            want = sorted(cand, key=lambda x: (-x[0], x[1]))[:K]
            assert items[b].tolist() == [i for _, i in want], b
            assert np.array_equal(scores[b].view(np.int32), np.array([s for s, _ in want], np.float32).view(np.int32))
            assert set(far.tolist()) <= set(items[b].tolist())

        # catalogue ranks: positives = far rows, aliases and bulk rows; exclusions = some of each
        pos, excl = [], []
        for b in range(Bu):
            p = set(rng.choice(far, 4, replace=False).tolist()) | set(rng.choice(alias, 2, replace=False).tolist())
            p |= {int(x) for x in rng.integers(0, 1000, 2)} - pl
            e = set(rng.choice(planted, 6, replace=False).tolist()) - p
            pos.append(sorted(p))
            excl.append(sorted(e))
        po, pi = (dev(x, t) for x, t in zip(_csr_np(pos), (torch.int64, torch.int32)))
        eo, ei = (dev(x, t) for x, t in zip(_csr_np(excl), (torch.int64, torch.int32)))
        mp = max(len(p) for p in pos)
        auc, ndcg, rec = (t.cpu().numpy() for t in eng.score_rank(kind, user, uid, item, bias, po, pi, eo, ei, mp,
                                                                  at=AT))
        for b in range(Bu):
            P, E = set(pos[b]), set(excl[b])
            s = lambda i: s_of[b].get(i, float(bulk[b]))
            n_bulk = I - len(pl)
            bulk_p = sum(1 for x in P | E if x not in pl)
            bulk_e = sum(1 for x in E if x not in pl)
            n_eval = I - len(P | E)
            total, hits, dcg = 0, np.zeros(len(AT)), np.zeros(len(AT))
            for p in pos[b]:
                v = s(p)
                total += (n_bulk - bulk_p) * (bulk[b] <= v) + sum(1 for i in pl - P - E if s(i) <= v)
                if p in E:
                    continue
                r = (n_bulk - bulk_e) * (bulk[b] > v) + sum(1 for i in pl - E if s(i) > v)
                for j, at in enumerate(AT):
                    if r < at:
                        hits[j] += 1
                        dcg[j] += 1.0 / np.log2(r + 2.0)
            assert auc[b] == np.float32(total) / np.float32(len(P) * n_eval), b
            np.testing.assert_array_equal(rec[b], hits.astype(np.float32) / np.float32(len(P)))
            np.testing.assert_allclose(ndcg[b], dcg, rtol=1e-5)

        # listed: each user ranked against far rows and aliases only; the compact fp32 call on the gathered rows
        # (ids renumbered in order) gives the same bits, since listed metrics do not depend on I
        neg = [sorted(set(rng.choice(planted, 20, replace=False).tolist())) for _ in range(Bu)]
        lst = sorted(pl | {x for p in pos for x in p})
        ren = {g: j for j, g in enumerate(lst)}
        no, ni = (dev(x, t) for x, t in zip(_csr_np(neg), (torch.int64, torch.int32)))
        got = eng.score_rank_listed(kind, user, uid, item, bias, po, pi, no, ni, eo, ei, mp, at=AT)
        sub = dev(np.array(lst), torch.int64)
        rmap = lambda rows: [[ren[x] for x in r] for r in rows]
        po2, pi2 = (dev(x, t) for x, t in zip(_csr_np(rmap(pos)), (torch.int64, torch.int32)))
        no2, ni2 = (dev(x, t) for x, t in zip(_csr_np(rmap(neg)), (torch.int64, torch.int32)))
        eo2, ei2 = (dev(x, t) for x, t in zip(_csr_np(rmap(excl)), (torch.int64, torch.int32)))
        want = eng.score_rank_listed(kind, user.float(), uid, item[sub].float(), bias[sub], po2, pi2, no2, ni2, eo2,
                                     ei2, mp, at=AT)
        same_bits(got, want, "listed far")
    finally:
        del item, bias
        gc.collect()
        torch.cuda.empty_cache()


def _csr_np(rows):
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return off, np.array([x for r in rows for x in r], np.int32)


# ---- models -----------------------------------------------------------------------------------------------------
MODEL_U, MODEL_I, MODEL_D = 3000, 400_000, 128


def _datasets(rng):
    from openrec_b200.tf2.data.dataset import Dataset

    def mk(n, labelled=False):
        dt = [("user_id", np.int32), ("item_id", np.int32)] + ([("label", np.float32)] if labelled else [])
        raw = np.empty(n, dtype=dt)
        raw["user_id"], raw["item_id"] = rng.integers(0, MODEL_U, n), rng.integers(0, MODEL_I, n)
        if labelled:
            raw["label"] = (rng.random(n) < 0.3).astype(np.float32)
            return Dataset(raw_data=raw, total_users=MODEL_U, total_items=MODEL_I, implicit_negative=False)
        return Dataset(raw_data=raw, total_users=MODEL_U, total_items=MODEL_I)
    return mk(60000), mk(4000), mk(20000, labelled=True)


def _peak_rise(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("cls_name", ["BPR", "UCML", "GMF", "WRMF"])
def test_models_score_bf16_in_place(eng, cls_name):
    """bf16 BPR / UCML / GMF / WRMF through inference, RankingEvaluator, CandidateEvaluator and Retriever: the bits of
    the fp32 model holding the upcast tables, the bf16 dispatch ops, and a peak-memory rise per call below the bf16
    item table's bytes (an fp32 copy of both tables would be twice that)."""
    from openrec_b200.tf2 import recommenders as Rm
    from openrec_b200.tf2.metrics.evaluator import CandidateEvaluator, RankingEvaluator
    rng = np.random.default_rng(17)
    cls = getattr(Rm, cls_name)
    model = cls(MODEL_D, MODEL_D, MODEL_U, MODEL_I, embedding_dtype="bfloat16")
    ref = cls(MODEL_D, MODEL_D, MODEL_U, MODEL_I)
    for v in model.variables:      # spread values and a non-zero bias, so scores differ and ties are rare
        if v.t.dtype == torch.bfloat16:
            v.assign(rng.uniform(-0.5, 0.5, tuple(v.t.shape)).astype(np.float32))
        elif v.t.dim() == 2 and v.t.shape[1] == 1:
            v.assign(rng.uniform(-0.1, 0.1, tuple(v.t.shape)).astype(np.float32))
    for a, b in zip(ref.variables, model.variables):
        a.assign(b.numpy())
    item_bytes = model.item_latent_factor.embeddings.t.numel() * 2
    train, val, labelled = _datasets(rng)
    users = np.arange(0, MODEL_U, 97, dtype=np.int32)

    a, rise = _peak_rise(lambda: model.inference(users).numpy())
    assert a.nbytes < item_bytes / 2 and rise < item_bytes, ("inference", rise)
    same_bits(torch.from_numpy(a), torch.from_numpy(ref.inference(users).numpy()), "inference")

    eng.debug_dispatch_log()
    x, rise = _peak_rise(lambda: [t.numpy() for t in Rm.Retriever(k=50, batch_size=64).recommend(model, users)])
    assert rise < item_bytes, ("recommend", rise)
    assert {r.op for r in eng.debug_dispatch_log()} == {N.ORX_OP_SCORE_TOPK_BF16}
    y = [t.numpy() for t in Rm.Retriever(k=50, batch_size=64).recommend(ref, users)]
    for s, t in zip(x, y):
        same_bits(torch.from_numpy(s), torch.from_numpy(t), "recommend")

    ev = RankingEvaluator(val, excl_datasets=[train], at=[10, 50], batch_size=256)
    eng.debug_dispatch_log()
    ra, rise = _peak_rise(lambda: {k: v.numpy() for k, v in ev.evaluate(model).items()})
    assert rise < item_bytes, ("RankingEvaluator", rise)
    assert {r.op for r in eng.debug_dispatch_log()} == {N.ORX_OP_SCORE_RANK_BF16}
    rb = {k: v.numpy() for k, v in ev.evaluate(ref).items()}
    for k in ra:
        same_bits(torch.from_numpy(ra[k]), torch.from_numpy(rb[k]), f"RankingEvaluator {k}")

    cev = CandidateEvaluator(labelled, excl_datasets=[train], at=[5, 20], batch_size=256)
    eng.debug_dispatch_log()
    ca, rise = _peak_rise(lambda: {k: v.numpy() for k, v in cev.evaluate(model).items()})
    assert rise < item_bytes, ("CandidateEvaluator", rise)
    assert eng.debug_dispatch_log() == []        # orx_score_rank_listed_bf16 writes no record
    cb = {k: v.numpy() for k, v in cev.evaluate(ref).items()}
    for k in ca:
        same_bits(torch.from_numpy(ca[k]), torch.from_numpy(cb[k]), f"CandidateEvaluator {k}")
