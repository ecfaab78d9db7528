"""The hot-row cases of tests/hot_rows.py are exact and their bar is sound, on CPU.

  - every case tests/test_gpu_hot_rows.py runs keeps each element's sum of |contribution| below 2^24 units of its grid,
    with exact SGD / momentum / Nesterov updates, and the cluster ids wrap their probe chains at every index size used;
  - the float32 step, its lookups summed in several random orders, equals the float64 step bit for bit under SGD,
    momentum and Nesterov, and stays within 1/4 of the exact bar under Adagrad, row-wise Adagrad and both Adams;
  - the exact bar rejects a hot row that loses one contribution, one counted twice, one sent to a neighbouring staged
    row and an item bias that loses one side's contributions;
  - step_bar's own bar accepts the lost contribution at the Zipf(1.05) shape bench.py times: the gap the exact cases
    close."""
import numpy as np
import pytest

import hot_rows as H
import momentum_bar as MB
import step_bar as S
from oracle import openrec_oracle as O

HEADROOM, MARGIN, ORDERS = 0.25, 4.0, 5


def _all_specs():
    return H.pair_specs() + H.point_specs()


def test_batch_sizes_exact():
    tail = H.tail_batch()
    assert tail % 8 and tail < 64 and H.batch_exact(tail)
    for B in (1, 2, 4096, 65536):
        assert H.batch_exact(B)
    assert not all(H.batch_exact(B) for B in range(1, 64)), "some batch sizes do not qualify"
    for spec in _all_specs():
        if spec[0] in ("bpr", "gmf"):
            assert H.batch_exact(spec[3]), spec


@pytest.mark.parametrize("kind", H.KINDS)
def test_every_gpu_case_is_exact(kind):
    n = 0
    for spec in _all_specs():
        if spec[0] != kind:
            continue
        for k in ((0, 1) if spec[5] == "prefetch" else (0,)):
            H.assert_exact(H.build(spec, k))
            n += 1
    assert n


@pytest.mark.parametrize("pattern", H.PATTERNS)
@pytest.mark.parametrize("kind", H.KINDS)
def test_patterns_exact(kind, pattern):
    """Each builder under each pattern at 4096 and 65 536 lookups (clusters at 4096: their tables grow with the index)."""
    for B in ((4096,) if pattern == "cluster" else (4096, 65536)):
        H.assert_exact(H.make_case(kind, MB.OPT_NESTEROV, 32, B, pattern, H.seed_of("pattern", kind, pattern, B)))


def test_cluster_ids_wrap():
    """The cluster ids of every batch size the GPU file uses wrap their linear-probe chains, on the user side (index
    for B lookups) and the item side (2 B); the same ids at a larger index (a handle grown for a bigger batch) do not
    all home into its last slots."""
    sizes = {s[3] for s in _all_specs() if s[4] == "cluster"}
    assert sizes
    for B in sorted(sizes):
        for pair in (True, False):
            rng, hot = np.random.default_rng(B), np.random.default_rng(B + 1)
            U, I, ids = (H.pair_ids if pair else H.point_ids)("cluster", B, rng, hot)
            sides = ((ids[0], B), (np.concatenate(ids[1:]), 2 * B)) if pair else ((ids[0], B), (ids[1], 2 * B))
            for x, lookups in sides:
                if len(x) > H.CLUSTER_SPAN:
                    assert H.wrapped(x, lookups), (B, pair, lookups)
                cap, lg = H.hash_shape(lookups)
                assert (H.home_slot(x, lg) >= cap - H.CLUSTER_SPAN).mean() > 0.5 or len(x) < 4
    x = H.cluster_ids(2 * 16384, 4096, np.random.default_rng(0))
    assert H.wrapped(x, 4096) and not H.wrapped(x, 8 * 4096)


def test_hash_shape_rule():
    assert H.hash_shape(1) == (1024, 10) and H.hash_shape(256) == (1024, 10) and H.hash_shape(257) == (2048, 11)
    assert H.hash_shape(4096) == (16384, 14) and H.hash_shape(2 * 65536) == (2 ** 19, 19)


def _emulation_specs():
    out = []
    for kind in H.KINDS:
        for opt in H.OPTS:
            for pattern in H.PATTERNS:
                out.append((kind, opt, 12 if opt % 2 else 64, 4096, pattern))
    return out


@pytest.mark.parametrize("kind,opt,D,B,pattern", _emulation_specs())
def test_float32_emulation(kind, opt, D, B, pattern):
    c = H.make_case(kind, opt, D, B, pattern, H.seed_of("emul", kind, opt, D, B, pattern))
    bar = H.ExactBar(c)
    ref = H.oracle_step(c)
    if opt in H.EXACT_OPTS:
        bar.exact(ref, "float64 oracle")      # the bar's reference is the oracle's step
    rng = np.random.default_rng(1)
    for k in range(ORDERS):
        got = H.f32_step(c, rng if k else None)
        if opt in H.EXACT_OPTS:
            bar.exact(got, f"float32 order {k}")
        else:
            q, where = bar.worst(got)
            assert q <= HEADROOM, (k, where, q)


@pytest.mark.parametrize("kind,opt,mutant", [(k, o, m) for k in H.KINDS for o in H.OPTS for m in H.MUTANTS
                                              if m != "bias_one_side" or k in S.PAIR_KINDS])
def test_exact_bar_rejects_mutants(kind, opt, mutant):
    """(A pointwise item bias is referenced from one side only: bias_one_side is a pairwise mutant.)"""
    c = H.make_case(kind, opt, 32, 4096, "zipf", H.seed_of("mutant", kind, opt))
    q, where = H.ExactBar(c).worst(H.mutant_step(c, mutant))
    assert q >= MARGIN, (where, q)


def _zipf_shape_case(opt):
    """step_bar's random tables (BPR scale 0.05) at U = I = 100 000, D = 32 with a batch of 65 536 Zipf(1.05) triplets,
    c_loss = B, c_l2 = 0."""
    rng = np.random.default_rng(11)
    U = I = 100_000
    B, D = 65536, 32
    tabs = [rng.uniform(-0.05, 0.05, s) for s in ((U, D), (I, D), (I, 1))]
    ur, ir = rng.permutation(U), rng.permutation(I)
    ids = (H.zipf_draw(U, B, rng, ur), H.zipf_draw(I, B, rng, ir), H.zipf_draw(I, B, rng, ir))
    return S.Case("bpr", opt, tabs, ids, c_loss=float(B), c_l2=0.0)


@pytest.mark.parametrize("opt", (O.OPT_SGD, O.OPT_ADAGRAD))
def test_step_bar_misses_a_lost_hot_contribution(opt, capsys):
    """The gap: at bench.py's Zipf shape step_bar's bar accepts a step whose hottest user row lost one of its ~7 000
    contributions (the hottest item row, with twice the lookups, hides it further)."""
    c = _zipf_shape_case(opt)
    st = c.state()
    _, rows = S.lookups(c, st)
    name, r = H.hottest(c, rows, ("user",))
    n = int((rows[name][0] == r).sum())
    assert n > 5000, n
    ratio, where = S.Bar(c).worst(H.mutant_step(c, "lose_hot", ("user",)))
    with capsys.disabled():
        print(f"\nstep_bar, opt {opt}: one of {n} contributions to the hottest {name} row lost, err/tol {ratio:.3f}")
    assert ratio < 1, ratio
