"""CPU side of SGD with momentum and Nesterov momentum: the float64 reference against hand-written loops, the update bar
against the float32 emulation and its mutants, the C-ABI constants, the Keras SGD surface, the sharded step's refusals
and the checkpoint of the momentum slot."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import momentum_bar as MB
import step_bar as S
from openrec_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the reference ----------------------------------------------------------------------------------------------------
def _loop(var, a, ids, vals, lr, m, nesterov):
    """SparseApplyKerasMomentum, row by row over the unique ids in first-occurrence order."""
    var, a = var.copy(), a.copy()
    for r in dict.fromkeys(int(i) for i in ids):
        G = vals[ids == r].sum(0)
        a[r] = m * a[r] - lr * G
        var[r] += (m * a[r] - lr * G) if nesterov else a[r]
    return var, a


def test_reference_hand_worked_row():
    """Row 1 of a [3, 2] table is looked up twice, gradients (1, 2) and (3, 0): G = (4, 2).  lr 0.5, m 0.5, a = (1, -1):
    a -> (0.5 - 2, -0.5 - 1) = (-1.5, -1.5); MOMENTUM var += a; NESTEROV var += 0.5 a - 0.5 G = (-2.75, -1.75)."""
    for nest, step in ((False, [-1.5, -1.5]), (True, [-2.75, -1.75])):
        var = np.array([[1.0, 1.0], [2.0, -2.0], [3.0, 3.0]])
        a = np.array([[0.25, 0.25], [1.0, -1.0], [0.5, 0.5]])
        MB.momentum_sparse(var, a, np.array([1, 1]), np.array([[1.0, 2.0], [3.0, 0.0]]), 0.5, 0.5, nest)
        np.testing.assert_array_equal(a, [[0.25, 0.25], [-1.5, -1.5], [0.5, 0.5]])
        np.testing.assert_array_equal(var, [[1, 1], [2 + step[0], -2 + step[1]], [3, 3]])


@pytest.mark.parametrize("nesterov", (False, True))
def test_reference_against_loop(nesterov):
    rng = np.random.default_rng(3)
    var, a = rng.uniform(-1, 1, (40, 6)), rng.uniform(-0.1, 0.1, (40, 6))
    ids, vals = rng.integers(0, 30, 100), rng.standard_normal((100, 6))
    want = _loop(var, a, ids, vals, 0.05, 0.9, nesterov)
    MB.momentum_sparse(var, a, ids, vals, 0.05, 0.9, nesterov)
    np.testing.assert_allclose(var, want[0], rtol=0, atol=1e-14)
    np.testing.assert_allclose(a, want[1], rtol=0, atol=1e-14)
    assert np.array_equal(var[30:], want[0][30:])


@pytest.mark.parametrize("nesterov", (False, True))
def test_reference_dense_is_sparse_on_every_row(nesterov):
    rng = np.random.default_rng(4)
    var, a, g = rng.uniform(-1, 1, (7, 5)), rng.uniform(-0.1, 0.1, (7, 5)), rng.standard_normal((7, 5))
    v1, a1, v2, a2 = var.copy(), a.copy(), var.copy(), a.copy()
    MB.momentum_dense(v1, a1, g, 0.05, 0.9, nesterov)
    MB.momentum_sparse(v2, a2, np.arange(7), g, 0.05, 0.9, nesterov)
    np.testing.assert_array_equal(v1, v2)
    np.testing.assert_array_equal(a1, a2)


def test_momentum_zero_is_sgd():
    """At m = 0 both forms are SGD (the slot ends as -lr G): what Keras SGD(momentum=0) runs without a slot."""
    from oracle import openrec_oracle as O
    rng = np.random.default_rng(5)
    var, ids, vals = rng.uniform(-1, 1, (20, 4)), rng.integers(0, 20, 30), rng.standard_normal((30, 4))
    want = var.copy()
    O.sgd_sparse(want, ids, vals, 0.05)
    for nest in (False, True):
        v = var.copy()
        MB.momentum_sparse(v, np.zeros_like(v), ids, vals, 0.05, 0.0, nest)
        np.testing.assert_allclose(v, want, rtol=0, atol=1e-15)


# ---- the bar ----------------------------------------------------------------------------------------------------------
BAR_SPECS = [(arm, k, o, D, 203, "mixed", "step") for arm in S.ARMS for k in S.PAIR_KINDS for o in MB.KINDS
             for D in (32, 50)]
BAR_SPECS += [(arm, k, o, 64, 237, "mixed", "step") for arm in S.ARMS for k in ("gmf", "wrmf") for o in MB.KINDS]
BAR_SPECS += [("a", "bpr", o, 64, B, ids, "step") for o in MB.KINDS for ids, B in (("owned", 203), ("staged", 200))]


@pytest.mark.parametrize("spec", BAR_SPECS, ids=lambda s: "-".join(map(str, s)))
def test_bar_holds_float32_and_rejects_mutants(spec):
    """The float32 emulation of the kernels' arithmetic sits inside the bar; a slot one step stale, the other form and
    a slot that does not decay fall outside it (the last two only where a is nonzero before the step)."""
    c = MB.build(spec)
    bar = MB.MomBar(c)
    q = bar.worst(MB.f32_step(c))[0]
    assert q <= 0.5, (spec, bar.ratios(MB.f32_step(c)))
    ref = MB.step(c)
    for name in c.names:
        np.testing.assert_allclose(ref[name][0], bar.ref[name][0], rtol=0, atol=1e-15)
        np.testing.assert_allclose(ref[name][1], bar.ref[name][1], rtol=0, atol=1e-15)
    nontrivial = c.init != "keras"
    for mutant in MB.MUTANTS:
        if mutant == "no_decay" and not nontrivial:
            continue
        assert bar.worst(MB.step(c, mutant))[0] > 1.0, (spec, mutant)


def test_bar_exact_elements():
    """Rows the batch does not touch have tolerance 0 in value and slot; so does a touched row whose slot is 0 and whose
    every contribution is an exact zero (arm (c)'s users 0 and 1 under the Keras initialisation)."""
    c = MB.build(("c", "bpr", MB.OPT_MOMENTUM, 32, 203, "mixed", "step"))
    c.slots = {n: (np.zeros_like(c.tabs[n]), None) for n in c.names}
    bar = MB.MomBar(c)
    tv, ta, _ = bar.tol["user"]
    assert not tv[:2].any() and not ta[:2].any()
    untouched = np.setdiff1d(np.arange(c.tabs["user"].shape[0]), c.ids[0])
    assert len(untouched) and not tv[untouched].any() and not ta[untouched].any()


# ---- constants, Keras surface, refusals --------------------------------------------------------------------------------
def test_constants_match_header():
    hdr = open(os.path.join(ROOT, "include", "orx.h")).read()
    assert int(re.search(r"ORX_OPT_MOMENTUM = (\d+)", hdr).group(1)) == L.ORX_OPT_MOMENTUM == MB.OPT_MOMENTUM == 6
    assert int(re.search(r"ORX_OPT_NESTEROV = (\d+)", hdr).group(1)) == L.ORX_OPT_NESTEROV == MB.OPT_NESTEROV == 8
    from openrec_b200 import native as N
    assert {"ORX_OPT_MOMENTUM", "ORX_OPT_NESTEROV"} <= set(N.__all__)
    kinds = {getattr(N, k) for k in N.__all__ if k.startswith("ORX_OPT_")}
    assert kinds == {0, 1, 2, 3, 5, 6, 8} and not kinds & {4, 7}


def _var(shape):
    from openrec_b200.tfshim.core import Variable
    v = Variable.__new__(Variable)
    v.t, v.trainable, v.name = torch.zeros(shape), True, "v"
    return v


def test_keras_sgd_surface():
    from openrec_b200 import native as N
    from openrec_b200.tfshim.keras.optimizers import SGD
    o = SGD()
    assert (o.learning_rate, o.momentum, o.nesterov) == (0.01, 0.0, False)
    assert o.get_config() == {"name": "SGD", "learning_rate": 0.01, "momentum": 0.0, "nesterov": False}
    for m in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            SGD(momentum=m)
    for kw in (dict(), dict(momentum=0.0, nesterov=True)):      # plain SGD: no slot, whatever nesterov says
        o = SGD(learning_rate=0.1, **kw)
        assert o._kind == N.ORX_OPT_SGD and o.slots(_var((5, 3))) == (None, None)
        assert o.opt_struct().beta1 == 0.0                      # not the base class's 0.9
    for nest, kind in ((False, N.ORX_OPT_MOMENTUM), (True, N.ORX_OPT_NESTEROV)):
        o = SGD(learning_rate=0.1, momentum=0.5, nesterov=nest)
        assert o._kind == kind and o.get_config()["momentum"] == 0.5 and o.get_config()["nesterov"] is nest
        s0, s1 = o.slots(_var((5, 3)))
        assert tuple(s0.shape) == (5, 3) and not s0.any() and s1 is None
        st = o.opt_struct()
        assert (st.kind, st.beta1) == (kind, 0.5) and abs(st.lr - 0.1) < 1e-7
    assert SGD(momentum=1.0)._kind == N.ORX_OPT_MOMENTUM
    assert SGD()._kind == N.ORX_OPT_SGD and SGD._kind == N.ORX_OPT_SGD      # the class default stays plain SGD


def test_sharded_pairwise_refusals_keep_their_message():
    """HomeRoutedPairwise refuses the kinds orx_shard_step has not got before it touches the engine, with the message
    the older kinds' tests read; the momentum kinds pass that check."""
    from openrec_b200.sharded import HomeRoutedPairwise
    for k in (3, 4, 5, 7):
        with pytest.raises(ValueError, match="supports SGD, Adagrad and row-sparse Adam"):
            HomeRoutedPairwise(None, 0, 1, 10, 10, 8, 4, opt_kind=k)
    for k in (6, 8):
        with pytest.raises(AttributeError):          # past the kind check: eng=None has no device
            HomeRoutedPairwise(None, 0, 1, 10, 10, 8, 4, opt_kind=k)


SCRIPT = r"""
import sys
sys.path[:0] = [{compat!r}, {root!r}, {tests!r}]
import numpy as np, torch
import fake_engine
fake_engine.install()
import tensorflow as tf
from openrec.tf2.recommenders import BPR
from openrec_b200.tf2 import checkpoint
U, I, D = 40, 60, 8
for nest in (False, True):
    m1, o1 = BPR(D, D, U, I), tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nest)
    for v in m1.variables:
        o1.slots(v)[0].uniform_(-0.1, 0.1)
    o1.iterations = 3
    checkpoint.save({path!r}, m1, o1)
    m2, o2 = BPR(D, D, U, I), tf.keras.optimizers.SGD(learning_rate=0.05, momentum=0.9, nesterov=nest)
    checkpoint.load({path!r}, m2, o2)
    assert o2.iterations == 3
    for a, b in zip(m1.variables, m2.variables):
        assert np.array_equal(a.numpy(), b.numpy()) and torch.equal(o1.slots(a)[0], o2.slots(b)[0])
        assert o2.slots(b)[1] is None
print("momentum checkpoint ok")
"""


def test_momentum_checkpoint_roundtrip(tmp_path):
    """checkpoint.save / load carry the momentum slot as slot0, for both forms."""
    code = SCRIPT.format(compat=os.path.join(ROOT, "compat"), root=ROOT, tests=os.path.join(ROOT, "tests"),
                         path=str(tmp_path / "ck.npz"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "momentum checkpoint ok" in r.stdout, r.stdout + r.stderr
