"""CPU side of row-wise Adagrad: the float64 reference against a hand-worked row, the C-ABI constant, native.table's
accumulator check, RowwiseAdagrad's slot shape per variable kind and the checkpoint's strict slot shapes."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import rowwise_bar as RB
from openrec_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_hand_worked_row():
    """Row 1 of a [3, 2] table is looked up twice, gradients (1, 2) and (3, 0): G = (4, 2), mean G^2 = 10;
    acc 0.1 -> 10.1, var -= 0.5 * G / (sqrt(10.1) + 0.1).  Rows 0 and 2 are untouched."""
    var = np.array([[1.0, 1.0], [2.0, -2.0], [3.0, 3.0]])
    acc = np.full(3, 0.1)
    RB.adagrad_rowwise_sparse(var, acc, np.array([1, 1]), np.array([[1.0, 2.0], [3.0, 0.0]]), lr=0.5, eps=0.1)
    d = np.sqrt(10.1) + 0.1
    np.testing.assert_allclose(acc, [0.1, 10.1, 0.1], rtol=0, atol=1e-15)
    np.testing.assert_allclose(var, [[1, 1], [2 - 2.0 / d, -2 - 1.0 / d], [3, 3]], rtol=0, atol=1e-15)


def test_reference_dim1_is_adagrad():
    from oracle import openrec_oracle as O
    rng = np.random.default_rng(0)
    var, acc = rng.uniform(-1, 1, (20, 1)), rng.uniform(0.1, 1, (20, 1))
    ids, vals = rng.integers(0, 20, 30), rng.standard_normal((30, 1))
    v1, a1, v2, a2 = var.copy(), acc.copy(), var.copy(), acc.copy()
    RB.adagrad_rowwise_sparse(v1, a1, ids, vals, 0.05)
    O.adagrad_sparse(v2, a2, ids, vals, 0.05)
    np.testing.assert_allclose(v1, v2, rtol=1e-15)
    np.testing.assert_allclose(a1, a2, rtol=1e-15)


def test_ctypes_constant_matches_header():
    hdr = open(os.path.join(ROOT, "include", "orx.h")).read()
    assert int(re.search(r"ORX_OPT_ROWWISE_ADAGRAD = (\d+)", hdr).group(1)) == L.ORX_OPT_ROWWISE_ADAGRAD == 5
    assert RB.OPT_ROWWISE_ADAGRAD == L.ORX_OPT_ROWWISE_ADAGRAD
    from openrec_b200 import native as N
    assert N.ORX_OPT_ROWWISE_ADAGRAD == 5 and "ORX_OPT_ROWWISE_ADAGRAD" in N.__all__


def test_table_checks_rowwise_accumulator(monkeypatch):
    """native.table(kind=ROWWISE) takes a [rows] or [rows, 1] accumulator and refuses any other shape; without the kind
    the check is what it was."""
    from openrec_b200 import native as N
    monkeypatch.setattr(N, "_f32", lambda t, name: t)     # CPU tensors: the device check is not what this tests
    var = torch.zeros(10, 8)
    for s0 in (torch.zeros(10), torch.zeros(10, 1)):
        assert N.table(var, s0, kind=N.ORX_OPT_ROWWISE_ADAGRAD).rows == 10
    for s0 in (torch.zeros(10, 8), torch.zeros(9), torch.zeros(1, 10)):
        with pytest.raises(ValueError):
            N.table(var, s0, kind=N.ORX_OPT_ROWWISE_ADAGRAD)
    N.table(var, torch.zeros(10, 8))
    N.table(var, torch.zeros(10, 8), kind=N.ORX_OPT_ADAGRAD)


def test_slot_shape_follows_the_variable():
    """RowwiseAdagrad: a row table ([rows, D], [rows, 1]) gets a [rows] accumulator at 0.1; any other variable an
    element-wise one; Adagrad stays element-wise everywhere."""
    from openrec_b200.tfshim.core import Variable
    from openrec_b200.tfshim.keras.optimizers import Adagrad, RowwiseAdagrad

    def var(shape, row):
        v = Variable.__new__(Variable)
        v.t, v.trainable, v.name = torch.zeros(shape), True, "v"
        if row:
            v.row_table = True
        return v

    o, a = RowwiseAdagrad(), Adagrad()
    assert (o.learning_rate, o.initial_accumulator_value, o.epsilon) == (0.001, 0.1, 1e-7)
    for shape, row, want in (((50, 16), True, (50,)), ((50, 1), True, (50,)), ((16, 1), False, (16, 1)),
                             ((8, 4), False, (8, 4)), ((4,), False, (4,))):
        v = var(shape, row)
        s0, s1 = o.slots(v)
        assert tuple(s0.shape) == want and s1 is None and torch.all(s0 == 0.1)
        assert tuple(a.slots(v)[0].shape) == shape


SCRIPT = r"""
import sys
sys.path[:0] = [{compat!r}, {root!r}, {tests!r}]
import numpy as np, torch
import fake_engine
fake_engine.install()
import tensorflow as tf
from openrec.tf2.recommenders import BPR
from openrec_b200.tf2 import checkpoint
from openrec_b200.tfshim.keras.optimizers import RowwiseAdagrad
U, I, D = 40, 60, 8

def saved(opt_cls, path):
    m, o = BPR(D, D, U, I), opt_cls(learning_rate=0.05)
    for v in m.variables:
        for s in o.slots(v):
            if s is not None:
                s.uniform_(0.1, 0.3)
    o.iterations = 3
    checkpoint.save(path, m, o)
    return m, o

m1, o1 = saved(RowwiseAdagrad, {path!r} + "_rw")
for v in m1.variables:
    assert tuple(o1.slots(v)[0].shape) == (v.shape[0],)
m2, o2 = BPR(D, D, U, I), RowwiseAdagrad(learning_rate=0.05)
checkpoint.load({path!r} + "_rw", m2, o2)
assert o2.iterations == 3
for a, b in zip(m1.variables, m2.variables):
    assert np.array_equal(a.numpy(), b.numpy()) and torch.equal(o1.slots(a)[0], o2.slots(b)[0])
saved(tf.keras.optimizers.Adagrad, {path!r} + "_ada")
for src, opt_cls in (("_ada", RowwiseAdagrad), ("_rw", tf.keras.optimizers.Adagrad)):
    m3, o3 = BPR(D, D, U, I), opt_cls(learning_rate=0.05)
    before = [v.numpy().copy() for v in m3.variables]
    try:
        checkpoint.load({path!r} + src, m3, o3)
        raise SystemExit("mixed Adagrad / row-wise slots loaded " + src)
    except ValueError as e:
        assert "slot0/0" in str(e), e
    assert all(np.array_equal(b, v.numpy()) for b, v in zip(before, m3.variables)), "a refused load changed the model"
print("rowwise checkpoint ok")
"""


def test_rowwise_checkpoint_roundtrip_and_refusals(tmp_path):
    """Save / load under RowwiseAdagrad restores the [rows] accumulators; loading Adagrad's slots into RowwiseAdagrad,
    or the reverse, is a ValueError naming the slot (copy_ would broadcast them) and leaves the model as it was."""
    code = SCRIPT.format(compat=os.path.join(ROOT, "compat"), root=ROOT, tests=os.path.join(ROOT, "tests"),
                         path=str(tmp_path / "ck"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "rowwise checkpoint ok" in r.stdout, r.stdout + r.stderr
