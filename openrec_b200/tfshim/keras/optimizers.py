"""tf.keras.optimizers.{SGD, Adagrad, Adam} with Keras OptimizerV2 sparse semantics, executed by
liborx (fused into the recommender step when the whole gradient set of a step node is applied).

[TF-mem] defaults: SGD lr=0.01, momentum=0.0, nesterov=False; Adagrad lr=0.001, initial_accumulator_value=0.1, eps=1e-7;
Adam lr=0.001, beta_1=0.9, beta_2=0.999, eps=1e-7.  Keras-2.0 Adam on IndexedSlices is NOT lazy:
``Adam()`` therefore maps to liborx's ADAM_DENSE mode (whole-table sweep, exact reference semantics);
``LazyAdam`` (an addition, not in the reference) is the row-sparse variant.  ``RowwiseAdagrad`` (an addition too) keeps
one Adagrad accumulator per embedding-table row, updated with the mean of the row's squared gradient.
"""
from __future__ import annotations

import torch

from ... import native as N
from ..core import SparseGrad, Tensor, Variable, unwrap


def _table(var, s0, s1, **kind):
    """orx_table_t (float32 variable) or orx_table_bf16_t (bfloat16 table) of var with its slots; kind=: see N.table."""
    make = N.table_bf16 if var.t.dtype == torch.bfloat16 else N.table
    return make(var.t, s0, s1, **kind)


class Optimizer:
    _kind = None
    _n_slots = 0

    def __init__(self, learning_rate, name=None, **kwargs):
        if "lr" in kwargs:
            learning_rate = kwargs.pop("lr")
        if kwargs:
            raise NotImplementedError(f"optimizer options {sorted(kwargs)} are not supported")
        self.learning_rate = float(learning_rate)
        self.epsilon = 1e-7
        self.beta_1, self.beta_2 = 0.9, 0.999
        self.iterations = 0
        self.name = name or type(self).__name__
        self._slots = {}

    lr = property(lambda self: self.learning_rate)

    # slot tensors are created on first use (Keras creates them at first apply)
    def slots(self, var: Variable):
        ent = self._slots.get(id(var))
        if ent is None or ent[0]() is not var:      # id() of a dead variable can be reused: check the object itself
            import weakref
            s = tuple(self._init_slot(var, k) for k in range(self._n_slots)) + (None,) * (2 - self._n_slots)
            ent = self._slots[id(var)] = (weakref.ref(var), s)
        return ent[1]

    def slots_if_any(self, var: Variable):
        """The slot tensors of ``var`` if they exist already (checkpoint save), else ()."""
        ent = self._slots.get(id(var))
        return ent[1] if ent is not None and ent[0]() is var else ()

    # slots are float32 whatever the variable's dtype (a bf16 table keeps fp32 optimizer state)
    def _init_slot(self, var, k):
        return torch.zeros_like(var.t, dtype=torch.float32)

    def table(self, var: Variable):
        s0, s1 = self.slots(var)
        return _table(var, s0, s1)

    def opt_struct(self):
        return N.opt(self._kind, self.learning_rate, self.epsilon, self.beta_1, self.beta_2, self.iterations)

    def apply_gradients(self, grads_and_vars, name=None, **kwargs):
        pairs = [(g, v) for g, v in grads_and_vars if g is not None]
        if not pairs:
            raise ValueError("No gradients provided for any variable")
        self.iterations += 1
        by_node, dense = {}, []
        for g, v in pairs:
            if isinstance(g, SparseGrad):
                by_node.setdefault(id(g.node), (g.node, []))[1].append((g, v))
            else:
                dense.append((g, v))
        for node, gv in by_node.values():
            node.model._orx_apply(node, gv, self)
        for g, v in dense:
            gt = unwrap(g)
            if not torch.is_tensor(gt) or tuple(gt.shape) != tuple(v.t.shape):
                raise NotImplementedError("apply_gradients: dense gradient must match the variable's shape")
            s0, s1 = self.slots(v)
            N.engine().dense_apply(v.t, s0, s1, gt.to(torch.float32).contiguous(), self.opt_struct())
        return None

    def get_config(self):
        return {"name": self.name, "learning_rate": self.learning_rate}


class SGD(Optimizer):
    """Keras SGD.  With ``momentum > 0`` each touched row r keeps a velocity a (slot 0, zero-initialised):
    ``a[r] = momentum * a[r] - lr * G[r]``, then ``var[r] += a[r]``, or with ``nesterov=True``
    ``var[r] += momentum * a[r] - lr * G[r]``.  Rows a step does not touch keep their value and velocity, as Keras
    momentum on IndexedSlices does.  ``momentum == 0`` is plain SGD with no slot, whatever ``nesterov`` says."""
    _kind = N.ORX_OPT_SGD
    _n_slots = 0

    def __init__(self, learning_rate=0.01, momentum=0.0, nesterov=False, name="SGD", **kwargs):
        super().__init__(learning_rate, name, **kwargs)
        momentum = float(momentum)
        if not 0.0 <= momentum <= 1.0:
            raise ValueError("`momentum` must be between [0, 1].")
        self.momentum, self.nesterov = momentum, bool(nesterov)
        # every path that builds an orx_opt_t passes beta_1: it carries the momentum, never the base class's 0.9
        self.beta_1 = momentum
        if momentum > 0.0:
            self._kind = N.ORX_OPT_NESTEROV if self.nesterov else N.ORX_OPT_MOMENTUM
            self._n_slots = 1

    def get_config(self):
        return {**super().get_config(), "momentum": self.momentum, "nesterov": self.nesterov}


class Adagrad(Optimizer):
    _kind = N.ORX_OPT_ADAGRAD
    _n_slots = 1

    def __init__(self, learning_rate=0.001, initial_accumulator_value=0.1, epsilon=1e-7, name="Adagrad", **kwargs):
        super().__init__(learning_rate, name, **kwargs)
        self.initial_accumulator_value = float(initial_accumulator_value)
        self.epsilon = float(epsilon)

    def _init_slot(self, var, k):
        return torch.full_like(var.t, self.initial_accumulator_value, dtype=torch.float32)


class Adam(Optimizer):
    _kind = N.ORX_OPT_ADAM_DENSE
    _n_slots = 2

    def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7, amsgrad=False, name="Adam",
                 **kwargs):
        if amsgrad:
            raise NotImplementedError("amsgrad is not on the openrec.tf2 path")
        super().__init__(learning_rate, name, **kwargs)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)


class LazyAdam(Adam):
    """Row-sparse Adam (moments of untouched rows are left alone).  NOT the reference's semantics."""
    _kind = N.ORX_OPT_ADAM_LAZY


class RowwiseAdagrad(Adagrad):
    """Row-wise Adagrad: one accumulator per embedding-table row, ``acc[r] += mean_j G[r, j]^2`` and
    ``var[r] -= lr * G[r] / (sqrt(acc[r]) + eps)`` for the rows a step touches (G summed over the step's lookups of r).
    Same per-row adaptivity as Adagrad for about SGD's memory traffic; its slot is 1/dim of Adagrad's.  NOT in the
    reference.  Embedding tables (variables created with ``row_table = True``: Embedding / LatentFactor and the sharded
    models' table shards) get a ``[rows]`` accumulator; every other variable (Dense kernels and biases, GMF's w) gets
    element-wise Adagrad with an element-wise accumulator."""
    _kind = N.ORX_OPT_ROWWISE_ADAGRAD

    def __init__(self, learning_rate=0.001, initial_accumulator_value=0.1, epsilon=1e-7, name="RowwiseAdagrad",
                 **kwargs):
        super().__init__(learning_rate, initial_accumulator_value, epsilon, name, **kwargs)

    def table(self, var: Variable):
        s0, s1 = self.slots(var)
        return _table(var, s0, s1, kind=self._kind)   # checks that s0 holds one accumulator per row

    def _init_slot(self, var, k):
        if getattr(var, "row_table", False):
            return torch.full((var.t.shape[0],), self.initial_accumulator_value, dtype=torch.float32,
                              device=var.t.device)
        return super()._init_slot(var, k)
