"""Core of the minimal ``tensorflow`` surface that the openrec.tf2 examples touch.

Design (SURVEY section 7, "deferred-execution trick"): the reference's step protocol is three
calls -- ``model(...)`` under a ``GradientTape``, ``tape.gradient(...)``, ``optimizer.apply_gradients``
(tf2_examples/bpr_citeulike.py:33-39).  Here ``model(...)`` only records a *step node* (ids + model)
and returns lazy scalars; ``tape.gradient`` returns symbolic sparse gradients pointing at the node;
``apply_gradients``, on seeing the complete set for a node, issues ONE fused liborx step
(gather + score + loss + gradient + dedup + optimizer) and the lazy scalars then read their values from
the step's output.  Reading a lazy scalar before ``apply_gradients`` runs the forward-only kernel.

Tensors wrap torch CUDA tensors (device memory + streams = plumbing); all hot-path arithmetic is liborx.
"""
from __future__ import annotations

import numpy as np
import torch

# ---- dtypes ------------------------------------------------------------------------------
float32, float64, int32, int64, bool_ = torch.float32, torch.float64, torch.int32, torch.int64, torch.bool
uint8 = torch.uint8

_NP2T = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64, np.dtype("int32"): torch.int32,
         np.dtype("int64"): torch.int64, np.dtype("bool"): torch.bool, np.dtype("uint8"): torch.uint8}


def device():
    if not torch.cuda.is_available():
        raise RuntimeError("openrec_b200: no CUDA device -- the tensorflow shim has no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


class Tensor:
    """Eager tensor: a torch CUDA tensor with the few TF methods the examples use."""

    __slots__ = ("t",)
    __array_priority__ = 100

    def __init__(self, t):
        self.t = t

    # -- TF surface
    def numpy(self):
        return self.t.detach().cpu().numpy()

    @property
    def shape(self):
        return tuple(self.t.shape)

    @property
    def dtype(self):
        return self.t.dtype

    def __array__(self, dtype=None, copy=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None else a

    def __float__(self):
        return float(self.t.item())

    def __int__(self):
        return int(self.t.item())

    def __len__(self):
        return self.t.shape[0]

    def __getitem__(self, k):
        return Tensor(self.t[unwrap(k)])

    def __repr__(self):
        return f"<orx.Tensor shape={self.shape} dtype={self.dtype}>"

    # -- glue arithmetic (NOT the hot path)
    def _bin(self, o, f):
        return Tensor(f(self.t, unwrap(o)))

    def __add__(self, o): return self._bin(o, torch.add)
    def __radd__(self, o): return self._bin(o, torch.add)
    def __sub__(self, o): return self._bin(o, torch.sub)
    def __rsub__(self, o): return Tensor(unwrap(o) - self.t)
    def __mul__(self, o): return self._bin(o, torch.mul)
    def __rmul__(self, o): return self._bin(o, torch.mul)
    def __truediv__(self, o): return self._bin(o, torch.div)
    def __rtruediv__(self, o): return Tensor(unwrap(o) / self.t)
    def __neg__(self): return Tensor(-self.t)


def unwrap(x):
    if isinstance(x, Tensor):
        return x.t
    if isinstance(x, Variable):
        return x.t
    if isinstance(x, LazyScalar):
        return x.value().t
    return x


def convert(value, dtype=None, *, pin=True):
    """tf.constant / tf.convert_to_tensor: host data -> device Tensor."""
    if isinstance(value, (Tensor, Variable)):
        t = value.t
        return Tensor(t.to(dtype) if dtype is not None and t.dtype != dtype else t)
    if isinstance(value, LazyScalar):
        return value.value()
    if torch.is_tensor(value):
        t = value
    else:
        a = np.asarray(value)
        if a.dtype == np.float64 and dtype is None:
            a = a.astype(np.float32)  # TF's default float
        if a.dtype not in _NP2T:
            a = a.astype(np.int64 if a.dtype.kind in "iu" else np.float32)
        t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    dev = device()
    if t.device != dev:
        if pin and t.numel() > 0 and dev.type == "cuda" and not t.is_cuda:
            t = t.pin_memory()
        t = t.to(dev, non_blocking=True)
    return Tensor(t)


class Variable:
    """tf.Variable: a named, trainable device tensor."""
    row_table = False   # an embedding table (rows looked up by id): a row-wise optimizer keeps one slot entry per row

    def __init__(self, initial_value, trainable=True, name=None, dtype=None):
        t = convert(initial_value, dtype).t
        self.t = t.clone() if not isinstance(initial_value, (list, tuple, np.ndarray, float, int)) else t
        self.trainable = trainable
        self.name = name or "Variable"

    def numpy(self):
        t = self.t.detach()
        if t.dtype == torch.bfloat16:   # a bf16 table reads as its exact float32 upcast
            t = t.float()
        return t.cpu().numpy()

    @property
    def shape(self):
        return tuple(self.t.shape)

    @property
    def dtype(self):
        return self.t.dtype

    def value(self):
        return Tensor(self.t)

    def assign(self, v):
        if self.t.dtype == torch.bfloat16:   # float32 first, then round to nearest even
            self.t.copy_(torch.as_tensor(unwrap(v), dtype=torch.float32, device=self.t.device).to(torch.bfloat16))
            return self
        self.t.copy_(torch.as_tensor(unwrap(v), dtype=self.t.dtype, device=self.t.device))
        return self

    def assign_add(self, v):
        self.t.add_(torch.as_tensor(unwrap(v), dtype=self.t.dtype, device=self.t.device))
        return self

    def assign_sub(self, v):
        self.t.sub_(torch.as_tensor(unwrap(v), dtype=self.t.dtype, device=self.t.device))
        return self

    def scatter_nd_update(self, indices, updates):
        idx = unwrap(indices).reshape(-1).long()
        self.t[idx] = unwrap(updates)
        return self

    def __array__(self, dtype=None, copy=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None else a

    def __truediv__(self, o): return Tensor(self.t / unwrap(o))
    def __mul__(self, o): return Tensor(self.t * unwrap(o))
    def __add__(self, o): return Tensor(self.t + unwrap(o))
    def __sub__(self, o): return Tensor(self.t - unwrap(o))

    def __repr__(self):
        return f"<orx.Variable {self.name} shape={self.shape}>"


# ---- the lazy step protocol --------------------------------------------------------------

_tape_stack = []


class StepNode:
    """One ``model(...)`` call: everything needed to run either the forward-only kernel or the
    fused training step.  ``outputs`` names the lazy scalars the model returns (e.g. loss, l2_loss)."""

    def __init__(self, model, n_outputs):
        self.model = model
        self.n_outputs = n_outputs
        self.out = None        # device float tensor [4] once a kernel has produced the values
        self.stepped = False   # the fused training step has run (tables already updated)
        self.tape = _tape_stack[-1] if _tape_stack else None
        self.out_host = None   # pinned host float[4] + event when the step went through host buffers
        self.event = None
        self._vals = None      # resolved python floats

    def host_values(self):
        """Python floats of the outputs if the step wrote them to pinned host memory (waits for the
        step's event), else None."""
        if self._vals is None and self.out_host is not None:
            self.event.synchronize()
            self._vals = self.out_host.tolist()
            self.out_host = self.event = None
        return self._vals

    def ensure_forward(self):
        if self.out is None:
            hv = self.host_values()
            if hv is not None:
                self.out = torch.tensor(hv, dtype=torch.float32, device=device())
            else:
                self.out = torch.zeros(4, dtype=torch.float32, device=device())
                self.model._orx_forward(self)   # forward-only kernel fills out[0..n_outputs)
        return self.out


class LazyScalar:
    """A linear combination sum_k coef[k]*node.out[k] + const of one step node's scalar outputs."""

    __slots__ = ("node", "coef", "const")

    def __init__(self, node, coef, const=0.0):
        self.node, self.coef, self.const = node, coef, const

    def value(self):
        out = self.node.ensure_forward()
        t = None
        for k, c in self.coef.items():
            term = out[k] * c if c != 1.0 else out[k]
            t = term if t is None else t + term
        if t is None:
            t = torch.zeros((), device=out.device)
        if self.const:
            t = t + self.const
        return Tensor(t)

    def numpy(self):
        hv = self.node.host_values()
        if hv is not None:   # loss already sits in pinned host memory: no device op, no extra sync
            return np.float32(sum(c * hv[k] for k, c in self.coef.items()) + self.const)
        return self.value().numpy()

    def __float__(self):
        return float(self.numpy())

    def __array__(self, dtype=None, copy=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None else a

    @property
    def shape(self):
        return ()

    @property
    def dtype(self):
        return float32

    def _lin(self, o, sign=1.0):
        if isinstance(o, LazyScalar):
            if o.node is not self.node:
                return NotImplemented
            coef = dict(self.coef)
            for k, c in o.coef.items():
                coef[k] = coef.get(k, 0.0) + sign * c
            return LazyScalar(self.node, coef, self.const + sign * o.const)
        if isinstance(o, (int, float)):
            return LazyScalar(self.node, dict(self.coef), self.const + sign * float(o))
        return NotImplemented

    def __add__(self, o):
        r = self._lin(o)
        return self.value() + o if r is NotImplemented else r

    __radd__ = __add__

    def __sub__(self, o):
        r = self._lin(o, -1.0)
        return self.value() - o if r is NotImplemented else r

    def __mul__(self, o):
        if isinstance(o, (int, float)):
            return LazyScalar(self.node, {k: c * float(o) for k, c in self.coef.items()}, self.const * float(o))
        return self.value() * o

    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, (int, float)):
            return self * (1.0 / float(o))
        return self.value() / o

    def __neg__(self):
        return self * -1.0

    def __repr__(self):
        return f"<orx.LazyScalar coef={self.coef}>"


class SparseGrad:
    """Symbolic IndexedSlices: d(target)/d(var) of a step node, target = sum_k coef[k]*out[k]."""

    __slots__ = ("node", "var", "coef")

    def __init__(self, node, var, coef):
        self.node, self.var, self.coef = node, var, coef

    def _materialize(self):
        return self.node.model._orx_materialize_grad(self.node, self.var, self.coef)

    @property
    def indices(self):
        return self._materialize()[0]

    @property
    def values(self):
        return self._materialize()[1]

    @property
    def dense_shape(self):
        return self.var.shape


def _combine_targets(target):
    """tape.gradient target: a LazyScalar or a (nested) list/tuple of them => gradient of the SUM
    (TF semantics; bpr_citeulike.py:36-37 passes the tuple (loss, l2_loss), SURVEY Q3)."""
    if isinstance(target, LazyScalar):
        return target
    if isinstance(target, (list, tuple)):
        acc = None
        for t in target:
            c = _combine_targets(t)
            acc = c if acc is None else acc + c
            if not isinstance(acc, LazyScalar):
                raise NotImplementedError("tape.gradient: targets must come from one model call")
        return acc
    raise NotImplementedError(
        "tape.gradient: only scalars produced by an openrec.tf2 recommender call are differentiable in this shim")


class GradientTape:
    """tf.GradientTape for the openrec.tf2 step protocol (see module docstring)."""

    def __init__(self, persistent=False, watch_accessed_variables=True):
        self.persistent = persistent

    def __enter__(self):
        _tape_stack.append(self)
        return self

    def __exit__(self, *exc):
        _tape_stack.pop()
        return False

    def watch(self, tensor):
        return None

    def gradient(self, target, sources, output_gradients=None, unconnected_gradients="none"):
        if output_gradients is not None:
            raise NotImplementedError("tape.gradient(output_gradients=...) is not supported")
        tgt = _combine_targets(target)
        node = tgt.node
        single = not isinstance(sources, (list, tuple))
        srcs = [sources] if single else list(sources)
        owned = {id(v) for v in node.model._orx_step_variables()}
        grads = [SparseGrad(node, v, dict(tgt.coef)) if id(v) in owned else None for v in srcs]
        return grads[0] if single else grads


def function(func=None, **kwargs):
    """tf.function: there is no tracing compiler here -- CUDA streams run the kernels -- so this is
    the identity decorator (supports both @tf.function and @tf.function(...))."""
    if func is None:
        return lambda f: f
    return func
