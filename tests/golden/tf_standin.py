"""A torch(CPU, float64-capable) stand-in for the handful of ``tensorflow`` symbols that
the reference's openrec/tf2/{modules,recommenders,metrics,data} touch.

TEST INFRASTRUCTURE used ONLY by tests/golden/make_golden.py to execute the reference's own
Python composition verbatim and record golden vectors.  It is not the product's tensorflow
shim (that is openrec_b200/tfshim, which dispatches to CUDA kernels) and is never imported
by the product.  Tensors are plain torch tensors; gradients come from torch autograd.
"""
from __future__ import annotations

import sys
import types

import torch

DTYPE = [torch.float64]  # default float dtype for variables / constants (mutable cell)


def _mod(name):
    m = types.ModuleType(name)
    sys.modules[name] = m
    return m


class Variable:
    def __init__(self, value):
        self.t = value.clone().requires_grad_(value.is_floating_point())

    def scatter_nd_update(self, indices, updates):
        with torch.no_grad():
            self.t[indices.reshape(-1).long()] = updates.detach()
        return self

    def assign(self, v):
        with torch.no_grad():
            self.t.copy_(torch.as_tensor(v, dtype=self.t.dtype))

    def assign_add(self, v):
        with torch.no_grad():
            self.t.add_(torch.as_tensor(v, dtype=self.t.dtype))

    def numpy(self):
        return self.t.detach().numpy()

    def __rmul__(self, o):
        return o * self.t

    def __rsub__(self, o):
        return o - self.t


def _t(x):
    return x.t if isinstance(x, Variable) else x


class Layer:
    def __init__(self, name=None, **kw):
        self.name = name

    def __call__(self, *a, **kw):
        return self.call(*a, **kw)

    def _collect(self, seen):
        out = []
        for v in self.__dict__.values():
            items = v if isinstance(v, (list, tuple)) else [v]
            for it in items:
                if isinstance(it, Variable) and id(it) not in seen:
                    seen.add(id(it))
                    out.append(it)
                elif isinstance(it, Layer) and id(it) not in seen:
                    seen.add(id(it))
                    out += it._collect(seen)
        return out

    @property
    def trainable_variables(self):
        return self._collect(set())

    variables = trainable_variables


class Embedding(Layer):
    def __init__(self, input_dim, output_dim, embeddings_initializer="uniform", name=None):
        super().__init__(name=name)
        if embeddings_initializer == "zeros":
            w = torch.zeros(input_dim, output_dim, dtype=DTYPE[0])
        else:  # keras 'uniform' = U(-0.05, 0.05)
            w = (torch.rand(input_dim, output_dim, dtype=DTYPE[0]) - 0.5) * 0.1
        self.embeddings = Variable(w)

    def call(self, ids):
        return self.embeddings.t[torch.as_tensor(ids).long()]

    def __call__(self, ids):
        return self.call(ids)


class Dense(Layer):
    def __init__(self, units, activation=None, use_bias=True):
        super().__init__()
        self.units, self.activation, self.use_bias = units, activation, use_bias
        self.kernel = None
        self.bias = None

    def call(self, x):
        if self.kernel is None:
            fan_in = x.shape[-1]
            lim = (6.0 / (fan_in + self.units)) ** 0.5  # glorot uniform
            self.kernel = Variable((torch.rand(fan_in, self.units, dtype=DTYPE[0]) * 2 - 1) * lim)
            if self.use_bias:
                self.bias = Variable(torch.zeros(self.units, dtype=DTYPE[0]))
        y = x @ self.kernel.t
        if self.use_bias:
            y = y + self.bias.t
        if self.activation == "relu":
            y = torch.relu(y)
        elif self.activation == "sigmoid":
            y = torch.sigmoid(y)
        return y


class Sequential(Layer):
    def __init__(self):
        super().__init__()
        self.layers = []

    def add(self, l):
        self.layers.append(l)

    def call(self, x):
        for l in self.layers:
            x = l(x)
        return x


class Model(Layer):
    pass


class _LowerTri:
    def __init__(self, m):
        self.m = m

    def to_dense(self):
        return torch.tril(self.m)


def _band_part(x, lo, hi):
    n = x.shape[-1]
    i = torch.arange(n).reshape(-1, 1)
    j = torch.arange(n).reshape(1, -1)
    keep = torch.ones(n, n, dtype=torch.bool)
    if lo >= 0:
        keep &= (i - j) <= lo
    if hi >= 0:
        keep &= (j - i) <= hi
    return x * keep.to(x.dtype)


def _reduce(fn):
    def f(x, axis=None, keepdims=False, name=None, dtype=None):
        x = _t(x)
        if axis is None:
            return fn(x)
        return fn(x, dim=axis, keepdim=keepdims)
    return f


def _count_nonzero(x, axis=None, dtype=None):
    r = (x != 0).sum() if axis is None else (x != 0).sum(dim=axis)
    return r.to(dtype) if dtype is not None else r


def _unique(x):
    x = torch.as_tensor(x)
    seen, out = set(), []
    for v in x.tolist():
        if v not in seen:
            seen.add(v)
            out.append(v)
    return torch.tensor(out, dtype=x.dtype), None


def _map_fn(fn, elems, parallel_iterations=None, dtype=None):
    n = len(elems[0])
    return torch.stack([torch.as_tensor(fn(tuple(e[i] for e in elems))) for i in range(n)])


def _constant(v, dtype=None):
    if dtype is None:
        t = torch.as_tensor(v)
        return t.to(DTYPE[0]) if t.is_floating_point() else t
    return torch.as_tensor(v).to(dtype)


def _boolean_mask(x, mask):
    return x[mask.bool()] if mask.dim() == x.dim() else x[mask.bool()]


class _MSE:
    def __call__(self, y_true, y_pred):
        return ((y_true.to(y_pred.dtype) - y_pred) ** 2).mean()


class _BCE:
    def __init__(self, from_logits=False):
        self.from_logits = from_logits

    def __call__(self, y_true, y_pred):
        y = y_true.to(y_pred.dtype)
        if self.from_logits:
            z = y_pred
            return (torch.clamp(z, min=0) - z * y + torch.log1p(torch.exp(-z.abs()))).mean()
        eps = 1e-7
        p = torch.clamp(y_pred, eps, 1 - eps)
        return -(y * torch.log(p + eps) + (1 - y) * torch.log(1 - p + eps)).mean()


def install():
    """Create the fake ``tensorflow`` module tree in sys.modules and return it."""
    for k in [k for k in sys.modules if k == "tensorflow" or k.startswith("tensorflow.")]:
        del sys.modules[k]
    tf = _mod("tensorflow")
    keras = _mod("tensorflow.keras")
    layers = _mod("tensorflow.keras.layers")
    losses = _mod("tensorflow.keras.losses")
    math = _mod("tensorflow.math")
    nn = _mod("tensorflow.nn")
    linalg = _mod("tensorflow.linalg")
    tf.keras, tf.math, tf.nn, tf.linalg = keras, math, nn, linalg
    keras.layers, keras.losses = layers, losses
    keras.Model, keras.Sequential = Model, Sequential
    layers.Layer, layers.Embedding, layers.Dense = Layer, Embedding, Dense
    losses.MeanSquaredError, losses.BinaryCrossentropy = _MSE, _BCE

    tf.float32, tf.int32, tf.bool = torch.float32, torch.int32, torch.bool
    tf.Variable = lambda v: Variable(torch.as_tensor(v))
    tf.constant = _constant
    tf.zeros = lambda shape, dtype=None: torch.zeros(*([int(s) for s in shape] if len(shape) else []), dtype=dtype)
    tf.reshape = lambda x, s: _t(x).reshape(*[int(v) for v in s])
    tf.cast = lambda x, dtype: (x if torch.is_tensor(x) else torch.as_tensor(x)).to(dtype)
    tf.shape = lambda x: _t(x).shape
    tf.size = lambda x: x.numel()
    tf.ones_like = torch.ones_like
    tf.concat = lambda xs, axis: torch.cat(list(xs), dim=axis)
    tf.stack = lambda xs, axis=0: torch.stack(list(xs), dim=axis)
    tf.unstack = lambda x, axis=0: list(torch.unbind(torch.as_tensor(x), dim=axis))
    tf.expand_dims = lambda x, axis: _t(x).unsqueeze(axis)
    tf.squeeze = lambda x, axis=None: x.squeeze(axis)
    tf.tile = lambda x, reps: x.repeat(*reps)
    tf.gather = lambda params, indices: _t(params)[indices.long()]
    tf.unique = _unique
    tf.norm = lambda x, axis=None, keepdims=False: torch.linalg.vector_norm(x, dim=axis, keepdim=keepdims)
    tf.boolean_mask = _boolean_mask
    tf.clip_by_value = lambda x, lo, hi: torch.clamp(x, lo, hi)
    tf.map_fn = _map_fn
    tf.maximum = lambda a, b: torch.maximum(torch.as_tensor(a, dtype=DTYPE[0]), torch.as_tensor(b, dtype=DTYPE[0]))
    tf.square = lambda x: x * x
    tf.reduce_sum = _reduce(torch.sum)
    tf.matmul = lambda a, b, transpose_b=False: _t(a) @ (_t(b).transpose(-1, -2) if transpose_b else _t(b))

    math.reduce_sum = _reduce(torch.sum)
    math.reduce_mean = _reduce(torch.mean)
    math.square = tf.square
    math.multiply = lambda a, b: a * b
    math.maximum = tf.maximum
    math.sigmoid = torch.sigmoid
    math.log_sigmoid = torch.nn.functional.logsigmoid
    math.log = lambda x: torch.log(torch.as_tensor(x, dtype=DTYPE[0]) if not torch.is_tensor(x) else x)
    math.exp = torch.exp
    math.reciprocal = torch.reciprocal
    math.logical_not = torch.logical_not
    math.logical_or = torch.logical_or
    math.count_nonzero = _count_nonzero
    nn.l2_loss = lambda x: (_t(x) ** 2).sum() / 2
    linalg.matmul = tf.matmul
    linalg.band_part = _band_part
    linalg.LinearOperatorLowerTriangular = _LowerTri
    return tf
