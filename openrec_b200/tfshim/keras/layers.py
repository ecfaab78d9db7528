"""tf.keras.layers.{Layer, Embedding, Dense} -- only what openrec.tf2 composes."""
from __future__ import annotations

import itertools

import torch

from ... import native as N
from ..core import Tensor, Variable, convert, device

_seed = itertools.count(20260923)


def next_seed():
    return next(_seed)


def set_seed(seed):
    """tf.random.set_seed: restarts the counter the on-device initialisers draw from."""
    global _seed
    _seed = itertools.count(int(seed))


_VERSION = [0]   # bumped whenever any layer attribute is (re)assigned: invalidates the cached variable lists


class Layer:
    def __init__(self, name=None, trainable=True, **kwargs):
        self.name = name or type(self).__name__.lower()
        self.trainable = trainable

    def __setattr__(self, key, value):
        if not key.startswith("_orx_cache"):
            _VERSION[0] += 1
        object.__setattr__(self, key, value)

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, *args, **kwargs):
        raise NotImplementedError

    def _own_variables(self):
        return []

    def _sublayers(self):
        subs = []
        for v in self.__dict__.values():
            for it in (v if isinstance(v, (list, tuple)) else [v]):
                if isinstance(it, Layer):
                    subs.append(it)
        return subs

    @property
    def variables(self):
        cache = self.__dict__.get("_orx_cache_vars")
        if cache is not None and cache[0] == _VERSION[0]:
            return list(cache[1])
        out, seen = [], set()
        for v in self._own_variables() + [w for s in self._sublayers() for w in s.variables]:
            if id(v) not in seen:
                seen.add(id(v))
                out.append(v)
        self._orx_cache_vars = (_VERSION[0], out)
        return list(out)

    @property
    def trainable_variables(self):
        return [v for v in self.variables if v.trainable]

    weights = variables
    trainable_weights = trainable_variables


class Embedding(Layer):
    """keras Embedding: table [input_dim, output_dim], 'uniform' = U(-0.05, 0.05) [TF-mem], 'zeros'."""

    def __init__(self, input_dim, output_dim, embeddings_initializer="uniform", name=None, **kwargs):
        super().__init__(name=name)
        self.input_dim, self.output_dim = int(input_dim), int(output_dim)
        t = torch.empty((self.input_dim, self.output_dim), dtype=torch.float32, device=device())
        if embeddings_initializer == "zeros":
            t.zero_()
        elif embeddings_initializer == "uniform":
            N.engine().fill_uniform(t, -0.05, 0.05, next_seed())
        else:
            raise NotImplementedError(f"embeddings_initializer={embeddings_initializer!r}")
        self.embeddings = Variable.__new__(Variable)
        self.embeddings.t, self.embeddings.trainable, self.embeddings.name = t, True, f"{self.name}/embeddings"
        self.embeddings.row_table = True

    def _own_variables(self):
        return [self.embeddings]

    def call(self, ids):
        ids_t = convert(ids).t
        rows = N.engine().gather(self.embeddings.t, ids_t if ids_t.dtype == torch.int64 else ids_t.to(torch.int32))
        return Tensor(rows.reshape(tuple(ids_t.shape) + (self.output_dim,)))


class Dense(Layer):
    """keras Dense: glorot-uniform kernel [in, units], zero bias; built on first call (or .build)."""

    def __init__(self, units, activation=None, use_bias=True, name=None, **kwargs):
        super().__init__(name=name)
        if activation not in (None, "relu", "sigmoid", "linear"):
            raise NotImplementedError(f"activation={activation!r}")
        self.units, self.activation, self.use_bias = int(units), activation, use_bias
        self.kernel = None
        self.bias = None

    def build(self, in_dim):
        if self.kernel is not None:
            return
        lim = (6.0 / (in_dim + self.units)) ** 0.5
        k = torch.empty((in_dim, self.units), dtype=torch.float32, device=device())
        N.engine().fill_uniform(k, -lim, lim, next_seed())
        self.kernel = Variable.__new__(Variable)
        self.kernel.t, self.kernel.trainable, self.kernel.name = k, True, f"{self.name}/kernel"
        if self.use_bias:
            self.bias = Variable.__new__(Variable)
            self.bias.t = torch.zeros(self.units, dtype=torch.float32, device=device())
            self.bias.trainable, self.bias.name = True, f"{self.name}/bias"

    def _own_variables(self):
        return [v for v in (self.kernel, self.bias) if v is not None]

    def call(self, x):
        from ...tf2 import mlp_ops
        xt = convert(x).t.to(torch.float32)
        self.build(xt.shape[-1])
        return Tensor(mlp_ops.dense_forward(xt, self.kernel.t, None if self.bias is None else self.bias.t,
                                            self.activation))
