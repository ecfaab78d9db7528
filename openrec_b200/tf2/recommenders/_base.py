"""Shared machinery of the fused-step recommenders (BPR, UCML, GMF, WRMF).

The step protocol (tf2_examples/bpr_citeulike.py:33-39) is executed as ONE liborx call when
``optimizer.apply_gradients`` receives the full symbolic gradient set of a step node; see
openrec_b200/tfshim/core.py."""
from __future__ import annotations

import numpy as np
import torch

from ... import native as N
from ..._lib import OrxTable
from ...tfshim.core import LazyScalar, StepNode, Tensor, convert
from ...tfshim.keras import Model


def _check_dtype(embedding_dtype):
    """The embedding_dtype keyword of the fused-step recommenders: "float32" or "bfloat16"."""
    if embedding_dtype not in ("float32", "bfloat16"):
        raise ValueError(f"embedding_dtype must be 'float32' or 'bfloat16', got {embedding_dtype!r}")
    return embedding_dtype


def ids_of(x):
    """int32 device ids from whatever the caller feeds (Keras Embedding casts to int32)."""
    return N.ids32(convert(x).t)


def ids_any(x):
    """-> (int32 ids, on_host).  Host data (numpy / CPU tensors) stays on the host in pinned memory so the
    fused step can take it through the C-ABI's host-buffer entry point (one call: H2D + kernels + D2H)."""
    from ...tfshim import core
    if type(x) is torch.Tensor and x.dtype == torch.int32 and x.dim() == 1 and not x.is_cuda and x.is_pinned() \
            and core.device().type == "cuda":
        return x, True                       # fast path: already a pinned int32 host batch
    if isinstance(x, (core.Tensor, core.Variable)):
        t = x.t
    elif torch.is_tensor(x):
        t = x
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x)))
    if t.is_cuda or core.device().type != "cuda":
        return N.ids32(t), False
    t = t.reshape(-1)
    if t.dtype != torch.int32:
        t = t.to(torch.int32)
    t = t.contiguous()
    return (t if t.is_pinned() else t.pin_memory()), True


class _OutRing:
    """Pinned float[4] result buffers + events, recycled.  A slot also keeps the step's pinned HOST id tensors alive:
    orx_pairwise_step_host only enqueues the upload (on liborx's side stream), so the buffers must not go back to
    torch's host allocator before the step's event has completed -- a later ``pin_memory()`` could otherwise be handed
    the same block and overwrite ids that the GPU has not read yet.  A slot is reused only after its event is done."""

    def __init__(self, n=32):
        self.bufs = [torch.zeros(4, dtype=torch.float32).pin_memory() for _ in range(n)]
        self.events = [torch.cuda.Event() for _ in range(n)]
        self.owner = [None] * n
        self.keep = [None] * n
        self.used = [False] * n
        self.i = 0

    def take(self, node, keep=None):
        k = self.i
        self.i = (k + 1) % len(self.bufs)
        old = self.owner[k]
        if old is not None and old.out_host is self.bufs[k]:
            old.host_values()                    # waits for that step's event and copies the floats out
        elif self.used[k]:
            self.events[k].synchronize()         # the step that used this slot (and its id upload) has finished
        self.owner[k], self.keep[k], self.used[k] = node, keep, True
        return self.bufs[k], self.events[k]


class FusedRecommender(Model):
    """Base: subclasses define the kernels behind _orx_forward / _orx_run_step / _orx_run_grad."""

    def _tables(self, optimizer=None):
        """orx_table_t structs of (user, item, bias) for ``optimizer`` (None: no slots).  Cached per optimizer OBJECT:
        the entry holds a weak reference to it (an id() can be reused by a new optimizer) and strong references to
        the slot tensors whose raw pointers sit in the structs."""
        cache = self.__dict__.setdefault("_orx_cache_tables", {})
        key = id(optimizer)
        ent = cache.get(key)
        if ent is not None and (optimizer is None or ent[1]() is optimizer):
            return ent[0]
        vs = (self.user_latent_factor.embeddings, self.item_latent_factor.embeddings, self.item_bias.embeddings)
        if optimizer is None:
            ent = (tuple((N.table_bf16 if v.t.dtype == torch.bfloat16 else N.table)(v.t) for v in vs), None, None)
        else:
            import weakref
            ent = (tuple(optimizer.table(v) for v in vs), weakref.ref(optimizer), [optimizer.slots(v) for v in vs])
            for k in [k for k, e in cache.items() if e[1] is not None and e[1]() is None]:
                del cache[k]                     # entries of optimizers that are gone
        cache[key] = ent
        return ent[0]

    def _orx_step_variables(self):
        return self.trainable_variables

    def _new_node(self, *ids, host_ids=None):
        if self.user_latent_factor.output_dim != self.item_latent_factor.output_dim:
            raise ValueError("user and item embedding dims must match (the reference multiplies them elementwise)")
        node = StepNode(self, 2)
        node.ids = ids if ids else None
        node.host_ids = host_ids
        return node, LazyScalar(node, {0: 1.0}), LazyScalar(node, {1: 1.0})

    def _device_ids(self, node):
        """ids on the device (staged from pinned host memory on first use)."""
        if node.ids is None:
            dev = self.user_latent_factor.embeddings.t.device
            node.ids = tuple(t.to(dev, non_blocking=True) for t in node.host_ids)
        return node.ids

    def _out_ring(self):
        ring = getattr(self, "_orx_ring", None)
        if ring is None:
            ring = self._orx_ring = _OutRing()
        return ring

    def _orx_apply(self, node, grads_and_vars, optimizer):
        if node.stepped:
            raise RuntimeError("this model call's gradients were already applied")
        want = {id(v) for v in self._orx_step_variables()}
        got = {id(v) for _, v in grads_and_vars}
        coefs = [g.coef for g, _ in grads_and_vars]
        if got != want or any(c != coefs[0] for c in coefs):
            raise NotImplementedError(
                "apply_gradients: the fused step needs the gradients of ALL of the model's trainable variables "
                "w.r.t. one objective (as tape.gradient(loss, model.trainable_variables) returns them)")
        c_loss, c_l2 = float(coefs[0].get(0, 0.0)), float(coefs[0].get(1, 0.0))
        if node.host_ids is not None and hasattr(self, "_orx_run_step_host"):
            node.out = None
            self._orx_run_step_host(node, optimizer, c_loss, c_l2)
        else:
            if node.out is None:
                node.out = torch.zeros(4, dtype=torch.float32, device=self._device_ids(node)[0].device)
            self._orx_run_step(node, optimizer, c_loss, c_l2)
        node.stepped = True
        node.ids = node.host_ids = None   # the batch is consumed; keep unread loss handles light

    def _orx_materialize_grad(self, node, var, coef):
        """IndexedSlices (indices, values) of d(objective)/d(var), not deduplicated (TF form)."""
        if node.stepped:
            raise RuntimeError("gradients requested after the step was applied (tables already updated)")
        return self._orx_run_grad(node, var, float(coef.get(0, 0.0)), float(coef.get(1, 0.0)))


def w_table(var, s0=None, s1=None):
    """GMF's Dense(1) kernel [D,1] viewed as a 1-row table (rows=1, dim=D)."""
    return OrxTable(var.data_ptr(), s0.data_ptr() if s0 is not None else None,
                    s1.data_ptr() if s1 is not None else None, 1, var.numel())
