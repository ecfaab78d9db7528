"""ShardedGMF / ShardedWRMF -- the GMF / WRMF class surface (openrec/tf2/recommenders/gmf.py:5-34, wrmf.py:5-34: same
constructor arguments, same ``model(user_id, item_id, label) -> (loss, l2_loss)``, same GradientTape /
``optimizer.apply_gradients`` step protocol) on ROW-SHARDED tables: one process per GPU under ``torch.distributed``,
row r of the user table, the item table and the item bias on rank ``r % world_size`` (the layout of ShardedBPR, so
RankingEvaluator and Retriever serve these models where their rows live).  GMF's Dense(1) kernel ``w`` is replicated:
built on every rank, then set to rank 0's copy.

Every rank calls the model with ITS part of the global batch (the same local batch size on every rank);
``apply_gradients`` runs one sharded step (openrec_b200.sharded.pointwise_step_sharded) and the (loss, l2_loss) it
returns are those of the GLOBAL batch, identical on every rank.  SGD, Adagrad, LazyAdam and Keras ``Adam()`` (each owner
sweeps its own shards, which is the whole-table sweep).  ``openrec_b200.tf2.checkpoint`` saves one rank's shards, slots
and w replica (one file per rank)."""
from __future__ import annotations

import torch
import torch.distributed as dist

from ... import native as N
from ...sharded import DistExchange, PointwiseShard, pointwise_step_sharded, row_offsets
from ...tfshim.core import LazyScalar, StepNode, convert
from ..modules import MLP, PointwiseMSELoss
from ._base import ids_of
from .sharded import _ShardedFactors


class ShardedWRMF(_ShardedFactors):
    _kind = N.ORX_POINT_WRMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, a=1.0, b=1.0, seed=0):
        super().__init__(dim_user_embed, dim_item_embed, total_users, total_items, seed)
        self._init_head(a, b)
        self._xchg = DistExchange()

    def _check_sizes(self):
        R = self._world
        row_offsets([R * ((self._U + R - 1) // R), self._I])    # the exchange's row space must fit int32: refuse now

    def _init_head(self, a, b):
        self.pointwise_mse_loss = PointwiseMSELoss(a=a, b=b)

    def _point_params(self):
        l = self.pointwise_mse_loss
        return float(l._a), float(l._b), bool(l._sigmoid)

    def call(self, user_id, item_id, label):
        """-> (loss, l2_loss) of the GLOBAL batch as lazy scalars; this rank contributes the samples it was given."""
        node = StepNode(self, 2)
        node.inputs = (ids_of(user_id), ids_of(item_id),
                       convert(label).t.to(torch.float32).reshape(-1).contiguous())
        return LazyScalar(node, {0: 1.0}), LazyScalar(node, {1: 1.0})

    def _part(self, optimizer):
        vs = self.variables
        a, b, sig = self._point_params()
        w = self._w()
        return PointwiseShard(self._eng, self._rank, self._world, self._U, self._I, self._D, self._kind,
                              *(v.t for v in vs[:3]), [optimizer.slots(v) for v in vs[:3]],
                              w=None if w is None else w.t, w_slots=optimizer.slots(w) if w is not None else (None, None),
                              a=a, b=b, use_sigmoid=sig)

    def _orx_apply(self, node, grads_and_vars, optimizer):
        coef, opt_args = self._step_args(node, grads_and_vars, optimizer)
        node.out = pointwise_step_sharded([self._part(optimizer)], self._xchg, [node.inputs], opt_args,
                                          c_loss=float(coef.get(0, 0.0)), c_l2=float(coef.get(1, 0.0)))[0]
        node.stepped = True
        node.inputs = None


class ShardedGMF(ShardedWRMF):
    _kind = N.ORX_POINT_GMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, seed=0):
        super().__init__(dim_user_embed, dim_item_embed, total_users, total_items, seed=seed)

    def _init_head(self, a, b):
        self.mlp = MLP(units_list=[1], use_bias=False)
        self.mlp.build(self._D)                     # Dense(1) kernel [D, 1], glorot uniform (gmf.py:19)
        dist.broadcast(self.mlp.layers[0].kernel.t, 0)   # one replica: rank 0's

    def _point_params(self):
        return 1.0, 1.0, False

    def _w(self):
        return self.mlp.layers[0].kernel
