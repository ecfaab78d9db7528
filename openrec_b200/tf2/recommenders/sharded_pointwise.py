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
from ...tfshim.keras import Model
from ..modules import MLP, PointwiseMSELoss
from ._base import ids_of
from .sharded import ShardedBPR, _Shard


class ShardedWRMF(Model):
    _kind = N.ORX_POINT_WRMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, a=1.0, b=1.0, seed=0):
        super().__init__()
        if not dist.is_initialized():
            raise RuntimeError(f"{type(self).__name__} needs torch.distributed (one process per GPU; world size 1 is "
                               "allowed)")
        if dim_user_embed != dim_item_embed:
            raise ValueError("user and item embedding dims must match (the reference multiplies them elementwise)")
        self._rank, self._world = dist.get_rank(), dist.get_world_size()
        self._U, self._I, self._D = int(total_users), int(total_items), int(dim_user_embed)
        r, R = self._rank, self._world
        row_offsets([R * ((self._U + R - 1) // R), self._I])    # the exchange's row space must fit int32: refuse now
        eng = self._eng = N.engine()
        ru, ri = (self._U - r + R - 1) // R, (self._I - r + R - 1) // R
        mk = lambda rows, cols, k, name: ShardedBPR._new_var(eng, rows, cols, seed * 1000003 + r * 17 + k, name)
        self.user_latent_factor = _Shard(mk(max(ru, 1), self._D, 0, "user_latent_factor"), self._U, self._D)
        self.item_latent_factor = _Shard(mk(max(ri, 1), self._D, 1, "item_latent_factor"), self._I, self._D)
        self.item_bias = _Shard(mk(max(ri, 1), 1, 2, "item_bias"), self._I, 1)
        self._init_head(a, b)
        self._xchg = DistExchange()

    def _init_head(self, a, b):
        self.pointwise_mse_loss = PointwiseMSELoss(a=a, b=b)

    def _point_params(self):
        l = self.pointwise_mse_loss
        return float(l._a), float(l._b), bool(l._sigmoid)

    def _w(self):
        return None

    @property
    def variables(self):
        vs = [self.user_latent_factor.embeddings, self.item_latent_factor.embeddings, self.item_bias.embeddings]
        w = self._w()
        return vs + ([w] if w is not None else [])

    trainable_variables = variables

    def _orx_step_variables(self):
        return self.variables

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

    def _orx_forward(self, node):
        raise NotImplementedError("a sharded model's loss exists only as part of the training step "
                                  "(read it after optimizer.apply_gradients)")

    def _orx_materialize_grad(self, node, var, coef):
        raise NotImplementedError("explicit IndexedSlices are not available for row-sharded tables")

    def _orx_apply(self, node, grads_and_vars, optimizer):
        if node.stepped:
            raise RuntimeError("this model call's gradients were already applied")
        want = {id(v) for v in self.variables}
        coefs = [g.coef for g, _ in grads_and_vars]
        if {id(v) for _, v in grads_and_vars} != want or any(c != coefs[0] for c in coefs):
            raise NotImplementedError("apply_gradients: the sharded step needs the gradients of ALL of the model's "
                                      "variables w.r.t. one objective")
        opt_args = (optimizer._kind, optimizer.learning_rate, optimizer.epsilon, optimizer.beta_1, optimizer.beta_2,
                    optimizer.iterations)
        node.out = pointwise_step_sharded([self._part(optimizer)], self._xchg, [node.inputs], opt_args,
                                          c_loss=float(coefs[0].get(0, 0.0)), c_l2=float(coefs[0].get(1, 0.0)))[0]
        node.stepped = True
        node.inputs = None

    def _sharded_score_operands(self):
        """(score kind, user shard, item shard, item bias shard as a flat [rows] view, native.RowShard, process group,
        scale: GMF's w as a flat [dim] view, else None) of the catalogue evaluation and retrieval over the shards
        (RankingEvaluator.evaluate, Retriever.recommend: one collective call on every rank)."""
        g = N.rowshard(self._world, self._rank, self._U, self._I)
        w = self._w()
        return (N.ORX_SCORE_DOT, self.user_latent_factor.embeddings.t, self.item_latent_factor.embeddings.t,
                self.item_bias.embeddings.t.reshape(-1), g, None, None if w is None else w.t.reshape(-1))

    def inference(self, user_id):
        raise NotImplementedError("full-catalogue scoring needs the whole item table on one device; a sharded model's "
                                  "top-k items come from Retriever.recommend")


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
