"""ShardedDLRM -- the DLRM class surface (openrec/tf2/recommenders/dlrm.py:6-100: same constructor arguments, same
``model(dense, sparse, label) -> loss``, same GradientTape / ``optimizer.apply_gradients`` step protocol) with the
embedding tables ROW-SHARDED over the GPUs of a box: one process per GPU under ``torch.distributed``.

The T tables are one concatenated row space (table k starts at row_off[k] = the sum of the vocabularies before it);
global row g lives on rank ``g % world_size``.  Each rank holds one embedding shard with its optimizer slots, and a
replica of every Dense layer.  Every rank calls the model with ITS part of the global batch (the same local batch size
on every rank); ``apply_gradients`` runs one sharded step (openrec_b200.sharded.dlrm_step_sharded) and the loss is that
of the GLOBAL batch, identical on every rank.  SGD, Adagrad, LazyAdam and Keras ``Adam()`` (each owner sweeps its own
shard, which is the whole-table sweep).  ``openrec_b200.tf2.checkpoint`` saves one rank's shard and replicas (one file
per rank).

``arch_interaction_op="cross"`` (with ``cross_layers`` / ``cross_projection_dim``) replaces the dot interaction by the
DCN-v2 cross network, exactly as in DLRM; its variables are replicas like the Dense layers'.

``bag_sizes`` / ``pooling`` make every sparse feature multi-hot, exactly as in DLRM: ``sparse_features`` is [B, sum(L)],
table k's bag being its column block, pooled by a sum or a mean over the bag's valid ids.  The bags' rows are
deduplicated over this rank's batch before they travel, and each owner applies every row once per step.  The shard
layout, and so a checkpoint, does not depend on the bags."""
from __future__ import annotations

import sys

import torch.distributed as dist

from ... import native as N
from ...sharded import DistExchange, DLRMShard, dlrm_inference_sharded, dlrm_step_sharded, row_offsets
from ...tfshim.core import LazyScalar, StepNode, Tensor
from ..mlp_ops import ACT, interaction_width
from ..modules import MLP, CrossNetwork
from .dlrm import DLRM, bag_layout, cross_projections
from .sharded import _ShardedModel


class ShardedDLRM(_ShardedModel):
    def __init__(self, m_spa, ln_emb, ln_bot, ln_top, arch_interaction_op="dot", arch_interaction_itself=False,
                 sigmoid_bot=False, sigmoid_top=True, loss_func="mse", loss_threshold=0.0,
                 interaction_mode="reference", seed=0, bag_sizes=None, pooling="sum", cross_layers=3,
                 cross_projection_dim=None):
        super().__init__()
        self._bag_sizes, self._col_off, self._pooling = bag_layout(bag_sizes, pooling, len(ln_emb))
        if arch_interaction_op not in ("dot", "cross") and self._arch_interaction_op != "cat":   # as DLRM (SURVEY Q2)
            sys.exit("ERROR: arch_interaction_op=" + self._arch_interaction_op + " is not supported")
        if loss_func not in ("mse", "bce"):
            sys.exit("ERROR: loss_func=" + loss_func + " is not supported")
        self._m_spa = int(m_spa)
        self._vocab = [int(v) for v in ln_emb]
        self._row_off = row_offsets(self._vocab)
        self._loss_threshold, self._loss_func = loss_threshold, loss_func
        self._self_interaction, self._interaction_mode = bool(arch_interaction_itself), interaction_mode
        rows = N.shard_rows(self._row_off[-1], self._rank, self._world)
        self.embedding_shard = self._new_var(max(rows, 1), self._m_spa, seed * 1000003 + self._rank * 17,
                                             "embedding_shard")
        self._mlp_bot = MLP(units_list=ln_bot, out_activation="sigmoid" if sigmoid_bot else "relu")
        self._mlp_top = MLP(units_list=ln_top, out_activation="sigmoid" if sigmoid_top else "relu")
        self._cross = CrossNetwork(cross_layers, cross_projection_dim) if arch_interaction_op == "cross" else None
        self._xchg = DistExchange()

    def _own_variables(self):
        return [self.embedding_shard]

    def _orx_step_variables(self):
        return self.trainable_variables

    def _build(self, n_dense):
        """Create the Dense layers (keras builds them during the first call) and make every rank's replicas rank 0's."""
        if self._mlp_bot.layers[0].kernel is not None:
            return
        self._mlp_bot.build(n_dense)
        if self._cross is not None:
            self._cross.build((len(self._vocab) + 1) * self._m_spa)
            self._mlp_top.build((len(self._vocab) + 1) * self._m_spa)
        else:
            self._mlp_top.build(self._m_spa + interaction_width(len(self._vocab) + 1, self._self_interaction))
        for var in self._dense_vars():
            dist.broadcast(var.t, 0)

    def _dense_vars(self):
        """The Dense kernels and biases, then the cross network's: DLRMShard.dense_vars() as Variables."""
        out = [var for mlp in (self._mlp_bot, self._mlp_top) for l in mlp.layers for var in (l.kernel, l.bias)
               if var is not None]
        if self._cross is not None:
            out += [var for p in self._cross.projections() for pair in p for var in pair if var is not None]
        return out

    def _part(self, optimizer=None):
        def layers(mlp):
            return [(l.kernel.t, None if l.bias is None else l.bias.t, ACT[l.activation]) for l in mlp.layers]
        slots = optimizer.slots(self.embedding_shard) if optimizer is not None else (None, None)
        dense_slots = [optimizer.slots(var) if optimizer is not None else (None, None) for var in self._dense_vars()]
        clip = float(self._loss_threshold) if 0.0 < self._loss_threshold < 1.0 else 0.0
        return DLRMShard(self._eng, self._rank, self._world, self._vocab, self._m_spa, layers(self._mlp_bot),
                         layers(self._mlp_top), self.embedding_shard.t, slots, dense_slots,
                         self_interaction=self._self_interaction, mode=self._interaction_mode,
                         loss_kind=0 if self._loss_func == "mse" else 1, clip=clip, col_off=self._col_off,
                         pooling=self._pooling, cross=None if self._cross is None else cross_projections(self._cross))

    def _inputs(self, dense_features, sparse_features, label=None):
        dense, sparse, lab = DLRM._inputs(dense_features, sparse_features, label)
        if self._col_off is not None:
            if sparse.dim() != 2 or sparse.shape[1] != self._col_off[-1]:
                raise ValueError(f"sparse_features must be [B, {self._col_off[-1]}] (the sum of bag_sizes), got "
                                 f"{tuple(sparse.shape)}")
        elif sparse.dim() != 2 or sparse.shape[1] != len(self._vocab):
            raise ValueError(f"sparse features must be [B, {len(self._vocab)}] (one id per table)")
        return dense, sparse, lab

    def call(self, dense_features, sparse_features, label):
        """-> the loss of the GLOBAL batch (a lazy scalar); this rank contributes the samples it was given."""
        node = StepNode(self, 1)
        node.inputs = self._inputs(dense_features, sparse_features, label)
        self._build(node.inputs[0].shape[1])
        return LazyScalar(node, {0: 1.0})

    def inference(self, dense_features, sparse_features):
        """-> this rank's predictions [B].  A collective call: every rank calls it with its own samples (any B >= 0)."""
        dense, sparse, _ = self._inputs(dense_features, sparse_features)
        self._build(dense.shape[1])
        return Tensor(dlrm_inference_sharded([self._part()], self._xchg, [(dense, sparse)])[0])

    def _orx_apply(self, node, grads_and_vars, optimizer):
        coef, opt_args = self._step_args(node, grads_and_vars, optimizer)
        node.out = dlrm_step_sharded([self._part(optimizer)], self._xchg, [node.inputs], opt_args,
                                     c_loss=float(coef.get(0, 0.0)))[0]
        node.stepped = True
        node.inputs = None
