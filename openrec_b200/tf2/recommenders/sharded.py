"""ShardedBPR / ShardedUCML -- the BPR / UCML class surface (openrec/tf2/recommenders/bpr.py:7-19, ucml.py:7-19: same
constructor arguments, same ``model(user_id, p_item_id, n_item_id) -> (loss, l2_loss)``, same GradientTape /
``optimizer.apply_gradients`` step protocol) on ROW-SHARDED tables: one process per GPU under ``torch.distributed``,
row r of the user / item tables on rank ``r % world_size`` (openrec_b200/sharded.py, csrc/orx_shard.cu).  The reference is
single-device; this is what lets the 100M-item table of BASELINE configs[4] exist at all.

Every rank calls the model with ITS part of the global batch (any user / item ids); ``apply_gradients`` runs the one
sharded step; the (loss, l2_loss) it returns are those of the GLOBAL batch, identical on every rank.  The model's
variables are the local shards; the keras optimizer owns the slot tensors, so ``openrec_b200.tf2.checkpoint`` saves and
restores a rank's shard like any other model (one file per rank).  SGD, Adagrad and LazyAdam (row-sparse Adam; Keras'
``Adam()`` sweeps whole tables every step and is not offered sharded).

``ShardedUCML.censor_vec(u, p, n)`` -- UCML's training loop is "step, then censor_vec" -- is a collective call too:
every rank passes its part of the global batch, and each rank censors the rows it owns among every rank's ids, as the
single-device censor_vec does on the concatenated batch.  ``user_latent_factor.censor(ids)`` / ``item_latent_factor
.censor(ids)`` (LatentFactor.censor on one sharded table) are collective as well and accept a different number of ids
per rank.

The bases of every sharded Keras model live here too: ``_ShardedModel`` (process group, engine, the step protocol's
checks; ShardedDLRM) and ``_ShardedFactors`` (the user / item / item-bias shards; ShardedWRMF / ShardedGMF as well)."""
from __future__ import annotations

import torch
import torch.distributed as dist

from ... import native as N
from ...sharded import HomeRoutedPairwise, censor_vec_sharded
from ...tfshim.core import LazyScalar, StepNode, Variable
from ...tfshim.keras import Model
from ._base import ids_of


class _Shard:
    """Stand-in for the LatentFactor attribute of the reference models: ``.embeddings`` / ``.variables[0]`` is this rank's
    shard ([rows r with r % world == rank, dim]) of a table split over the default process group."""

    def __init__(self, var, total, dim):
        self.embeddings, self.input_dim, self.output_dim = var, total, dim
        self.variables = self.trainable_variables = [var]

    def censor(self, censor_id):
        """LatentFactor.censor (latent_factor.py:17-23) of the sharded table, a COLLECTIVE call: the rows of the unique
        ids of every rank's censor_id <- row / max(||row||, 0.1), in place, each on its owner.  The ranks may pass
        different numbers of ids: the counts are all-gathered first (one host read) and every rank's ids padded to the
        largest count with -1, then one all-gather of the ids.  Returns ``embeddings``, as LatentFactor.censor does."""
        world, rank = dist.get_world_size(), dist.get_rank()
        ids = ids_of(censor_id)
        t = self.embeddings.t
        counts = torch.empty(world, dtype=torch.int32, device=t.device)
        dist.all_gather_into_tensor(counts, torch.tensor([ids.numel()], dtype=torch.int32, device=t.device))
        n = int(counts.max().item())
        if n:
            padded = torch.full((n,), -1, dtype=torch.int32, device=t.device)
            padded[:ids.numel()] = ids.to(t.device)
            gathered = torch.empty(world * n, dtype=torch.int32, device=t.device)
            dist.all_gather_into_tensor(gathered, padded)
            N.engine().censor_shard(t, self.input_dim, world, rank, gathered, n, n, world)
        return self.embeddings


class _ShardedModel(Model):
    """What every row-sharded model shares: one process per GPU under ``torch.distributed`` (world size 1 allowed), this
    rank's engine, and the checks of the step protocol -- the loss exists only inside the step, which takes the
    gradients of all of the model's step variables w.r.t. one objective."""

    def __init__(self):
        super().__init__()
        if not dist.is_initialized():
            raise RuntimeError(f"{type(self).__name__} needs torch.distributed (one process per GPU; world size 1 is "
                               "allowed)")
        self._rank, self._world = dist.get_rank(), dist.get_world_size()
        self._eng = N.engine()

    def _new_var(self, rows, cols, seed, name):
        t = torch.empty(rows, cols, dtype=torch.float32, device=self._eng.device)
        self._eng.fill_uniform(t, -0.05, 0.05, seed)                 # LatentFactor's 'uniform' initializer
        v = Variable.__new__(Variable)
        v.t, v.trainable, v.name, v.row_table = t, True, name, True   # a table shard
        return v

    def _orx_forward(self, node):
        raise NotImplementedError("a sharded model's loss exists only as part of the training step "
                                  "(read it after optimizer.apply_gradients)")

    def _orx_materialize_grad(self, node, var, coef):
        raise NotImplementedError("explicit IndexedSlices are not available for row-sharded tables")

    def _step_args(self, node, grads_and_vars, optimizer):
        """-> (coef, opt_args) of one sharded step: the objective's {output: coefficient} and (kind, lr, eps, beta1,
        beta2, step) of ``optimizer``, after refusing a node already stepped or a gradient set that is not ALL of the
        step variables w.r.t. one objective."""
        if node.stepped:
            raise RuntimeError("this model call's gradients were already applied")
        want = {id(v) for v in self._orx_step_variables()}
        coefs = [g.coef for g, _ in grads_and_vars]
        if {id(v) for _, v in grads_and_vars} != want or any(c != coefs[0] for c in coefs):
            raise NotImplementedError("apply_gradients: the sharded step needs the gradients of ALL of the model's "
                                      "trainable variables w.r.t. one objective")
        return coefs[0], (optimizer._kind, optimizer.learning_rate, optimizer.epsilon, optimizer.beta_1,
                          optimizer.beta_2, optimizer.iterations)


class _ShardedFactors(_ShardedModel):
    """The user / item / item-bias layout of the sharded factor models (ShardedBPR / ShardedUCML, ShardedWRMF /
    ShardedGMF): row r of each table on rank r % world at local row r // world, a 1-row dummy on a rank without rows;
    the tables are ``variables`` in that order, seeded per rank and table."""
    _score = N.ORX_SCORE_DOT

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, seed):
        super().__init__()
        if dim_user_embed != dim_item_embed:
            raise ValueError("user and item embedding dims must match (the reference multiplies them elementwise)")
        self._U, self._I, self._D = int(total_users), int(total_items), int(dim_user_embed)
        self._check_sizes()
        r, R = self._rank, self._world

        def shard(total, cols, k, name):
            var = self._new_var(max(N.shard_rows(total, r, R), 1), cols, seed * 1000003 + r * 17 + k, name)
            return _Shard(var, total, cols)
        self.user_latent_factor = shard(self._U, self._D, 0, "user_latent_factor")
        self.item_latent_factor = shard(self._I, self._D, 1, "item_latent_factor")
        self.item_bias = shard(self._I, 1, 2, "item_bias")

    def _check_sizes(self):
        """Refuse sizes the model cannot shard (called before any table is allocated)."""

    def _w(self):
        """GMF's w (the scale of the score), else None."""
        return None

    @property
    def variables(self):
        vs = [self.user_latent_factor.embeddings, self.item_latent_factor.embeddings, self.item_bias.embeddings]
        w = self._w()
        return vs + ([w] if w is not None else [])

    trainable_variables = variables

    def _orx_step_variables(self):
        return self.variables

    def _sharded_score_operands(self):
        """(score kind, user shard, item shard, item bias shard as a flat [rows] view, native.RowShard, process group,
        scale: GMF's w as a flat [dim] view, else None) of the catalogue evaluation and retrieval over the shards
        (RankingEvaluator.evaluate, Retriever.recommend: one collective call on every rank)."""
        g = N.rowshard(self._world, self._rank, self._U, self._I)
        w = self._w()
        return (self._score, self.user_latent_factor.embeddings.t, self.item_latent_factor.embeddings.t,
                self.item_bias.embeddings.t.reshape(-1), g, None, None if w is None else w.t.reshape(-1))

    def inference(self, user_id):
        raise NotImplementedError("full-catalogue scoring needs the whole item table on one device; a sharded model's "
                                  "top-k items come from Retriever.recommend")


class ShardedBPR(_ShardedFactors):
    _kind = N.ORX_PAIR_BPR

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, seed=0):
        super().__init__(dim_user_embed, dim_item_embed, total_users, total_items, seed)
        self._impl = None
        self._impl_key = None

    def _get_margin(self):
        return 0.0

    def call(self, user_id, p_item_id, n_item_id):
        """-> (loss, l2_loss) of the GLOBAL batch as lazy scalars; this rank contributes the triplets it was given."""
        node = StepNode(self, 2)
        node.ids = tuple(ids_of(x) for x in (user_id, p_item_id, n_item_id))
        return LazyScalar(node, {0: 1.0}), LazyScalar(node, {1: 1.0})

    def _orx_apply(self, node, grads_and_vars, optimizer):
        coef, _ = self._step_args(node, grads_and_vars, optimizer)
        kind = optimizer._kind
        if kind not in (N.ORX_OPT_SGD, N.ORX_OPT_ADAGRAD, N.ORX_OPT_ADAM_LAZY, N.ORX_OPT_MOMENTUM, N.ORX_OPT_NESTEROV):
            raise NotImplementedError("sharded BPR / UCML tables: use SGD (with or without momentum), Adagrad or "
                                      "LazyAdam (Keras Adam() sweeps whole tables; the home-routed step has no "
                                      "RowwiseAdagrad)")
        B = node.ids[0].numel()
        key = (id(optimizer), kind)
        if self._impl is None or self._impl_key != key or B > self._impl.B:
            if self._impl is not None:
                self._impl.close()
            vs = self.variables
            self._impl = HomeRoutedPairwise(self._eng, self._rank, self._world, self._U, self._I, self._D, B, kind=self._kind,
                                            opt_kind=kind, tables=tuple(v.t for v in vs),
                                            slots=tuple(optimizer.slots(v) for v in vs))
            self._impl_key, self._impl_opt = key, optimizer          # strong reference: the slots' raw pointers are in use
        m = self._impl
        m.lr, m.eps, m.b1, m.b2 = optimizer.learning_rate, optimizer.epsilon, optimizer.beta_1, optimizer.beta_2
        m.margin = self._get_margin()
        m.iterations = optimizer.iterations - 1                      # HomeRoutedPairwise.step increments it
        out = m.step(*node.ids, c_loss=float(coef.get(0, 0.0)), c_l2=float(coef.get(1, 0.0)))
        node.out = m._out[m.iterations % 16]
        node.stepped = True
        node.ids = None

    def check(self):
        """Raise if the sharded step flagged an error (peer timeout, mailbox overflow)."""
        if self._impl is not None:
            self._impl.check()


class ShardedUCML(ShardedBPR):
    _kind = N.ORX_PAIR_UCML
    _score = N.ORX_SCORE_NEG_SQDIST

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, margin=0.5, seed=0):
        super().__init__(dim_user_embed, dim_item_embed, total_users, total_items, seed=seed)
        self.margin = margin

    def _get_margin(self):
        return float(self.margin)

    def censor_vec(self, user_id, p_item_id, n_item_id):
        """UCML.censor_vec (ucml.py:44-48) on the shards, a COLLECTIVE call: every rank passes its part of the global
        batch, the same number of ids on every rank, as in the step (not checked: a mismatch leaves the all-gather
        hanging).  The tables end as the single-device censor_vec leaves them on the concatenation of every rank's ids
        (openrec_b200.sharded.censor_vec_sharded: one all-gather of the ids, no host sync)."""
        ids = [ids_of(x) for x in (user_id, p_item_id, n_item_id)]
        user, item = self.user_latent_factor.embeddings, self.item_latent_factor.embeddings
        censor_vec_sharded(self._eng, user.t, item.t, self._U, self._I, self._world, self._rank, *ids)
        return user, item, item
