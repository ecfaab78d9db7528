"""DLRM -- mirrors openrec/tf2/recommenders/dlrm.py:6-100 on liborx (gathers, interaction, Dense layers,
loss, sparse + dense optimizer applies); same lazy step protocol as the other recommenders.  ``bag_sizes`` adds
multi-hot sparse features (a pooled bag of ids per table) and ``arch_interaction_op="cross"`` the DCN-v2 cross network
(MLPerf DLRM-DCNv2), which the reference does not have."""
import sys

import torch

from ... import native as N
from ..._lib import ORX_BAG_MAX_TABLES
from ...tfshim.core import LazyScalar, StepNode, Tensor, convert
from ...tfshim.keras import Model
from ..mlp_ops import ACT, DLRMGraph
from ..modules import MLP, CrossNetwork, LatentFactor, SecondOrderFeatureInteraction
from ._base import _check_dtype

_M64 = (1 << 64) - 1


def _mix64(z):
    """splitmix64's finalizer (include/orx.h), a bijection of the uint64s."""
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & _M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & _M64
    return z ^ (z >> 31)


def table_rounding_seed(rounding_seed, k):
    """The stochastic-rounding seed of DLRM's bf16 table k: mix64(rounding_seed + k) (mod 2^64).  Each table's apply
    rounds as table 0 of the orx.h rule under its own seed; mix64 is a bijection, so every table of a model gets a
    distinct seed, whatever the number of tables (keying tables by t in mix64(2 * step + t) would give table 2 at step s
    the bits of table 0 at step s + 1)."""
    return _mix64((int(rounding_seed) + int(k)) & _M64)


def bag_layout(bag_sizes, pooling, n_tables):
    """The checked multi-hot layout of DLRM / ShardedDLRM: -> (bag sizes, col_off [T + 1] with table k's bag at columns
    col_off[k] .. col_off[k+1], pooling 0 for 'sum' / 1 for 'mean'); the first two are None when bag_sizes is None.
    ValueError for an unknown pooling, a bag_sizes length other than n_tables, a size < 1 or more than
    ORX_BAG_MAX_TABLES tables."""
    if pooling not in ("sum", "mean"):
        raise ValueError(f"pooling must be 'sum' or 'mean', got {pooling!r}")
    sizes = col_off = None
    if bag_sizes is not None:
        sizes = [int(L) for L in bag_sizes]
        if len(sizes) != n_tables:
            raise ValueError(f"bag_sizes has {len(sizes)} entries for {n_tables} embedding tables")
        if any(L < 1 for L in sizes):
            raise ValueError("every bag size must be >= 1")
        if len(sizes) > ORX_BAG_MAX_TABLES:
            raise ValueError(f"multi-hot DLRM takes at most {ORX_BAG_MAX_TABLES} tables")
        col_off = [0]
        for L in sizes:
            col_off.append(col_off[-1] + L)
    return sizes, col_off, 0 if pooling == "sum" else 1


def cross_projections(cross):
    """DLRMGraph's ``cross`` argument: the tensors of a built CrossNetwork's projections."""
    return [[(w.t, None if b is None else b.t) for w, b in p] for p in cross.projections()]


def _dense_groups(model, bot_g, top_g, cross_g):
    """(variables, gradients) of every Dense kernel / bias and cross projection, in the order the step applies them."""
    out = []
    for mlp, grads in ((model._mlp_bot, bot_g), (model._mlp_top, top_g)):
        for layer, (dw, db) in zip(mlp.layers, grads):
            out.append((layer.kernel, dw))
            if layer.bias is not None:
                out.append((layer.bias, db))
    cross = model._cross
    for p, grads in zip(cross.projections() if cross is not None else [], cross_g):
        for (w, b), (dw, db) in zip(p, grads):
            out.append((w, dw))
            if b is not None:
                out.append((b, db))
    return out


class DLRM(Model):
    def __init__(self, m_spa, ln_emb, ln_bot, ln_top, arch_interaction_op="dot", arch_interaction_itself=False,
                 sigmoid_bot=False, sigmoid_top=True, loss_func="mse", loss_threshold=0.0,
                 interaction_mode="reference", bag_sizes=None, pooling="sum", cross_layers=3,
                 cross_projection_dim=None, embedding_dtype="float32", rounding_seed=0):
        """Reference signature (dlrm.py:8-19) + ``interaction_mode``: 'reference' reproduces the reference's
        dot interaction bit for bit (identically zero, SURVEY Q1), 'dlrm' is the strictly-lower triangle.

        ``bag_sizes = [L_0 .. L_{T-1}]`` makes every sparse feature multi-hot: ``sparse_features`` is then [B, sum(L)],
        table k's bag for sample b being columns sum(L[:k]) .. sum(L[:k+1]) - 1 of row b, pooled by ``pooling`` ('sum'
        or 'mean' over the bag's valid ids).  An id < 0 is padding; an id >= the vocabulary adds nothing and gets no
        gradient; a bag without a valid id pools to the zero row.  None (the default): one id per table, [B, T].

        ``arch_interaction_op="cross"`` replaces the dot interaction by a DCN-v2 CrossNetwork(cross_layers,
        cross_projection_dim) over x0 = (dense_vec | Z_0 | .. | Z_{T-1}), W = (T + 1) * m_spa wide; the top MLP reads
        its [B, W] output.  ``arch_interaction_itself`` and ``interaction_mode`` apply to the dot interaction only.

        ``embedding_dtype="bfloat16"`` stores the embedding tables in bfloat16 (optimizer slots, Dense layers, cross
        projections, Z and every activation stay float32).  A lookup widens rows exactly; each apply rounds table k's
        updated elements stochastically under seed ``table_rounding_seed(rounding_seed, k)`` and the optimizer's step,
        so a run repeats bit for bit."""
        self.embedding_dtype, self.rounding_seed = _check_dtype(embedding_dtype), int(rounding_seed)
        super().__init__()
        self._bag_sizes, self._col_off, self._pooling = bag_layout(bag_sizes, pooling, len(ln_emb))
        self._m_spa = int(m_spa)
        self._loss_threshold = loss_threshold
        self._loss_func = loss_func
        self._latent_factors = [LatentFactor(num_instances=int(num), dim=m_spa, dtype=embedding_dtype) for num in ln_emb]
        self._mlp_bot = MLP(units_list=ln_bot, out_activation="sigmoid" if sigmoid_bot else "relu")
        self._mlp_top = MLP(units_list=ln_top, out_activation="sigmoid" if sigmoid_top else "relu")
        self._dot_interaction = self._cross = None
        if arch_interaction_op == "dot":
            self._dot_interaction = SecondOrderFeatureInteraction(self_interaction=arch_interaction_itself,
                                                                  mode=interaction_mode)
        elif arch_interaction_op == "cross":
            self._cross = CrossNetwork(cross_layers, cross_projection_dim)
        elif self._arch_interaction_op != "cat":   # the reference never assigns this attribute: AttributeError (Q2)
            sys.exit("ERROR: arch_interaction_op=" + self._arch_interaction_op + " is not supported")
        if loss_func not in ("mse", "bce"):
            sys.exit("ERROR: loss_func=" + loss_func + " is not supported")
        self._self_interaction = bool(arch_interaction_itself)
        self._interaction_mode = interaction_mode

    # ---- graph over the current variables
    def _graph(self, n_dense):
        T = len(self._latent_factors)
        width = T + 1
        P = width * (width + 1) // 2 if self._self_interaction else width * (width - 1) // 2
        self._mlp_bot.build(n_dense)
        cross = self._cross
        if cross is not None:
            cross.build(width * self._m_spa)
            self._mlp_top.build(width * self._m_spa)
        else:
            self._mlp_top.build(self._m_spa + P)

        def layers(mlp):
            return [(l.kernel.t, None if l.bias is None else l.bias.t, ACT[l.activation]) for l in mlp.layers]
        clip = float(self._loss_threshold) if 0.0 < self._loss_threshold < 1.0 else 0.0
        return DLRMGraph([lf.embeddings.t for lf in self._latent_factors], layers(self._mlp_bot),
                         layers(self._mlp_top), self._m_spa, self._self_interaction, self._interaction_mode,
                         0 if self._loss_func == "mse" else 1, clip, self._col_off, self._pooling,
                         cross=None if cross is None else cross_projections(cross))

    def _checked_inputs(self, dense_features, sparse_features, label=None):
        dense, sparse, lab = self._inputs(dense_features, sparse_features, label)
        if self._col_off is not None and (sparse.dim() != 2 or sparse.shape[1] != self._col_off[-1]):
            raise ValueError(f"sparse_features must be [B, {self._col_off[-1]}] (the sum of bag_sizes), got "
                             f"{tuple(sparse.shape)}")
        return dense, sparse, lab

    @staticmethod
    def _inputs(dense_features, sparse_features, label=None):
        dense = convert(dense_features).t.to(torch.float32).contiguous()
        sparse = convert(sparse_features).t.to(torch.int32).contiguous()   # Embedding casts ids to int32
        lab = None if label is None else convert(label).t.to(torch.float32).reshape(-1).contiguous()
        return dense, sparse, lab

    def call(self, dense_features, sparse_features, label):
        """-> loss (a single lazy scalar, dlrm.py:63-74)."""
        node = StepNode(self, 1)
        node.inputs = self._checked_inputs(dense_features, sparse_features, label)
        self._graph(node.inputs[0].shape[1])   # keras builds the Dense layers during the first call
        return LazyScalar(node, {0: 1.0})

    def inference(self, dense_features, sparse_features):
        """-> predictions [B] (dlrm.py:76-100)."""
        dense, sparse, _ = self._checked_inputs(dense_features, sparse_features)
        return Tensor(self._graph(dense.shape[1]).forward(dense, sparse)["pred"])

    # ---- step protocol hooks (openrec_b200/tfshim/core.py)
    def _orx_step_variables(self):
        return self.trainable_variables

    def _orx_forward(self, node):
        dense, sparse, lab = node.inputs
        node.out.copy_(self._graph(dense.shape[1]).forward(dense, sparse, lab)["out4"])

    def _fwd_bwd(self, node, scale):
        dense, sparse, lab = node.inputs
        g = self._graph(dense.shape[1])
        c = g.forward(dense, sparse, lab, want_grad=True)
        if scale != 1.0:
            c["dpred"].mul_(scale)
        return c, g.backward(c)

    def _orx_apply(self, node, grads_and_vars, optimizer):
        if node.stepped:
            raise RuntimeError("this model call's gradients were already applied")
        dense, sparse, lab = node.inputs
        self._graph(dense.shape[1])                                   # make sure Dense layers exist
        want = {id(v) for v in self.trainable_variables}
        got = {id(v) for _, v in grads_and_vars}
        coefs = [g.coef for g, _ in grads_and_vars]
        if got != want or any(c != coefs[0] for c in coefs):
            raise NotImplementedError("apply_gradients: DLRM's fused step needs the gradients of ALL trainable "
                                      "variables w.r.t. one objective")
        c, (dZ, bot_g, top_g, cross_g) = self._fwd_bwd(node, float(coefs[0].get(0, 0.0)))
        eng, o = N.engine(), optimizer.opt_struct()
        for k, lf in enumerate(self._latent_factors):                 # IndexedSlices(ids = sparse[:,k], dZ[:,k,:])
            bf16 = {"sr_seed": table_rounding_seed(self.rounding_seed, k)} if self.embedding_dtype == "bfloat16" else {}
            if self._col_off is None:
                eng.sparse_apply_strided(optimizer.table(lf.embeddings), sparse, k, dZ, o, **bf16)
            else:                                                     # ... of every valid id of table k's bags
                eng.bag_sparse_apply(optimizer.table(lf.embeddings), sparse, self._col_off[k], self._bag_sizes[k],
                                     dZ[:, k, :], self._pooling, o, **bf16)
        for var, g in _dense_groups(self, bot_g, top_g, cross_g):
            eng.dense_apply(var.t, *optimizer.slots(var), g, o)
        node.out = c["out4"]
        node.stepped = True
        node.inputs = None

    def _launches_per_step(self):
        """liborx kernel launches of one training step (bench.py's gpu_launches): per table gather + index / apply / tail,
        per Dense layer forward (1) + backward (activation, column sum, dgrad, wgrad; split-K adds a reduce) + 2 dense
        applies, 2 interaction kernels, 1 loss kernel.  Multi-hot: one gather launch for all tables, and per table id
        compaction / index / apply / tail.  Cross network, in place of the interaction: per projection forward (1) +
        backward (column sum with a bias, dgrad, wgrad) + 1 apply per variable, per layer 2 cross kernels, and 1 final
        cross kernel."""
        T = len(self._latent_factors)
        n_dense = len(self._mlp_bot.layers) + len(self._mlp_top.layers)
        n = (4 * T if self._col_off is None else 1 + 4 * T) + n_dense * (1 + 4 + 2) + 1
        cross = self._cross
        if cross is None:
            return n + 2
        per_layer = 2 + (1 + 3 + 2 if cross.projection_dim is None else (1 + 2 + 1) + (1 + 3 + 2))
        return n + cross.num_layers * per_layer + 1

    def _orx_materialize_grad(self, node, var, coef):
        if node.stepped:
            raise RuntimeError("gradients requested after the step was applied")
        _, (dZ, bot_g, top_g, cross_g) = self._fwd_bwd(node, float(coef.get(0, 0.0)))
        for k, lf in enumerate(self._latent_factors):
            if var is lf.embeddings:
                if self._col_off is None:
                    return Tensor(node.inputs[1][:, k].contiguous()), Tensor(dZ[:, k, :].contiguous())
                return self._bag_slices(node.inputs[1], k, dZ[:, k, :])
        for v, g in _dense_groups(self, bot_g, top_g, cross_g):
            if var is v:
                return None, Tensor(g)
        raise KeyError("variable does not belong to this model")

    def _bag_slices(self, sparse, k, dz):
        """IndexedSlices of table k's bags: the valid ids in (b, l) order, each with its bag's gradient row dz[b]
        (divided by the bag's valid-id count for a mean) -- what orx_bag_sparse_apply applies."""
        lo, L = self._col_off[k], self._bag_sizes[k]
        ids = sparse[:, lo:lo + L]
        valid = (ids >= 0) & (ids < self._latent_factors[k].embeddings.t.shape[0])
        rows = dz.unsqueeze(1).expand(-1, L, -1)
        if self._pooling == 1:
            rows = rows / valid.sum(1).clamp_min(1).to(torch.float32).view(-1, 1, 1)
        return Tensor(ids[valid].contiguous()), Tensor(rows[valid].contiguous())
