"""WRMF -- mirrors openrec/tf2/recommenders/wrmf.py:5-40 on the fused liborx step (K4)."""
import torch

from ... import native as N
from ...tfshim.core import Tensor, convert
from ..modules import LatentFactor, PointwiseMSELoss
from ._base import FusedRecommender, _check_dtype, ids_of


class WRMF(FusedRecommender):
    """``embedding_dtype="bfloat16"`` stores the user and item tables in bfloat16 (the item bias and every optimizer
    slot stay float32); each step rounds its updates stochastically, seeded by ``rounding_seed`` and the optimizer's
    iteration count, so a run is reproducible bit for bit.  ``inference``, the evaluators and ``Retriever`` score the
    bfloat16 tables in place, with results bit-equal to scoring their float32 upcast."""
    _kind = N.ORX_POINT_WRMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, a=1.0, b=1.0,
                 embedding_dtype="float32", rounding_seed=0):
        super().__init__()
        self._latent_factors(dim_user_embed, dim_item_embed, total_users, total_items, embedding_dtype, rounding_seed)
        self.pointwise_mse_loss = PointwiseMSELoss(a=a, b=b)

    def _latent_factors(self, dim_user_embed, dim_item_embed, total_users, total_items, embedding_dtype,
                        rounding_seed):
        """user / item tables of embedding_dtype and the float32 item bias."""
        self.embedding_dtype, self.rounding_seed = _check_dtype(embedding_dtype), int(rounding_seed)
        self.user_latent_factor = LatentFactor(num_instances=total_users, dim=dim_user_embed,
                                               name="user_latent_factor", dtype=embedding_dtype)
        self.item_latent_factor = LatentFactor(num_instances=total_items, dim=dim_item_embed,
                                               name="item_latent_factor", dtype=embedding_dtype)
        self.item_bias = LatentFactor(num_instances=total_items, dim=1, name="item_bias")

    def _bf16(self):
        return self.embedding_dtype == "bfloat16"

    def _point_params(self):
        l = self.pointwise_mse_loss
        return float(l._a), float(l._b), bool(l._sigmoid)

    def _w(self, optimizer=None):
        return None

    def call(self, user_id, item_id, label):
        """-> (loss, l2_loss) (wrmf.py:21-34)."""
        lab = convert(label).t.to(torch.float32).reshape(-1).contiguous()
        _, loss, l2 = self._new_node(ids_of(user_id), ids_of(item_id), lab)
        return loss, l2

    def _orx_forward(self, node):
        a, b, sig = self._point_params()
        fwd = N.engine().pointwise_fwd_bf16 if self._bf16() else N.engine().pointwise_fwd
        fwd(self._kind, *self._tables(), self._w(), *self._device_ids(node), node.out, a, b, sig)

    def _orx_run_step(self, node, optimizer, c_loss, c_l2):
        a, b, sig = self._point_params()
        if self._bf16():
            N.engine().pointwise_step_bf16(self._kind, *self._tables(optimizer), self._w(optimizer),
                                           *self._device_ids(node), optimizer.opt_struct(), self.rounding_seed,
                                           node.out, a, b, sig, c_loss, c_l2)
            return
        N.engine().pointwise_step(self._kind, *self._tables(optimizer), self._w(optimizer), *self._device_ids(node),
                                  optimizer.opt_struct(), node.out, a, b, sig, c_loss, c_l2)

    def _orx_run_grad(self, node, var, c_loss, c_l2):
        uid, iid, lab = self._device_ids(node)
        B, D = uid.numel(), self.user_latent_factor.output_dim
        dev = uid.device
        a, b, sig = self._point_params()
        kw, idx = {}, iid
        if var is self.user_latent_factor.embeddings:
            kw["d_user"], idx = torch.empty(B, D, device=dev), uid
        elif var is self.item_latent_factor.embeddings:
            kw["d_item"] = torch.empty(B, D, device=dev)
        elif var is self.item_bias.embeddings:
            kw["d_bias"] = torch.empty(B, device=dev)
        else:
            kw["d_w"] = torch.empty(D, device=dev)
        grad = N.engine().pointwise_grad_bf16 if self._bf16() else N.engine().pointwise_grad
        grad(self._kind, *self._tables(), self._w(), uid, iid, lab, a, b, sig, c_loss, c_l2, **kw)
        if "d_w" in kw:   # dense variable: a dense gradient, like TF returns for Dense kernels
            return None, Tensor(kw["d_w"].reshape(tuple(var.t.shape)))
        val = next(iter(kw.values()))
        return Tensor(idx), Tensor(val.reshape(B, -1))

    def _score_tables(self):
        """(user, item) tables to score: the stored tables, so bf16 ones are read in place by the _bf16 entry points."""
        return self.user_latent_factor.embeddings.t, self.item_latent_factor.embeddings.t

    def _score_operands(self):
        """(kind, user table, item table, item bias, scale) of the full-catalogue score (inference, RankingEvaluator,
        CandidateEvaluator, Retriever), on the stored tables (_score_tables)."""
        return (N.ORX_SCORE_DOT, *self._score_tables(), self.item_bias.embeddings.t, None)

    def inference(self, user_id):
        """U[user] @ Item^T + bias (wrmf.py:36-40)."""
        kind, user, item, bias, scale = self._score_operands()
        return Tensor(N.engine().score_all(kind, user, ids_of(user_id), item, bias, scale=scale))
