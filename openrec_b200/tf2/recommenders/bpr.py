"""BPR -- mirrors openrec/tf2/recommenders/bpr.py:5-43 on the fused liborx step (K1)."""
import torch

from ... import native as N
from ...tfshim.core import Tensor
from ..modules import LatentFactor, PairwiseLogLoss
from ._base import FusedRecommender, _check_dtype, ids_any, ids_of


class BPR(FusedRecommender):
    """``embedding_dtype="bfloat16"`` stores the user and item tables in bfloat16 (the item bias and every optimizer
    slot stay float32); each step rounds its updates stochastically, seeded by ``rounding_seed`` and the optimizer's
    iteration count, so a run is reproducible bit for bit.  ``inference``, the evaluators and ``Retriever`` score the
    bfloat16 tables in place, with results bit-equal to scoring their float32 upcast."""
    _kind = N.ORX_PAIR_BPR
    _score = N.ORX_SCORE_DOT

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, embedding_dtype="float32",
                 rounding_seed=0):
        super().__init__()
        self.embedding_dtype, self.rounding_seed = _check_dtype(embedding_dtype), int(rounding_seed)
        self.user_latent_factor = LatentFactor(num_instances=total_users, dim=dim_user_embed,
                                               name="user_latent_factor", dtype=embedding_dtype)
        self.item_latent_factor = LatentFactor(num_instances=total_items, dim=dim_item_embed,
                                               name="item_latent_factor", dtype=embedding_dtype)
        self.item_bias = LatentFactor(num_instances=total_items, dim=1, name="item_bias")
        self.pairwise_log_loss = PairwiseLogLoss()

    def _bf16(self):
        return self.embedding_dtype == "bfloat16"

    def _get_margin(self):
        return 0.0

    def call(self, user_id, p_item_id, n_item_id):
        """-> (loss, l2_loss) as lazy scalars (bpr.py:21-37)."""
        ids = [ids_any(x) for x in (user_id, p_item_id, n_item_id)]
        if all(h for _, h in ids):     # host batch: stays in pinned memory until the fused step takes it
            _, loss, l2 = self._new_node(host_ids=tuple(t for t, _ in ids))
            return loss, l2
        dev = self.user_latent_factor.embeddings.t.device
        _, loss, l2 = self._new_node(*(t.to(dev, non_blocking=True) if h else t for t, h in ids))
        return loss, l2

    # ---- kernels behind the step protocol
    def _orx_forward(self, node):
        fwd = N.engine().pairwise_fwd_bf16 if self._bf16() else N.engine().pairwise_fwd
        fwd(self._kind, *self._tables(), *self._device_ids(node), node.out, self._get_margin())

    def _orx_run_step(self, node, optimizer, c_loss, c_l2):
        if self._bf16():
            N.engine().pairwise_step_bf16(self._kind, *self._tables(optimizer), *self._device_ids(node),
                                          optimizer.opt_struct(), self.rounding_seed, node.out, self._get_margin(),
                                          c_loss, c_l2)
            return
        N.engine().pairwise_step(self._kind, *self._tables(optimizer), *self._device_ids(node),
                                 optimizer.opt_struct(), node.out, self._get_margin(), c_loss, c_l2)

    def _orx_run_step_host(self, node, optimizer, c_loss, c_l2):
        """ids in pinned host memory -> orx_pairwise_step_host: H2D, the three kernels and the D2H of
        (loss, l2_loss) are one C call's worth of stream work; the result lands in a pinned buffer."""
        buf, ev = self._out_ring().take(node, keep=node.host_ids)
        if self._bf16():
            N.engine().pairwise_step_host_bf16(self._kind, *self._tables(optimizer), *node.host_ids,
                                               optimizer.opt_struct(), self.rounding_seed, buf, self._get_margin(),
                                               c_loss, c_l2)
        else:
            N.engine().pairwise_step_host(self._kind, *self._tables(optimizer), *node.host_ids,
                                          optimizer.opt_struct(), buf, self._get_margin(), c_loss, c_l2)
        ev.record()
        node.out_host, node.event = buf, ev

    def _orx_run_grad(self, node, var, c_loss, c_l2):
        uid, pid, nid = self._device_ids(node)
        B, D = uid.numel(), self.user_latent_factor.output_dim
        dev = uid.device
        kw = {}
        if var is self.user_latent_factor.embeddings:
            kw["d_user"] = out = torch.empty(B, D, device=dev)
            idx = uid
        elif var is self.item_latent_factor.embeddings:
            kw["d_pos"], kw["d_neg"] = torch.empty(B, D, device=dev), torch.empty(B, D, device=dev)
            idx = torch.cat([pid, nid])
        else:
            kw["d_bp"], kw["d_bn"] = torch.empty(B, device=dev), torch.empty(B, device=dev)
            idx = torch.cat([pid, nid])
        grad = N.engine().pairwise_grad_bf16 if self._bf16() else N.engine().pairwise_grad
        grad(self._kind, *self._tables(), uid, pid, nid, self._get_margin(), c_loss, c_l2, **kw)
        if "d_user" in kw:
            val = out
        elif "d_pos" in kw:
            val = torch.cat([kw["d_pos"], kw["d_neg"]])
        else:
            val = torch.cat([kw["d_bp"], kw["d_bn"]]).reshape(-1, 1)
        return Tensor(idx), Tensor(val)

    def _score_operands(self):
        """(kind, user table, item table, item bias, scale) of the full-catalogue score (inference, RankingEvaluator,
        CandidateEvaluator, Retriever): the stored tables, so bf16 ones are read in place by the _bf16 entry points."""
        return (self._score, self.user_latent_factor.embeddings.t, self.item_latent_factor.embeddings.t,
                self.item_bias.embeddings.t, None)

    def inference(self, user_id):
        """scores [Bu, total_items] = U[user] @ Item^T + bias (bpr.py:39-43)."""
        kind, user, item, bias, scale = self._score_operands()
        return Tensor(N.engine().score_all(kind, user, ids_of(user_id), item, bias, scale=scale))
