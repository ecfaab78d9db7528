"""GMF -- mirrors openrec/tf2/recommenders/gmf.py:5-41 on the fused liborx step (K3)."""
import torch

from ... import native as N
from ..modules import MLP
from ._base import FusedRecommender, w_table
from .wrmf import WRMF


class GMF(WRMF):
    """``embedding_dtype="bfloat16"`` stores the user and item tables in bfloat16 (the item bias, ``w`` and every
    optimizer slot stay float32); each step rounds its updates stochastically, seeded by ``rounding_seed`` and the
    optimizer's iteration count, so a run is reproducible bit for bit.  ``inference``, the evaluators and ``Retriever``
    score the bfloat16 tables in place (``w`` and the bias in float32), with results bit-equal to scoring their float32
    upcast."""
    _kind = N.ORX_POINT_GMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, embedding_dtype="float32",
                 rounding_seed=0):
        FusedRecommender.__init__(self)
        self._latent_factors(dim_user_embed, dim_item_embed, total_users, total_items, embedding_dtype, rounding_seed)
        self.mlp = MLP(units_list=[1], use_bias=False)
        self.mlp.build(dim_user_embed)   # Dense(1) kernel [D,1], glorot uniform (gmf.py:19)

    def _point_params(self):
        return 1.0, 1.0, False

    def _w(self, optimizer=None):
        k = self.mlp.layers[0].kernel
        if optimizer is None:
            return w_table(k.t)
        s0, s1 = optimizer.slots(k)
        return w_table(k.t, s0, s1)

    def _score_operands(self):
        """(u * w) . item^T + bias (gmf.py:36-41): WRMF's score with GMF's w as the user-side scale."""
        return (N.ORX_SCORE_DOT, *self._score_tables(), self.item_bias.embeddings.t,
                self.mlp.layers[0].kernel.t.reshape(-1))
