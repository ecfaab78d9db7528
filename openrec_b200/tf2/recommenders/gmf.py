"""GMF -- mirrors openrec/tf2/recommenders/gmf.py:5-41 on the fused liborx step (K3)."""
import torch

from ... import native as N
from ..modules import MLP, LatentFactor
from ._base import FusedRecommender, w_table
from .wrmf import WRMF


class GMF(WRMF):
    _kind = N.ORX_POINT_GMF

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items):
        FusedRecommender.__init__(self)
        self.user_latent_factor = LatentFactor(num_instances=total_users, dim=dim_user_embed,
                                               name="user_latent_factor")
        self.item_latent_factor = LatentFactor(num_instances=total_items, dim=dim_item_embed,
                                               name="item_latent_factor")
        self.item_bias = LatentFactor(num_instances=total_items, dim=1, name="item_bias")
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
        return (N.ORX_SCORE_DOT, self.user_latent_factor.embeddings.t, self.item_latent_factor.embeddings.t,
                self.item_bias.embeddings.t, self.mlp.layers[0].kernel.t.reshape(-1))
