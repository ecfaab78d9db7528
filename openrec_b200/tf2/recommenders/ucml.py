"""UCML -- mirrors openrec/tf2/recommenders/ucml.py:5-53 on the fused liborx step (K2)."""
from ... import native as N
from ..modules import LatentFactor
from .bpr import BPR
from ._base import FusedRecommender, _check_dtype


class UCML(BPR):
    _kind = N.ORX_PAIR_UCML
    _score = N.ORX_SCORE_NEG_SQDIST

    def __init__(self, dim_user_embed, dim_item_embed, total_users, total_items, margin=0.5, embedding_dtype="float32",
                 rounding_seed=0):
        FusedRecommender.__init__(self)
        self.embedding_dtype, self.rounding_seed = _check_dtype(embedding_dtype), int(rounding_seed)
        self.user_latent_factor = LatentFactor(num_instances=total_users, dim=dim_user_embed,
                                               name="user_latent_factor", dtype=embedding_dtype)
        self.item_latent_factor = LatentFactor(num_instances=total_items, dim=dim_item_embed,
                                               name="item_latent_factor", dtype=embedding_dtype)
        self.item_bias = LatentFactor(num_instances=total_items, dim=1, name="item_bias")
        self.margin = margin

    def _get_margin(self):
        return float(self.margin)

    def censor_vec(self, user_id, p_item_id, n_item_id):
        """three sequential censors, in the reference's order (ucml.py:44-48)."""
        return (self.user_latent_factor.censor(user_id), self.item_latent_factor.censor(p_item_id),
                self.item_latent_factor.censor(n_item_id))
