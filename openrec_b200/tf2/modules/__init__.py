"""The building blocks the tf2 recommenders are composed of: the five names ``openrec.tf2.modules`` exports, and the
DCN-v2 ``CrossNetwork`` (DLRM's arch_interaction_op="cross")."""
from importlib import import_module

_HOME = {"LatentFactor": "latent_factor", "PairwiseLogLoss": "pairwise_log_loss", "PointwiseMSELoss": "pointwise_mse_loss",
         "MLP": "multi_layer_perceptron", "SecondOrderFeatureInteraction": "second_order_feature_interaction",
         "CrossNetwork": "cross_network"}
for _cls, _module in _HOME.items():
    globals()[_cls] = getattr(import_module(f"{__name__}.{_module}"), _cls)
__all__ = sorted(_HOME)
