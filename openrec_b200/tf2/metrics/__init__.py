"""openrec.tf2.metrics surface (reference: openrec/tf2/metrics/__init__.py:1-2)."""
from .ranking_metrics import AUC, NDCG, Recall
from .dict_mean import DictMean
from .evaluator import CandidateEvaluator, RankingEvaluator

__all__ = ["AUC", "NDCG", "Recall", "DictMean", "RankingEvaluator", "CandidateEvaluator"]
