"""RankingEvaluator -- AUC / NDCG / Recall of every warm user of a dataset at catalogue scale, in one fused liborx call
per batch (orx_score_rank): the users are scored against the whole item table and the ranks counted in the same pass,
so neither the [users, items] score matrix nor the per-user masks of ``Dataset.evaluation`` are ever built.
CandidateEvaluator -- the same for a dataset with explicit negatives, each user ranked against its listed items only
(orx_score_rank_listed): only the listed items and the positives are scored.

The results equal those of the reference example's loop (``Dataset.evaluation`` + ``model.inference`` + ``AUC`` /
``NDCG`` / ``Recall``) for the same users in the same order.  The positives of ``val_dataset`` and the union of the
positives of ``excl_datasets`` become two CSR lists over user ids, uploaded once; a batch then only needs its user ids.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import native as N
from ..._lib import ORX_MAX_AT
from ...sharded import all_reduce_sum, score_rank_listed_sharded, score_rank_sharded
from ...tfshim.core import Tensor
from ..data.user_lists import positives_csr, user_csr


class _UserBatchEvaluator:
    """What RankingEvaluator and CandidateEvaluator share: the warm users of ``val_dataset``, their positives and the
    union of the positives of ``excl_datasets`` as CSR lists over user ids (uploaded once per device), and the walk
    over the warm users in batches of ``batch_size``, one fused liborx call per batch on one device or one collective
    sharded call per batch on every rank.  A subclass names its lists (``_lists``, in the call's argument order after
    the user ids), its engine method (``_one``) and its sharded driver (``_sharded``)."""

    _what = ""

    def __init__(self, store, excl_datasets, at, batch_size):
        if len(at) > ORX_MAX_AT:
            raise ValueError(f"at most {ORX_MAX_AT} cut-offs")
        if batch_size < 1:
            raise ValueError("batch_size must be positive")
        self.at = tuple(int(k) for k in at)
        self.batch_size = int(batch_size)
        n_users = store.total_users()
        self.warm_users = np.asarray(store.warm_users(), dtype=np.int64)
        self.pos_off, self.pos_items = user_csr(n_users, {u: store.get_positive_items(u) for u in self.warm_users})
        self.excl_off, self.excl_items = positives_csr(n_users, excl_datasets)
        self._pos_len = np.diff(self.pos_off)
        self.max_pos = int(self._pos_len.max()) if n_users else 0
        self._dev = None

    def _lists(self):
        return self.pos_off, self.pos_items, self.excl_off, self.excl_items

    def _upload(self, device):
        if self._dev is None or self._dev[0] != device:
            put = lambda a: torch.from_numpy(a).to(device)                       # noqa: E731
            self._dev = (device, put(self.warm_users.astype(np.int32))) + tuple(put(a) for a in self._lists())
        return self._dev[1:]

    def evaluate(self, model):
        """A row-sharded model (ShardedBPR / ShardedUCML / ShardedGMF / ShardedWRMF) is evaluated collectively: every
        rank builds the same evaluator and calls evaluate; each rank counts over its own item rows and every rank gets
        the same result."""
        sharded = getattr(model, "_sharded_score_operands", None)
        if sharded is not None:
            return self._evaluate_sharded(*sharded())
        ops = getattr(model, "_score_operands", None)
        if ops is None:
            raise NotImplementedError(f"{type(model).__name__}: {self._what} needs the model's whole item "
                                      "table on one device (BPR, UCML, GMF, WRMF) or its row shards (ShardedBPR, "
                                      "ShardedUCML, ShardedGMF, ShardedWRMF)")
        kind, user, item, bias, scale = ops()
        one = getattr(N.engine(), self._one)
        return self._batches(item.device, lambda uids, lists, max_pos: one(
            kind, user, uids, item, bias, *lists, max_pos, at=self.at, scale=scale))

    def _evaluate_sharded(self, kind, user, item, bias, g, group, scale=None):
        part = (N.engine(), kind, user, item, bias, g)
        reduce = all_reduce_sum(group)
        return self._batches(item.device, lambda uids, lists, max_pos: self._sharded(
            [part], reduce, uids, *lists, max_pos, at=self.at, scale=[scale])[0])

    def _batches(self, device, call):
        """call(uids, lists, max_pos) -> (auc, ndcg, recall) of one batch, over the warm users in order."""
        uids, *lists = self._upload(device)
        auc, ndcg, rec = [], [], []
        for b0 in range(0, len(self.warm_users), self.batch_size):
            b1 = min(b0 + self.batch_size, len(self.warm_users))
            max_pos = int(self._pos_len[self.warm_users[b0:b1]].max())
            a, n, r = call(uids[b0:b1], lists, max_pos)
            auc.append(a), ndcg.append(n), rec.append(r)
        return self._result(auc, ndcg, rec, device)

    def _result(self, auc, ndcg, rec, device):
        if not auc:
            empty = torch.zeros((0, len(self.at)), dtype=torch.float32, device=device)
            return {"AUC": Tensor(empty[:, 0]), "NDCG": Tensor(empty), "Recall": Tensor(empty.clone())}
        return {"AUC": Tensor(torch.cat(auc)), "NDCG": Tensor(torch.cat(ndcg)), "Recall": Tensor(torch.cat(rec))}


class RankingEvaluator(_UserBatchEvaluator):
    """``RankingEvaluator(val_dataset, excl_datasets=[train_dataset], at=[50, 100], batch_size=1024).evaluate(model)``
    -> {'AUC': [n_warm], 'NDCG': [n_warm, len(at)], 'Recall': [n_warm, len(at)]} in ``warm_users()`` order, ready for
    ``DictMean.update_state``.  Ranks against the whole catalogue, so a dataset with explicit negatives (ranked against
    its listed items only) is not supported: use ``CandidateEvaluator`` for those."""

    _what, _one, _sharded = "catalogue evaluation", "score_rank", staticmethod(score_rank_sharded)

    def __init__(self, val_dataset, excl_datasets=[], at=[100], batch_size=1024):
        store = val_dataset.datastore
        if store.contain_negatives():
            raise NotImplementedError("RankingEvaluator ranks against the whole catalogue; a dataset with explicit "
                                      "negatives ranks against its listed items only (use CandidateEvaluator)")
        super().__init__(store, excl_datasets, at, batch_size)


class CandidateEvaluator(_UserBatchEvaluator):
    """``CandidateEvaluator(val_dataset, excl_datasets=[], at=[100], batch_size=1024).evaluate(model)`` -> the dict of
    ``RankingEvaluator`` for a dataset with explicit negatives (``num_negatives`` or ``implicit_negative=False``): each
    warm user's positives ranked against that user's listed items only, as ``Dataset.evaluation`` masks them (items
    neither positive nor listed, and the positives of ``excl_datasets``, are left out).  One orx_score_rank_listed call
    per batch scores only the listed items and positives, never the whole catalogue."""

    _what, _one, _sharded = "listed-candidate evaluation", "score_rank_listed", staticmethod(score_rank_listed_sharded)

    def __init__(self, val_dataset, excl_datasets=[], at=[100], batch_size=1024):
        store = val_dataset.datastore
        if not store.contain_negatives():
            raise ValueError("CandidateEvaluator ranks against each user's listed negatives, and this dataset lists "
                             "none; rank against the whole catalogue with RankingEvaluator")
        super().__init__(store, excl_datasets, at, batch_size)
        self.neg_off, self.neg_items = user_csr(store.total_users(),
                                                {u: store.get_negative_items(u) for u in self.warm_users})

    def _lists(self):
        return self.pos_off, self.pos_items, self.neg_off, self.neg_items, self.excl_off, self.excl_items
