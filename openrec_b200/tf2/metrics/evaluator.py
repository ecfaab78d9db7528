"""RankingEvaluator -- AUC / NDCG / Recall of every warm user of a dataset at catalogue scale, in one fused liborx call
per batch (orx_score_rank): the users are scored against the whole item table and the ranks counted in the same pass,
so neither the [users, items] score matrix nor the per-user masks of ``Dataset.evaluation`` are ever built.

The results equal those of the reference example's loop (``Dataset.evaluation`` + ``model.inference`` + ``AUC`` /
``NDCG`` / ``Recall``) for the same users in the same order.  The positives of ``val_dataset`` and the union of the
positives of ``excl_datasets`` become two CSR lists over user ids, uploaded once; a batch then only needs its user ids.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import native as N
from ..._lib import ORX_MAX_AT
from ...sharded import all_reduce_sum, score_rank_sharded
from ...tfshim.core import Tensor
from ..data.user_lists import positives_csr, user_csr


class RankingEvaluator:
    """``RankingEvaluator(val_dataset, excl_datasets=[train_dataset], at=[50, 100], batch_size=1024).evaluate(model)``
    -> {'AUC': [n_warm], 'NDCG': [n_warm, len(at)], 'Recall': [n_warm, len(at)]} in ``warm_users()`` order, ready for
    ``DictMean.update_state``.  Ranks against the whole catalogue, so a dataset with explicit negatives (ranked against
    its listed items only) is not supported: use ``Dataset.evaluation`` for those."""

    def __init__(self, val_dataset, excl_datasets=[], at=[100], batch_size=1024):
        store = val_dataset.datastore
        if store.contain_negatives():
            raise NotImplementedError("RankingEvaluator ranks against the whole catalogue; a dataset with explicit "
                                      "negatives ranks against its listed items only (use Dataset.evaluation)")
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

    def _upload(self, device):
        if self._dev is None or self._dev[0] != device:
            put = lambda a: torch.from_numpy(a).to(device)                       # noqa: E731
            self._dev = (device, put(self.warm_users.astype(np.int32)), put(self.pos_off), put(self.pos_items),
                         put(self.excl_off), put(self.excl_items))
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
            raise NotImplementedError(f"{type(model).__name__}: catalogue evaluation needs the model's whole item "
                                      "table on one device (BPR, UCML, GMF, WRMF) or its row shards (ShardedBPR, "
                                      "ShardedUCML, ShardedGMF, ShardedWRMF)")
        kind, user, item, bias, scale = ops()
        uids, pos_off, pos_items, excl_off, excl_items = self._upload(item.device)
        eng = N.engine()
        auc, ndcg, rec = [], [], []
        for b0 in range(0, len(self.warm_users), self.batch_size):
            b1 = min(b0 + self.batch_size, len(self.warm_users))
            max_pos = int(self._pos_len[self.warm_users[b0:b1]].max())
            a, n, r = eng.score_rank(kind, user, uids[b0:b1], item, bias, pos_off, pos_items, excl_off, excl_items,
                                     max_pos, at=self.at, scale=scale)
            auc.append(a), ndcg.append(n), rec.append(r)
        return self._result(auc, ndcg, rec, item.device)

    def _evaluate_sharded(self, kind, user, item, bias, g, group, scale=None):
        uids, pos_off, pos_items, excl_off, excl_items = self._upload(item.device)
        part = (N.engine(), kind, user, item, bias, g)
        reduce = all_reduce_sum(group)
        auc, ndcg, rec = [], [], []
        for b0 in range(0, len(self.warm_users), self.batch_size):
            b1 = min(b0 + self.batch_size, len(self.warm_users))
            max_pos = int(self._pos_len[self.warm_users[b0:b1]].max())
            (a, n, r), = score_rank_sharded([part], reduce, uids[b0:b1], pos_off, pos_items, excl_off, excl_items,
                                            max_pos, at=self.at, scale=[scale])
            auc.append(a), ndcg.append(n), rec.append(r)
        return self._result(auc, ndcg, rec, item.device)

    def _result(self, auc, ndcg, rec, device):
        if not auc:
            empty = torch.zeros((0, len(self.at)), dtype=torch.float32, device=device)
            return {"AUC": Tensor(empty[:, 0]), "NDCG": Tensor(empty), "Recall": Tensor(empty.clone())}
        return {"AUC": Tensor(torch.cat(auc)), "NDCG": Tensor(torch.cat(ndcg)), "Recall": Tensor(torch.cat(rec))}
