"""Retriever -- each user's k best unseen items at catalogue scale, in one fused liborx call per batch of users
(orx_score_topk): the users are scored against the whole item table and only the k best items of each are kept, so the
[users, items] score matrix of ``model.inference`` is never built.

The result equals ``model.inference(users)`` with the users' excluded items left out, ordered by score descending and
then item id ascending (NaN scores are never returned), cut at k and padded with item -1 / score -inf when fewer items
remain.  The union of the positives of ``excl_datasets`` becomes one CSR list over user ids, uploaded once per device.
The reference's tf2 package has no serving path; its tf1 ``FastDotProductServer`` is the closest counterpart.

A row-sharded model (ShardedBPR / ShardedUCML / ShardedGMF / ShardedWRMF) is served where its rows live: ``recommend``
is then a collective call (orx_score_topk_shard) in which each rank keeps the k best of its own item rows and one merge
over the ranks' lists gives every rank the result of the single-device call on the gathered tables (GMF: the summed
user rows are scaled by w first, orx_rows_scale).  No table row crosses the interconnect."""
from __future__ import annotations

import torch
import torch.distributed as dist

from ... import native as N
from ..._lib import ORX_MAX_TOPK
from ...sharded import all_reduce_sum, score_topk_sharded
from ...tfshim.core import Tensor
from ..data.user_lists import positives_csr
from ._base import ids_of


class Retriever:
    """``Retriever(excl_datasets=[train_dataset], k=10, batch_size=1024).recommend(model, user_id)`` -> (items, scores),
    int32 / float32 ``Tensor``s of shape [n, k] on the model's device, n = the number of ids in ``user_id`` (a host or
    device array of ints of any shape, flattened).  Models: BPR, UCML, GMF, WRMF, and ShardedBPR / ShardedUCML /
    ShardedGMF / ShardedWRMF, on which every rank must call ``recommend`` with the same ids and gets the same result."""

    def __init__(self, excl_datasets=[], k=10, batch_size=1024):
        k = int(k)
        if not 1 <= k <= ORX_MAX_TOPK:
            raise ValueError(f"k must lie in [1, {ORX_MAX_TOPK}]")
        if batch_size < 1:
            raise ValueError("batch_size must be positive")
        totals = {int(ds.datastore.total_users()) for ds in excl_datasets}
        if len(totals) > 1:
            raise ValueError(f"excl_datasets disagree on total_users: {sorted(totals)}")
        self.k, self.batch_size = k, int(batch_size)
        self.excl_off, self.excl_items = positives_csr(totals.pop(), excl_datasets) if totals else (None, None)
        self._dev = None

    def _upload(self, device):
        if self.excl_off is None:
            return None, None
        if self._dev is None or self._dev[0] != device:
            self._dev = (device, torch.from_numpy(self.excl_off).to(device), torch.from_numpy(self.excl_items).to(device))
        return self._dev[1:]

    def recommend(self, model, user_id):
        sharded = getattr(model, "_sharded_score_operands", None)
        if sharded is not None:
            return self._recommend_sharded(ids_of(user_id), *sharded())
        ops = getattr(model, "_score_operands", None)
        if ops is None:
            raise NotImplementedError(f"{type(model).__name__}: catalogue retrieval needs the model's whole item "
                                      "table on one device (BPR, UCML, GMF, WRMF) or its row shards (ShardedBPR, "
                                      "ShardedUCML, ShardedGMF, ShardedWRMF)")
        kind, user, item, bias, scale = ops()
        uids = ids_of(user_id)
        excl_off, excl_items = self._upload(item.device)
        eng = N.engine()
        items, scores = [], []
        for b0 in range(0, uids.numel(), self.batch_size):
            it, sc = eng.score_topk(kind, user, uids[b0:b0 + self.batch_size], item, bias, excl_off, excl_items,
                                    self.k, scale=scale)
            items.append(it), scores.append(sc)
        return self._result(items, scores, item.device)

    def _recommend_sharded(self, uids, kind, user, item, bias, g, group, scale=None):
        # every rank must issue the same batches: unequal id counts would leave some ranks waiting in the exchange
        n = torch.tensor([uids.numel(), -uids.numel()], dtype=torch.int64, device=item.device)
        dist.all_reduce(n, op=dist.ReduceOp.MIN, group=group)
        lo, hi = int(n[0]), -int(n[1])
        if lo != hi:
            raise ValueError(f"Retriever.recommend on a sharded model: the ranks passed between {lo} and {hi} user "
                             "ids; every rank must pass the same ids")
        excl_off, excl_items = self._upload(item.device)
        part = (N.engine(), kind, user, item, bias, g)
        reduce = all_reduce_sum(group)
        items, scores = [], []
        for b0 in range(0, uids.numel(), self.batch_size):
            (it, sc), = score_topk_sharded([part], reduce, uids[b0:b0 + self.batch_size], excl_off, excl_items, self.k,
                                           scale=[scale])
            items.append(it), scores.append(sc)
        return self._result(items, scores, item.device)

    def _result(self, items, scores, device):
        if not items:
            return (Tensor(torch.zeros((0, self.k), dtype=torch.int32, device=device)),
                    Tensor(torch.zeros((0, self.k), dtype=torch.float32, device=device)))
        return Tensor(torch.cat(items)), Tensor(torch.cat(scores))
