"""Per-user item lists as CSR arrays over user ids: the form in which the catalogue-scale calls (orx_score_rank,
orx_score_topk) take positives and exclusions, so that a batch only needs its user ids.  Used by
``openrec.tf2.metrics.RankingEvaluator`` and ``openrec.tf2.recommenders.Retriever``."""
from __future__ import annotations

import numpy as np


def user_csr(n_rows, rows):
    """{user: iterable of items} -> (offsets int64 [n_rows + 1], items int32): each row sorted and unique, users
    without an entry (or outside [0, n_rows)) empty."""
    lens = np.zeros(n_rows, dtype=np.int64)
    parts = {}
    for u, items in rows.items():
        u = int(u)
        if 0 <= u < n_rows:
            parts[u] = np.unique(np.fromiter(items, dtype=np.int64))
            lens[u] = len(parts[u])
    off = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    items = np.concatenate([parts[u] for u in sorted(parts)]) if parts else np.zeros(0, dtype=np.int64)
    return off, items.astype(np.int32)


def positives_csr(n_rows, datasets):
    """The union of the positives of ``datasets`` (``Dataset`` objects), one sorted, unique row per user."""
    rows = {}
    for ds in datasets:
        store = ds.datastore
        for u in store.warm_users():
            rows.setdefault(int(u), set()).update(store.get_positive_items(u))
    return user_csr(n_rows, rows)
