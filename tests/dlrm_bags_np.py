"""numpy restatement of multi-hot DLRM features (DLRM(bag_sizes=...), orx_bag_gather, orx_bag_sparse_apply): pooling in
float32 (the kernel's order, for exact comparisons) and float64, the IndexedSlices of a bag table, and one oracle
training step that runs the oracle's dlrm_forward / dlrm_backward on the pooled embeddings."""
import numpy as np

from oracle import openrec_oracle as O


def col_offsets(bag_sizes):
    return np.concatenate([[0], np.cumsum(bag_sizes)]).astype(np.int64)


def pool_f32(tables, sparse, col_off, mean):
    """-> (Z [B, T, D] float32, n [B, T] valid ids, n_bad): the valid rows added in column order in float32, starting
    from the first valid row; a mean divides by n; a bag without a valid id is the zero row."""
    B, T, D = sparse.shape[0], len(tables), tables[0].shape[1]
    Z = np.zeros((B, T, D), np.float32)
    cnt = np.zeros((B, T), np.int64)
    bad = 0
    for k, tab in enumerate(tables):
        tab = np.asarray(tab, np.float32)
        ids = sparse[:, col_off[k]:col_off[k + 1]]
        bad += int((ids >= tab.shape[0]).sum())
        acc = np.zeros((B, D), np.float32)
        n = np.zeros(B, np.int64)
        for l in range(ids.shape[1]):
            v = (ids[:, l] >= 0) & (ids[:, l] < tab.shape[0])
            row = tab[np.where(v, ids[:, l], 0)]
            acc = np.where((v & (n == 0))[:, None], row, np.where(v[:, None], acc + row, acc))
            n += v
        if mean:
            acc = np.where((n > 0)[:, None], acc / np.maximum(n, 1).astype(np.float32)[:, None], acc)
        Z[:, k], cnt[:, k] = acc, n
    return Z, cnt, bad


def pool64(tables, sparse, col_off, mean):
    """-> (Z [B, T, D] float64, n [B, T])."""
    B, T, D = sparse.shape[0], len(tables), tables[0].shape[1]
    Z = np.zeros((B, T, D))
    cnt = np.zeros((B, T), np.int64)
    for k, tab in enumerate(tables):
        tab = np.asarray(tab, np.float64)
        for c in range(col_off[k], col_off[k + 1]):
            v = (sparse[:, c] >= 0) & (sparse[:, c] < tab.shape[0])
            Z[:, k] += tab[np.where(v, sparse[:, c], 0)] * v[:, None]
            cnt[:, k] += v
        if mean:
            Z[:, k] /= np.maximum(cnt[:, k], 1)[:, None]
    return Z, cnt


def bag_slices(sparse, col_off, k, vocab, dz, mean):
    """IndexedSlices of table k: the valid ids in (b, l) order, each with dz[b] (/ the bag's valid ids for a mean)."""
    ids = sparse[:, col_off[k]:col_off[k + 1]]
    v = (ids >= 0) & (ids < vocab)
    rows = np.repeat(np.asarray(dz)[:, None, :], ids.shape[1], 1)
    if mean:
        rows = rows / np.maximum(v.sum(1), 1)[:, None, None]
    return ids[v].astype(np.int64), rows[v]


def forward(tabs, bot_w, bot_b, top_w, top_b, dense, sparse, col_off, mean, mode, **kw):
    """dlrm_forward of the pooled model: each pooled table is a [B, D] table looked up at row b."""
    Z, cnt = pool64(tabs, sparse, col_off, mean)
    B, T = Z.shape[0], Z.shape[1]
    ar = np.repeat(np.arange(B)[:, None], T, 1)
    pooled = [Z[:, k] for k in range(T)]
    cache = O.dlrm_forward(pooled, bot_w, bot_b, list(top_w), list(top_b), dense, ar, interaction_mode=mode, **kw)
    return cache, pooled, ar


def bag_grad_rows(sparse, col_off, k, vocab, dz, mean):
    """The IndexedSlices of table k already deduplicated: (unique valid ids, the sum of their rows), as one sparse
    [ids x B] product, so that a 100-id bag at B = 32768 needs no [B, L, D] copy."""
    import scipy.sparse as sps
    ids = sparse[:, col_off[k]:col_off[k + 1]]
    v = (ids >= 0) & (ids < vocab)
    b = np.repeat(np.arange(ids.shape[0])[:, None], ids.shape[1], 1)[v]
    w = (1.0 / np.maximum(v.sum(1), 1))[b] if mean else np.ones(len(b))
    uniq, row = np.unique(ids[v], return_inverse=True)
    M = sps.csr_matrix((w, (row.reshape(-1), b)), shape=(len(uniq), ids.shape[0]))
    return uniq.astype(np.int64), M @ np.asarray(dz, np.float64)


def train_step(kind, tabs, dvars, st, step, lr, dense, sparse, label, col_off, mean, mode, n_bot, apply_tables=None):
    """One oracle step in place on tabs (embedding tables; only those in apply_tables, default all) and dvars (Dense
    kernels / biases in model order), st the optimizer slots (tables first).  -> loss."""
    bot_w, bot_b = dvars[0:2 * n_bot:2], dvars[1:2 * n_bot:2]
    top_w, top_b = dvars[2 * n_bot::2], dvars[2 * n_bot + 1::2]
    cache, pooled, ar = forward(tabs, bot_w, bot_b, top_w, top_b, dense, sparse, col_off, mean, mode)
    loss, dpred = O.dlrm_loss(cache["pred"], label, "mse")
    gr = O.dlrm_backward(cache, pooled, bot_w, list(top_w), dense, ar, dpred, interaction_mode=mode)
    T = len(tabs)
    for k in range(T) if apply_tables is None else apply_tables:
        ids, rows = bag_grad_rows(sparse, col_off, k, tabs[k].shape[0], gr["emb"][k], mean)
        O.apply_sparse(kind, tabs[k], st[k][0], st[k][1], ids, rows, step, lr)
    dgr = []
    for l in range(n_bot):
        dgr += [gr["bot_w"][l], gr["bot_b"][l]]
    for l in range(len(top_w)):
        dgr += [gr["top_w"][l], gr["top_b"][l]]
    for j, g in enumerate(dgr):
        O.apply_dense(kind, dvars[j], st[T + j][0], st[T + j][1], g, step, lr)
    return loss
