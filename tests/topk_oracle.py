"""TEST INFRASTRUCTURE: numpy restatement of orx_score_topk's order and padding rules on a dense score matrix (the GPU
tests apply it to orx_score_all output, the CPU tests use it in the oracle-backed engine, bench_topk.py checks the fused
call with it)."""
import numpy as np


def topk(pred, excl_mask, k):
    """pred float32 [R, I], excl_mask bool [R, I] (or None) -> (items int32 [R, k], scores float32 [R, k]): per row the
    first k items that are not excluded and whose score is not NaN, in the order score descending (floats: -0.0 ==
    +0.0), then item id ascending; slots past the eligible items hold item -1 and score -inf."""
    pred = np.asarray(pred, np.float32)
    R, I = pred.shape
    items = np.full((R, k), -1, np.int32)
    scores = np.full((R, k), -np.inf, np.float32)
    for r in range(R):
        ok = ~np.isnan(pred[r])
        if excl_mask is not None:
            ok &= ~np.asarray(excl_mask[r], bool)
        idx = np.flatnonzero(ok)
        s = pred[r, idx]
        take = np.lexsort((idx, -s))[:k]     # primary key -s (sorts by comparison: -0.0 ties +0.0), then the id
        items[r, :len(take)] = idx[take]
        scores[r, :len(take)] = s[take]
    return items, scores
