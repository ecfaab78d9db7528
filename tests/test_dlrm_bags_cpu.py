"""CPU: DLRM(bag_sizes=...)'s constructor refusals and the numpy restatement of pooled bags (tests/dlrm_bags_np.py)."""
import os
import sys

import numpy as np
import pytest

import dlrm_bags_np as NB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("bad", [dict(bag_sizes=[1]), dict(bag_sizes=[2, 0]), dict(bag_sizes=[1, -3]),
                                 dict(bag_sizes=[1, 1], pooling="max"), dict(pooling="sqrtn"),
                                 dict(bag_sizes=[1] * 64, ln_emb=[10] * 64)])
def test_dlrm_bag_arguments_refused(bad):
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    from openrec.tf2.recommenders import DLRM
    kw = dict(m_spa=8, ln_emb=[10, 20], ln_bot=[8], ln_top=[4, 1])
    kw.update(bad)
    with pytest.raises(ValueError):
        DLRM(**kw)


def test_pooling_restatements_agree():
    rng = np.random.default_rng(3)
    sizes, vocab, B, D = [1, 4, 33], [5, 40, 300], 50, 6
    col_off = NB.col_offsets(sizes)
    sp = np.concatenate([rng.integers(-2, V + 2, (B, L)) for L, V in zip(sizes, vocab)], 1)
    sp[0, col_off[1]:col_off[2]] = -1                       # a bag of padding only
    tabs = [rng.standard_normal((V, D)).astype(np.float32) for V in vocab]
    for mean in (False, True):
        z32, n32, bad = NB.pool_f32(tabs, sp, col_off, mean)
        z64, n64 = NB.pool64(tabs, sp, col_off, mean)
        np.testing.assert_array_equal(n32, n64)
        np.testing.assert_allclose(z32, z64, atol=1e-5)
        assert not z32[0, 1].any() and bad == sum(int((sp[:, col_off[k]:col_off[k + 1]] >= V).sum())
                                                  for k, V in enumerate(vocab))
        dz = rng.standard_normal((B, D))
        for k in range(len(sizes)):
            ids, rows = NB.bag_slices(sp, col_off, k, vocab[k], dz, mean)
            uid, summed = NB.bag_grad_rows(sp, col_off, k, vocab[k], dz, mean)
            ref = np.zeros((vocab[k], D))
            np.add.at(ref, ids, rows)
            np.testing.assert_array_equal(uid, np.unique(ids))
            np.testing.assert_allclose(summed, ref[uid], atol=1e-12)
