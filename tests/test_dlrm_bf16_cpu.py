"""DLRM(embedding_dtype=...) without a GPU: the per-table rounding seeds restated in numpy, and the keyword refused before
any table is made."""
import numpy as np
import pytest

from openrec_b200.tf2.recommenders import DLRM
from openrec_b200.tf2.recommenders.dlrm import table_rounding_seed


def _seeds_np(rounding_seed, n):
    """mix64(rounding_seed + k) (mod 2^64) for k < n, in numpy uint64 arithmetic (wrapping multiplication)."""
    z = np.uint64(rounding_seed) + np.arange(n, dtype=np.uint64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


@pytest.mark.parametrize("rounding_seed", (0, 1, 7, 2 ** 32 + 5, 2 ** 64 - 3))
def test_table_seeds_distinct_and_restated(rounding_seed):
    n = 4096
    with np.errstate(over="ignore"):
        ref = _seeds_np(rounding_seed, n)
    got = np.array([table_rounding_seed(rounding_seed, k) for k in range(n)], dtype=np.uint64)
    assert np.array_equal(got, ref)
    assert len(np.unique(got)) == n
    assert all(0 <= int(s) < 2 ** 64 for s in got[:8])


@pytest.mark.parametrize("dtype", ("float16", "bf16", "float64", None))
def test_unknown_embedding_dtype_refused(dtype):
    with pytest.raises(ValueError, match="embedding_dtype"):
        DLRM(m_spa=4, ln_emb=[10 ** 12] * 3, ln_bot=[8, 4], ln_top=[16, 1], embedding_dtype=dtype)
