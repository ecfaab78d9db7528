"""The far-table layout of tests/far_tables.py, checked on the host: planted rows lie in the far band, each alias is the
exact 32-bit truncation of both the element and the byte offset and lies inside the table, and no id-driven case names
a mid-band row (whose truncated offset would point before the table)."""
import numpy as np
import pytest

import far_tables as F

DIMS = (1, 4, 50, 128, 512)


@pytest.mark.parametrize("D", DIMS)
def test_rows_cover_every_band(D):
    rows = F.far_rows(D)
    assert rows * D >= F.FAR_END and (rows - 65) * D < F.FAR_END
    if D == 128:
        assert rows == 2 ** 25 + 2 ** 22 + 64
    assert F.band((rows - 1) * D) in ("far", "past")


@pytest.mark.parametrize("D", DIMS)
def test_planted_rows_and_aliases(D):
    m = F.Mix(D, seed=D)
    assert len(m.far) >= 20 and len(m.aliased) and len(m.guarded) and len(m.guard)
    lo, hi = F.far_band_rows(D)
    assert m.far[0] == lo and m.far[-1] == hi - 1
    for r in m.far:
        assert F.row_bands(r, D) == ("far", "far"), r
    for r in np.concatenate([m.far, [m.last]]):
        o = int(r) * D
        a = F.alias_elem(r, D)
        assert a == o - 2 ** 32 == (o % 2 ** 32)                     # the element offset truncated to 32 bits
        assert a == F.alias_byte_elem(r, D) == ((4 * o) % 2 ** 32) // 4   # and the byte offset
        assert 0 <= a and a + D <= m.rows * D and a + D <= 2 ** 31       # in the table's low band
        ar = F.alias_rows(r, D)
        assert ar[0] * D <= a and (ar[-1] + 1) * D >= a + D and len(ar) <= 2
        assert len(ar) == 1 or D & (D - 1)                           # a power-of-two D never straddles
    assert set(m.alias) == {a for r in m.aliased for a in F.alias_rows(r, D)}
    assert not set(m.guard) & set(m.valid)                          # guard rows are never named


@pytest.mark.parametrize("D", DIMS)
def test_no_id_names_a_mid_band_row(D):
    m = F.Mix(D, seed=D + 1)
    valid = m.ids[(m.ids >= 0) & (m.ids < m.rows)]
    assert set(valid) == set(m.valid)
    for r in m.valid:
        assert "mid" not in F.row_bands(r, D), r
    assert m.last in m.valid
    assert (m.ids < 0).any() and (m.ids >= m.rows).any()            # padding and bad ids
    assert len(m.ids) > len(np.unique(m.ids))                        # duplicates
    bad = m.ids[(m.ids < 0) | (m.ids >= m.rows)]
    assert set(bad) <= set(m.bad)
    if D >= 4:                                                       # int32 ids reach the far band from D = 4 up
        assert m.ids.max() <= 2 ** 31 - 1


@pytest.mark.parametrize("D", DIMS)
def test_band_samples(D):
    s = F.band_samples(D, 6, np.random.default_rng(D))
    for name, rows in s.items():
        assert len(rows) >= 2
        for r in rows:
            assert F.row_bands(r, D) == (name, name), (name, r)
