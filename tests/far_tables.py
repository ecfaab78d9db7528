"""TEST INFRASTRUCTURE: the layout of a "far" table, a float32 [rows, D] table past 2^32 elements, built so that a
32-bit truncation of a row address shows up as a wrong value at a known row rather than as an out-of-bounds access.

Element offsets fall in three bands: low [0, 2^31), mid [2^31, 2^32) and far [2^32, 2^32 + 2^29).  A table has
rows(D) = ceil((2^32 + 2^29) / D) + 64 rows (2^25 + 2^22 + 64 at D = 128: 19.3 GB), so it covers all three.

For a row r whose element offset o = r * D lies at or above 2^32 (every far-band row, and the 64 rows past it), a
kernel that truncates o to 32 bits reads o - 2^32, and one that truncates the byte offset 4 * o reads byte
(4 * o) mod 2^32 = 4 * (o - 2^32) as well, since o - 2^32 < 2^30.  Both land on elements [o - 2^32, o - 2^32 + D) of
the low band: the row's alias, inside the table.  At D not a power of two the alias straddles two rows.

A mid-band row has no such alias (its truncated offset as an int32 is negative), so id-driven kernels (gathers,
applies, steps, censors, the score kernels' item ids) are only ever handed low rows and rows at or above 2^32 / D;
only the full-table sweeps (k_adam_sweep, orx_fill_uniform, orx_rows_scale) reach the mid band.

``Mix`` is the id set of one case: planted far rows (overwritten with values from a range disjoint from the
background), half of them with their alias rows named as ids too (so a wrap makes two lookups of one batch address the
same row), the other half with their alias rows left out (the guard rows, which must stay bit-identical), plain low
rows, duplicates, padding (-1), bad ids (= rows, and 2^31 - 1) and the last valid row.
"""
from __future__ import annotations

import numpy as np

LOW_END = 1 << 31
MID_END = 1 << 32
FAR_END = (1 << 32) + (1 << 29)
BANDS = ("low", "mid", "far", "past")


def far_rows(D):
    """Rows of the far table of width D: the far band covered, plus 64 rows past it."""
    return -(-FAR_END // D) + 64


def band(elem):
    """Band name of an element offset ("past": at or above 2^32 + 2^29, the rows after the far band)."""
    e = int(elem)
    return "low" if e < LOW_END else "mid" if e < MID_END else "far" if e < FAR_END else "past"


def row_bands(r, D):
    """The bands of the first and last element of row r."""
    return band(int(r) * D), band(int(r) * D + D - 1)


def alias_elem(r, D):
    """First element of row r's alias: its element offset truncated to 32 bits (r * D >= 2^32)."""
    o = int(r) * D
    assert o >= MID_END, (r, D)
    return o & 0xFFFFFFFF


def alias_byte_elem(r, D):
    """The element the row's byte offset truncated to 32 bits points at."""
    return ((int(r) * D * 4) & 0xFFFFFFFF) // 4


def alias_rows(r, D):
    """The rows holding row r's alias elements (one, or two when the alias straddles a row boundary)."""
    a = alias_elem(r, D)
    return list(range(a // D, (a + D - 1) // D + 1))


def far_band_rows(D):
    """[lo, hi): the rows lying wholly in the far band."""
    return -(-MID_END // D), FAR_END // D


def low_band_rows(D):
    """[0, hi): the rows lying wholly in the low band."""
    return 0, LOW_END // D


def band_samples(D, n, rng):
    """n rows of each band (low, mid, far, past) that lie wholly inside it, the band edges included: for checks of the
    full-table sweeps."""
    rows = far_rows(D)
    edges = {"low": (0, LOW_END // D), "mid": (-(-LOW_END // D), MID_END // D), "far": far_band_rows(D),
             "past": (-(-FAR_END // D), rows)}
    out = {}
    for name, (lo, hi) in edges.items():
        pick = {lo, hi - 1} | set(rng.integers(lo, hi, max(n - 2, 0)).tolist())
        out[name] = np.array(sorted(pick), np.int64)
    return out


class Mix:
    """The ids of one id-driven case on the far table of width D (see the module docstring).  Attributes (int64 numpy):
    far        planted far-band rows (sorted), far[0] the first far-band row, far[-1] the last
    aliased    the planted rows whose alias rows are named as ids; guarded: the others
    alias      the alias rows of `aliased` (named); guard: the alias rows of `guarded` (never named)
    low        plain low rows (named)
    last       rows - 1
    valid      every named valid row once (sorted)
    bad        padding and out-of-range ids used
    ids        the id list: every valid row, duplicates of some, and the bad ids, shuffled (int64)"""

    def __init__(self, D, seed=0, n_far=24, n_low=40, n_dup=48):
        rng = np.random.default_rng(seed)
        self.D, self.rows = D, far_rows(D)
        lo, hi = far_band_rows(D)
        far = {lo, hi - 1} | set(rng.integers(lo, hi, n_far - 2).tolist())
        self.far = np.array(sorted(far), np.int64)
        order = rng.permutation(len(self.far))
        self.aliased = np.sort(self.far[order[: len(order) // 2]])
        self.guarded = np.sort(self.far[order[len(order) // 2:]])
        self.alias = np.array(sorted({a for r in self.aliased for a in alias_rows(r, D)}), np.int64)
        guard = {a for r in self.guarded for a in alias_rows(r, D)} - set(self.alias.tolist())
        self.guard = np.array(sorted(guard), np.int64)
        self.last = self.rows - 1
        low = set()
        while len(low) < n_low:
            r = int(rng.integers(0, low_band_rows(D)[1]))
            if r not in guard:
                low.add(r)
        self.low = np.array(sorted(low | ({0} - guard)), np.int64)
        self.valid = np.unique(np.concatenate([self.far, self.alias, self.low, [self.last]]))
        self.bad = np.array([-1, -1, self.rows] + ([2 ** 31 - 1] if self.rows < 2 ** 31 - 1 else []), np.int64)
        dup = rng.choice(np.concatenate([self.far, self.alias, self.low]), n_dup)
        ids = np.concatenate([self.valid, dup, self.far[:3], self.bad])
        self.ids = ids[rng.permutation(len(ids))]

    @property
    def named_valid(self):
        """Valid ids of self.ids (with repeats), in order."""
        return self.ids[(self.ids >= 0) & (self.ids < self.rows)]
