"""CPU: the numpy restatement of bf16 table rounding (tests/bf16_np.py) against first principles, and the constructor
checks of the bf16 models."""
import numpy as np
import pytest

import bf16_np as H


def test_rne_matches_numpy_float32_to_bf16():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(1 << 16) * 0.1).astype(np.float32)
    b = H.up(H.rne(x))
    lo = H.up((x.view(np.uint32) >> 16).astype(np.uint16))     # truncation toward zero
    ulp = np.abs(H.up(((x.view(np.uint32) >> 16) + 1).astype(np.uint16)) - lo)
    assert np.all(np.abs(b - x) <= ulp / 2)


def test_sr_keeps_representable_values_and_specials():
    rng = np.random.default_rng(1)
    x = H.up(H.rne(rng.standard_normal(4096).astype(np.float32))).astype(np.float32)
    rows, cols = np.arange(4096) // 64, np.arange(4096) % 64
    assert np.array_equal(H.up(H.sr(x, 3, 5, 1, rows, cols)), x.astype(np.float64))
    sp = np.array([np.inf, -np.inf, 0.0, -0.0], np.float32)
    assert np.array_equal(H.sr(sp, 3, 5, 0, 0, np.arange(4)), (sp.view(np.uint32) >> 16).astype(np.uint16))
    assert np.isnan(H.up(H.sr(np.array([np.nan], np.float32), 3, 5, 0, 0, 0))).all()
    tiny = np.frombuffer(np.uint32(0x00000001).tobytes(), np.float32)   # smallest subnormal: up with P ~ 2^-16
    assert H.up(H.sr(tiny, 3, 5, 0, 0, 0))[0] in (0.0, H.up(np.uint16(1)))


def test_sr_picks_a_neighbour_with_the_right_odds():
    x = np.float32(0.0501)
    lo = H.up((np.array([x]).view(np.uint32) >> 16).astype(np.uint16))[0]
    hi = H.up(((np.array([x]).view(np.uint32) >> 16) + 1).astype(np.uint16))[0]
    p = (float(x) - lo) / (hi - lo)
    n = 1 << 14
    v = H.up(H.sr(np.full(n, x), 42, 7, 0, np.arange(n) // 128, np.arange(n) % 128))
    assert set(np.unique(v)) <= {lo, hi}
    assert abs((v == hi).mean() - p) < 4 * np.sqrt(p * (1 - p) / n)


def test_bits_depend_on_every_key():
    base = H.random_bits(1, 2, 0, np.arange(1024), 5)
    for args in ((2, 2, 0), (1, 3, 0), (1, 2, 1)):
        assert (H.random_bits(*args, np.arange(1024), 5) != base).mean() > 0.99
    assert (H.random_bits(1, 2, 0, np.arange(1024), 6) != base).mean() > 0.99
    assert (H.random_bits(1, 2, 0, np.arange(1, 1025), 5) != base).mean() > 0.99


def test_embedding_dtype_is_checked():
    from openrec_b200.tf2.recommenders import BPR, UCML
    for cls in (BPR, UCML):
        with pytest.raises(ValueError, match="embedding_dtype"):
            cls(8, 8, 10, 10, embedding_dtype="float16")
