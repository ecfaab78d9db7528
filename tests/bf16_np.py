"""numpy restatement of bf16 table storage (include/orx.h, orx_table_bf16_t): the exact upcast, round to nearest even,
and the stochastic rounding of an update, H(sr_seed, step, t, row, col) included.  CPU only."""
import numpy as np

M64 = (1 << 64) - 1


def _mix64(z):
    z &= M64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & M64
    return z ^ (z >> 31)


def mix32(x):
    """orx_mix32 on a uint32 array (or scalar)."""
    x = np.asarray(x, np.uint64) & 0xffffffff
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7feb352d)) & np.uint64(0xffffffff)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846ca68b)) & np.uint64(0xffffffff)
    x ^= x >> np.uint64(16)
    return x


def table_key(seed, step, t):
    return _mix64(int(seed) ^ _mix64(2 * int(step) + int(t))) >> 32


def random_bits(seed, step, t, rows, cols):
    """r = H(...) >> 16 of elements (rows[i], cols[i]) (broadcast)."""
    rows = np.asarray(rows, np.int64).astype(np.uint64) & np.uint64(0xffffffff)
    cols = np.asarray(cols, np.int64).astype(np.uint64) & np.uint64(0xffffffff)
    rk = mix32(np.uint64(table_key(seed, step, t)) ^ rows)
    h = mix32((rk + cols * np.uint64(0x9e3779b9)) & np.uint64(0xffffffff))
    return (h >> np.uint64(16)).astype(np.uint32)


def _special(u):
    return (u & 0x7f800000) == 0x7f800000


def _special_bits(u):
    return (u >> 16) | np.where((u & 0x007fffff) != 0, 0x40, 0).astype(np.uint32)


def sr(x, seed, step, t, rows, cols):
    """uint16 bits of the stochastic rounding of float32 values x at (rows, cols) of table t."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = random_bits(seed, step, t, rows, cols).astype(np.uint64)
    out = ((u + r) >> np.uint64(16)).astype(np.uint32)
    u32 = u.astype(np.uint32)
    return np.where(_special(u32), _special_bits(u32), out).astype(np.uint16)


def rne(x):
    """uint16 bits of float32 x rounded to nearest even."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    out = ((u + 0x7fff + ((u >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)).astype(np.uint32)
    u32 = u.astype(np.uint32)
    return np.where(_special(u32), _special_bits(u32), out).astype(np.uint16)


def up(b):
    """float64 values of uint16 bf16 bits (the exact upcast)."""
    return (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def round_table(a):
    """float64 array of float32-valued a rounded to the nearest bf16 (a bf16 table's start)."""
    return up(rne(np.asarray(a, np.float32)))


def sr_interval(x64, tol, seed, step, t, rows, cols):
    """-> (lo, hi) uint16-upcast float64 bounds: the stochastic rounding is monotone in its float32 input for fixed
    random bits, so a float32 result in [x64 - tol, x64 + tol] rounds to a value in [sr(x64 - tol), sr(x64 + tol)].
    When both ends round alike, that one neighbour -- the one H selects -- is the only answer."""
    a = up(sr(np.float32(x64 - tol), seed, step, t, rows, cols))
    b = up(sr(np.float32(x64 + tol), seed, step, t, rows, cols))
    return np.minimum(a, b), np.maximum(a, b)
