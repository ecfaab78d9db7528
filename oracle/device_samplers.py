"""NumPy restatement of liborx's counter-based draws -- TEST INFRASTRUCTURE, NOT PRODUCT.

Restates, bit for bit, the draw rules of ``openrec_b200/csrc/orx_sampler.cu`` (the three device samplers) and of
``k_fill_uniform`` in ``openrec_b200/csrc/orx_misc.cu``, so a test can compare every sample a kernel emits with an
independent computation instead of with statistical properties.  Both files use splitmix64 (Steele, Lea and Flood,
"Fast splittable pseudorandom number generators", OOPSLA 2014) as a stateless mixer:

    smix64(x)        = splitmix64's output function applied to x + 0x9E3779B97F4A7C15
    srand3(s, a, b)  = smix64(s ^ smix64((a << 24) ^ b))            (64-bit wrap-around arithmetic)

A sampler's inputs are given as numpy arrays with the fields of ``orx_sampler_t`` (include/orx.h): ``rec_user``,
``rec_item`` [n], ``perm_cur``, ``perm_next`` [n], ``cursor``, ``csr_off`` [U + 1], ``csr_items``, ``total_users``,
``total_items``.
"""
from __future__ import annotations

import numpy as np

_U = np.uint64
GIVE_UP = 1000000          # pairwise / stratified negatives: the last attempt is GIVE_UP + 1
DISTINCT_GIVE_UP = 100000  # per-positive: a duplicate candidate is kept once this many draws were made
COIN = 0xC01F              # the stratified coin's attempt number


def smix64(x):
    """splitmix64's mix of x + golden gamma, elementwise on uint64 (wraps like the device's uint64_t)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + _U(0x9E3779B97F4A7C15)
        x = (x ^ (x >> _U(30))) * _U(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> _U(27))) * _U(0x94D049BB133111EB)
        return x ^ (x >> _U(31))


def srand3(seed, a, b):
    """The draw of (seed, stream position a, attempt b); a and b broadcast."""
    a = np.asarray(a, dtype=np.int64).astype(np.uint64)
    b = np.asarray(b, dtype=np.int64).astype(np.uint64)
    return smix64(_U(seed) ^ smix64((a << _U(24)) ^ b))


def fill_uniform_u(seed, start, stop):
    """u_i = (splitmix64(seed * 0xD1342543DE82EF95 + i) >> 40) * 2^-24 as float32, i in [start, stop): the [0, 1)
    variate of ``k_fill_uniform`` (exact in float32: a 24-bit integer times a power of two)."""
    i = np.arange(start, stop, dtype=np.uint64)
    with np.errstate(over="ignore"):
        r = smix64(_U(seed) * _U(0xD1342543DE82EF95) + i)
    return ((r >> _U(40)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def record(sd, k):
    """Index of the k-th record consumed from the cursor on: the tail of perm_cur, then perm_next (k array)."""
    k = np.asarray(k, dtype=np.int64)
    n = len(sd["rec_user"])
    left = n - sd["cursor"]
    cur = sd["perm_cur"][np.minimum(sd["cursor"] + k, n - 1)]
    return np.where(k < left, cur, sd["perm_next"][np.maximum(k - left, 0) % n])


def _positives(sd, u):
    return sd["csr_items"][sd["csr_off"][u]:sd["csr_off"][u + 1]]


def _first_unobserved(draw, observed, first):
    """The first attempt a >= first whose draw(a) is not observed, else the draw of attempt GIVE_UP + 1 (the device
    loops break after that attempt whatever it drew).  draw(attempts) -> tuple of candidate arrays,
    observed(tuple) -> bool array.  -> tuple of the chosen candidate's fields."""
    a, width = first, 8
    while a <= GIVE_UP + 1:
        att = np.arange(a, min(a + width, GIVE_UP + 2), dtype=np.int64)
        c = draw(att)
        free = ~observed(c)
        if free.any():
            return tuple(x[int(np.argmax(free))] for x in c)
        a, width = a + len(att), min(width * 8, 1 << 20)
    return tuple(x[-1] for x in c)                      # attempt GIVE_UP + 1


def sample_pairwise(sd, seed, stream_pos, B):
    """k_sample_pairwise: slot b takes record b from the cursor and the first item % I not among the user's positives
    over attempts 0, 1, ... (srand3(seed, stream_pos + b, attempt)); a user positive on every item ends on attempt
    GIVE_UP + 1.  -> (uid, pid, nid) int32."""
    I = sd["total_items"]
    r = record(sd, np.arange(B))
    uid, pid = sd["rec_user"][r], sd["rec_item"][r]
    nid = (srand3(seed, stream_pos + np.arange(B), 0) % _U(I)).astype(np.int32)   # every slot's first draw at once
    keys = sd["rec_user"].astype(np.int64) * I + sd["rec_item"]
    for b in np.flatnonzero(np.isin(uid.astype(np.int64) * I + nid, keys)):
        pos = _positives(sd, uid[b])
        if len(pos) == I:                       # every draw is rejected: only the last attempt matters
            nid[b] = srand3(seed, stream_pos + b, GIVE_UP + 1) % _U(I)
            continue
        nid[b], = _first_unobserved(lambda att: ((srand3(seed, stream_pos + b, att) % _U(I)).astype(np.int64),),
                                    lambda c: np.isin(c[0], pos), 1)
    return uid.astype(np.int32), pid.astype(np.int32), nid


def sample_stratified(sd, seed, stream_pos, B, pos_ratio):
    """k_sample_stratified: slot b is a positive iff (x >> 11) * 2^-53 <= pos_ratio (the float32 ratio promoted to
    double), x = srand3(seed, stream_pos + b, COIN); the positives take consecutive records in slot order; a negative
    is (x >> 32) % U, (x & 0xffffffff) % I of the first unobserved attempt >= 1.  -> (uid, iid, label, n_pos)."""
    U, I = sd["total_users"], sd["total_items"]
    slots = stream_pos + np.arange(B, dtype=np.int64)
    coin = (srand3(seed, slots, COIN) >> _U(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    pos = coin <= np.float64(np.float32(pos_ratio))
    r = record(sd, np.cumsum(pos) - pos)               # exclusive scan of the coins
    uid = np.where(pos, sd["rec_user"][r], 0).astype(np.int32)
    iid = np.where(pos, sd["rec_item"][r], 0).astype(np.int32)
    full = len(sd["rec_user"]) == U * I                # every pair observed: every draw is rejected
    keys = sd["rec_user"].astype(np.int64) * I + sd["rec_item"]

    def draw(b):
        def f(att):
            x = srand3(seed, stream_pos + b, att)
            return ((x >> _U(32)) % _U(U)).astype(np.int64), ((x & _U(0xFFFFFFFF)) % _U(I)).astype(np.int64)
        return f

    def observed(c):
        return np.isin(c[0] * I + c[1], keys)

    neg = np.flatnonzero(~pos)
    x = srand3(seed, stream_pos + neg, GIVE_UP + 1 if full else 1)     # every slot's first draw at once
    u, i = ((x >> _U(32)) % _U(U)).astype(np.int64), ((x & _U(0xFFFFFFFF)) % _U(I)).astype(np.int64)
    uid[neg], iid[neg] = u, i
    for b in ([] if full else neg[observed((u, i))]):  # the rest redraw from attempt 2 on
        uid[b], iid[b] = _first_unobserved(draw(b), observed, 2)
    return uid, iid, pos.astype(np.float32), int(pos.sum())


def per_positive_group(seed, grp, quota, I, positive):
    """The negatives of group grp: quota + 1 candidates % I, distinct (a duplicate is redrawn until DISTINCT_GIVE_UP
    draws were made), in draw order, the positive removed, the first `quota` kept."""
    cand, attempt, draws = [], 0, np.empty(0, dtype=np.int64)
    while len(cand) < quota + 1:
        if attempt == len(draws):                      # draws are made ahead in blocks; only their order matters
            more = srand3(seed, grp, np.arange(attempt, attempt + 4 * quota + 16)) % _U(I)
            draws = np.concatenate([draws, more.astype(np.int64)])
        c = int(draws[attempt])
        attempt += 1
        if c in cand and attempt < DISTINCT_GIVE_UP:
            continue
        cand.append(c)
    return [c for c in cand if c != positive][:quota]


def sample_per_positive(sd, seed, stream_pos, B, quota):
    """k_sample_per_positive: stream position s = stream_pos + b lies in group s // (quota + 1); member 0 is the group's
    record (label 1), member m >= 1 its m-th negative (label 0).  The cursor points at the record of stream_pos's
    group.  -> (uid, iid, label)."""
    g = quota + 1
    s = stream_pos + np.arange(B, dtype=np.int64)
    grp, m = s // g, s % g
    r = record(sd, grp - stream_pos // g)
    uid, iid = sd["rec_user"][r].astype(np.int32), sd["rec_item"][r].astype(np.int32)
    negs = {}
    for b in np.flatnonzero(m > 0):
        k = int(grp[b])
        if k not in negs:
            negs[k] = per_positive_group(seed, k, quota, sd["total_items"], int(iid[b]))
        if m[b] <= len(negs[k]):                       # fewer than m kept (duplicates after the give-up): the positive
            iid[b] = negs[k][m[b] - 1]
    return uid, iid, (m == 0).astype(np.float32)
