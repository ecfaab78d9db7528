"""CPU checks of oracle/device_samplers.py, the numpy restatement the GPU sampler and fill tests compare against."""
import numpy as np

from oracle import device_samplers as S


def test_smix64_known_answer():
    """splitmix64 from state 0 (Vigna's reference splitmix64.c): the k-th output is smix64(k * golden gamma)."""
    assert int(S.smix64(0)) == 0xE220A8397B1DCDAF
    gamma = 0x9E3779B97F4A7C15
    got = S.smix64(np.array([(k * gamma) % 2 ** 64 for k in range(1, 4)], dtype=np.uint64))
    assert [int(x) for x in got] == [0x6E789E6AA1B965F4, 0x06C45D188009454F, 0xF88BB8A8724C81EC]


def test_srand3_and_fill_stream_match_python_ints():
    """The uint64 numpy arithmetic wraps exactly like Python integers reduced mod 2^64."""
    M = 2 ** 64 - 1

    def sm(x):
        x = (x + 0x9E3779B97F4A7C15) & M
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M
        return x ^ (x >> 31)

    for seed, a, b in ((0, 0, 0), (2 ** 64 - 1, 10 ** 12 + 7, 1000001), (12345, 2 ** 40 + 3, 0xC01F)):
        assert int(S.srand3(seed, a, b)) == sm(seed ^ sm(((a << 24) & M) ^ b))
    u = S.fill_uniform_u(2 ** 63 + 5, 7, 10)
    want = [(sm((((2 ** 63 + 5) * 0xD1342543DE82EF95) + i) & M) >> 40) / 2 ** 24 for i in range(7, 10)]
    assert u.dtype == np.float32 and u.tolist() == want


def _store(U, I, pairs, rng, cursor):
    users, items = pairs[:, 0].astype(np.int32), pairs[:, 1].astype(np.int32)
    order = np.lexsort((items, users))
    off = np.zeros(U + 1, dtype=np.int64)
    np.cumsum(np.bincount(users, minlength=U), out=off[1:])
    n = len(users)
    return dict(rec_user=users, rec_item=items, perm_cur=rng.permutation(n), perm_next=rng.permutation(n),
                cursor=cursor, csr_off=off, csr_items=items[order], total_users=U, total_items=I)


def test_restated_samplers_keep_their_invariants():
    """Records in permutation order across the epoch boundary, negatives never observed, per-positive negatives
    distinct and never the positive, stratified positives consecutive records."""
    rng = np.random.default_rng(0)
    U, I = 20, 40
    pairs = np.unique(np.stack([rng.integers(0, U, 300), rng.integers(0, I, 300)], 1), axis=0)
    sd = _store(U, I, pairs, rng, cursor=len(pairs) - 5)
    n = len(pairs)
    obs = set(map(tuple, pairs.tolist()))
    want = np.concatenate([sd["perm_cur"][n - 5:], sd["perm_next"][:10]])
    assert np.array_equal(S.record(sd, np.arange(15)), want)
    uid, pid, nid = S.sample_pairwise(sd, 9, 1000, 15)
    assert np.array_equal(uid, pairs[want, 0]) and np.array_equal(pid, pairs[want, 1])
    assert not any((u, i) in obs for u, i in zip(uid.tolist(), nid.tolist()))
    uid, iid, lab, npos = S.sample_stratified(sd, 9, 1000, 200, 0.3)
    assert npos == int(lab.sum()) and 0 < npos < 200
    assert np.array_equal(np.stack([uid, iid], 1)[lab == 1], pairs[S.record(sd, np.arange(npos))])
    assert all(((u, i) in obs) == (l == 1) for u, i, l in zip(uid.tolist(), iid.tolist(), lab.tolist()))
    negs = S.per_positive_group(9, 77, I - 1, I, 5)
    assert sorted(negs) == [i for i in range(I) if i != 5]
    uid, iid, lab = S.sample_per_positive(sd, 9, 3 * 5 + 2, 13, 4)     # starts inside group 3: members 2, 3, 4
    assert lab.tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0]
