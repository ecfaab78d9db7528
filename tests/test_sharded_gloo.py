"""CPU, world_size 2 and 3 over gloo: the row-sharded step's host logic (owner bucketing, the four
all-to-all exchanges, slot permutations, cross-rank duplicate handling) reproduces the single-process
oracle step on the same global batch.  Arithmetic = oracle via tests/fake_engine.py; the CUDA kernels
behind the same calls are checked in tests/test_gpu_kernels.py / test_gpu_sharded.py."""
import os

import numpy as np
import pytest
from _ranks import run_ranks

from oracle import openrec_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,kind,opt_kind", [(2, 0, 1), (3, 0, 0), (2, 1, 1), (2, 0, 2)])
def test_sharded_step_equals_single_process(tmp_path, world, kind, opt_kind):
    out = str(tmp_path / "res.npz")
    for rc, o in run_ranks(world, [os.path.join(ROOT, "tests", "_sharded_worker.py"), out, str(kind), str(opt_kind)],
                           f"sharded_gloo {kind} {opt_kind}"):
        assert rc == 0, o
    got = np.load(out)
    rng = np.random.default_rng(99)
    U, I, D, B = 61, 83, 16, 40
    sc = 0.05 if kind == 0 else 0.4
    user, item, bias = (rng.uniform(-sc, sc, s).astype(np.float32).astype(np.float64) for s in ((U, D), (I, D), (I, 1)))
    if opt_kind == 0:
        st = {k: (None, None) for k in ("user", "item", "bias")}
    elif opt_kind == 1:
        st = {k: (np.full_like(v, 0.1), None) for k, v in zip(("user", "item", "bias"), (user, item, bias))}
    else:
        st = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in zip(("user", "item", "bias"), (user, item, bias))}
    for step in range(3):
        ids = [rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
        loss, l2 = O.pairwise_train_step("bpr" if kind == 0 else "ucml", user, item, bias, *ids, opt_kind, st,
                                         step + 1, 0.05, margin=0.5)
        np.testing.assert_allclose(got["losses"][step], [loss, l2], rtol=1e-5)
    for name, ref in (("user", user), ("item", item), ("bias", bias)):
        np.testing.assert_allclose(got[name], ref, atol=1e-6)
