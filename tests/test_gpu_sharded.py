"""GPU, >= 2 devices: the row-sharded step on the real kernels over NCCL equals the single-process oracle
step on the same global batch (cross-rank duplicates included)."""
import os

import numpy as np
import pytest
import torch
from _ranks import run_ranks

from oracle import openrec_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# NCCL all-to-all form / home-routed peer-store mailboxes (the 1-GPU form of the latter: test_gpu_shard_loopback.py)
@pytest.mark.parametrize("mode", ["gpu", "home", "home_next"])
@pytest.mark.parametrize("kind,opt_kind", [(0, 1), (0, 0), (1, 1)])
def test_sharded_step_on_gpus(tmp_path, kind, opt_kind, mode):
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    out = str(tmp_path / "res.npz")
    for rc, o in run_ranks(world, [os.path.join(ROOT, "tests", "_sharded_worker.py"), out, str(kind), str(opt_kind),
                                   mode], f"gpu_sharded {kind} {opt_kind} {mode}", timeout=600):
        assert rc == 0, o
    got = np.load(out)
    rng = np.random.default_rng(99)
    U, I, D, B = 1501, 2003, 128, 1024
    sc = 0.05 if kind == 0 else 0.4
    user, item, bias = (rng.uniform(-sc, sc, s).astype(np.float32).astype(np.float64) for s in ((U, D), (I, D), (I, 1)))
    st = {k: ((np.full_like(v, 0.1), None) if opt_kind == 1 else (None, None))
          for k, v in zip(("user", "item", "bias"), (user, item, bias))}
    for step in range(5 if mode == "home_next" else 3):
        ids = [rng.integers(0, n, B * world).astype(np.int32) for n in (U, I, I)]
        loss, l2 = O.pairwise_train_step("bpr" if kind == 0 else "ucml", user, item, bias, *ids, opt_kind, st,
                                         step + 1, 0.05, margin=0.5)
        np.testing.assert_allclose(got["losses"][step], [loss, l2], rtol=3e-5)
    tol = 1e-5 if kind == 0 else 2e-4   # ucml: a float32 hinge flip moves a row by ~lr; none expected at this seed
    for name, ref in (("user", user), ("item", item), ("bias", bias)):
        np.testing.assert_allclose(got[name], ref, atol=tol)
