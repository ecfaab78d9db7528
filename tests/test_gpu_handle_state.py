"""GPU: what liborx keeps per handle stays with the handle -- split-K partials of two handles on two streams do not mix,
a destroyed handle returns its scratch and a new one starts clean, and kernels opted in to large shared memory run on
every device of the process."""
import numpy as np
import pytest
import torch

from openrec_b200 import _lib as L
from openrec_b200 import native as N

pytestmark = pytest.mark.gpu

TMA, SIMT = L.ORX_VARIANT_GEMM_TMA, L.ORX_VARIANT_GEMM_SIMT


def _cdiv(a, b):
    return -(-a // b)


@pytest.fixture
def handles():
    """Fresh handles (not the per-device engines other tests share), destroyed at the end of the test."""
    made = []

    def make(device=0):
        made.append(N.Engine(device))
        return made[-1]

    yield make
    torch.cuda.synchronize()
    for e in made:
        e.close()


def _layer_inputs(B, inn, out, seed, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(device)
    return r(B, inn), r(B, out), r(inn, out) * 0.3, r(B, out)   # x, y, w, dy


def _layer_bwd(eng, x, y, w, dy):
    """orx_mlp_layer_bwd with relu on a copy of dy (it is overwritten with dz) -> (dw, db, dx), enqueued on the current
    stream."""
    B, inn = x.shape
    out = w.shape[1]
    dz = dy.clone()
    dw, db, dx = torch.empty(inn, out, device=x.device), torch.empty(out, device=x.device), torch.empty(B, inn, device=x.device)
    eng.mlp_bwd(x, y, w, 1, dz, dx, dw, db)
    return dw, db, dx


# orx_mlp_layer_bwd shapes of test_gpu_dlrm.py whose column sum splits (B >= 4096), with the kernel of the split-K dw
SPLIT_BWD = [(6000, 300, 200, TMA), (8192, 13, 512, SIMT), (4096, 512, 256, TMA)]


@pytest.mark.parametrize("B,inn,out,variant", SPLIT_BWD)
def test_two_handles_two_streams_splitk(handles, B, inn, out, variant):
    """Two handles run the same split-K layer backward on different inputs, on two streams released by one event: each
    gets bit for bit what it gets running alone (the split-K reduction is deterministic)."""
    ea, eb = handles(), handles()
    ins = [_layer_inputs(B, inn, out, seed) for seed in (1, 2)]
    ea.debug_dispatch_log()
    alone = [_layer_bwd(e, *i) for e, i in zip((ea, eb), ins)]
    torch.cuda.synchronize()
    rec = ea.debug_dispatch_log()
    assert any(r.op == L.ORX_OP_GEMM and r.variant == variant and r.s > 1 for r in rec), rec
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda._sleep(20_000_000)                 # both calls are enqueued before either can start
    go = torch.cuda.Event()
    go.record()
    both = []
    for e, i, s in zip((ea, eb), ins, streams):
        s.wait_event(go)
        with torch.cuda.stream(s):
            both.append(_layer_bwd(e, *i))
    torch.cuda.synchronize()
    for k, (got, ref) in enumerate(zip(both, alone)):
        for name, g, r in zip(("dw", "db", "dx"), got, ref):
            assert torch.equal(g, r), f"handle {k}: {name} differs from the handle running alone"


def test_destroy_then_new_handle_splitk(handles):
    """A handle that ran a split-K layer is destroyed; a new handle then runs a split-K forward whose last split has no
    k-block, three times over, and gets the correct result each time."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B, out = 128, 128                               # one tile
    for nkb in range(32, 1 << 16):                  # the first K whose last split is empty (as test_gpu_dlrm.py)
        S = max(1, min(2 * sms, nkb // 8))
        if S > 1 and (S - 1) * _cdiv(nkb, S) >= nkb:
            break
    inn = 16 * nkb - 8
    g = torch.Generator().manual_seed(81)
    for _ in range(3):
        old = N.Engine(0)
        try:                                        # leaves non-zero partials behind in the memory it frees
            big = torch.randn(B, inn + 512, generator=g).cuda()
            old.mlp_fwd(big, torch.randn(inn + 512, out, generator=g).cuda(), None, 0, torch.empty(B, out, device="cuda"))
            torch.cuda.synchronize()
        finally:
            old.close()
        eng = handles()
        x, w = torch.randn(B, inn, generator=g).cuda(), torch.randn(inn, out, generator=g).cuda()
        y = torch.empty(B, out, device="cuda")
        eng.debug_dispatch_log()
        eng.mlp_fwd(x, w, None, 0, y)
        assert eng.debug_dispatch_log() == [N.Dispatch(L.ORX_OP_GEMM, TMA, 0, 0, B, out, inn, S)]
        x64, w64 = x.cpu().double().numpy(), w.cpu().double().numpy()
        e = np.max(np.abs(y.cpu().double().numpy() - x64 @ w64) / (np.abs(x64) @ np.abs(w64)))
        assert e <= 2.0 ** -18, e                   # the k_gemm_tma error bar of test_gpu_dlrm.py


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_devices_one_process(handles):
    """The TMA GEMM and the warp interaction kernels (dynamic shared memory above 48 KB) on device 0, then on device 1:
    both succeed with bit-identical outputs."""
    B, inn, out = 512, 256, 128
    F, D = 27, 128
    g = torch.Generator().manual_seed(5)
    x, w, b = torch.randn(B, inn, generator=g), torch.randn(inn, out, generator=g), torch.randn(out, generator=g)
    emb, dense = torch.randn(B, F - 1, D, generator=g), torch.randn(B, D, generator=g)
    P = F * (F - 1) // 2
    dout, ddense0 = torch.randn(B, P, generator=g), torch.randn(B, D, generator=g)
    res = []
    for d in (0, 1):
        eng = handles(d)
        dev = lambda t: t.to(f"cuda:{d}")
        with torch.cuda.device(d):
            y = torch.empty(B, out, device=f"cuda:{d}")
            eng.mlp_fwd(dev(x), dev(w), dev(b), 1, y)
            pairs = torch.empty(B, P, device=f"cuda:{d}")
            eng.interact_fwd(dev(emb), dev(dense), False, 1, pairs)
            demb, ddense = torch.empty(B, F - 1, D, device=f"cuda:{d}"), dev(ddense0)
            eng.interact_bwd(dev(emb), dev(dense), dev(dout), False, 1, demb, ddense)
            torch.cuda.synchronize(d)
            assert eng.debug_dispatch_log() == [
                N.Dispatch(L.ORX_OP_GEMM, TMA, 0, 0, B, out, inn, 1),
                N.Dispatch(L.ORX_OP_INTERACT_FWD, L.ORX_VARIANT_INTERACT_WARP, 0, 0, B, F, D, 1),
                N.Dispatch(L.ORX_OP_INTERACT_BWD, L.ORX_VARIANT_INTERACT_WARP, 0, 0, B, F, D, 1)]
        res.append([t.cpu() for t in (y, pairs, demb, ddense)])
    for name, a, c in zip(("y", "interaction", "demb", "ddense"), *res):
        assert torch.equal(a, c), f"{name}: device 1 differs from device 0"
