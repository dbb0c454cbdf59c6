"""GPU: the TMA / tensor-core weight-streaming linear operator in isolation, against a plain fp32 torch matmul on the
same bf16-rounded weights (the op-level reference for a floating-point kernel)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(M, K, R, split_lo, ksplit, gain, accumulate, seed=0):
    from mvb200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(M, K, generator=g) * 0.05).to(torch.bfloat16).cuda()
    x = torch.randn(R, K, generator=g).cuda()
    gw = (1 + 0.1 * torch.randn(K, generator=g)).to(torch.bfloat16).cuda() if gain else None
    out0 = torch.randn(R, M, generator=g).cuda() if accumulate else torch.zeros(R, M).cuda()
    out = out0.clone()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.mvb_linear(W.data_ptr(), M, K, x.data_ptr(), K, R, gw.data_ptr() if gain else None, 1e-5,
                              int(split_lo), ksplit, out.data_ptr(), M, int(accumulate), st))
    xin = x
    if gain:
        xin = (x * torch.rsqrt((x * x).mean(-1, keepdim=True) + 1e-5)) * gw.float()
    ref = xin.double() @ W.double().t()
    if accumulate:
        ref = ref + out0.double()
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    return err


@pytest.mark.parametrize("M,K,R", [(256, 256, 2), (6144, 2048, 2), (2048, 5632, 16), (2562, 2048, 5), (1024, 512, 96)])
def test_linear_split_activations_match_fp32(M, K, R):
    for ksplit in (1, 0):
        err = _run(M, K, R, True, ksplit, gain=False, accumulate=False)
        print(f"M={M} K={K} R={R} ksplit={'1' if ksplit else 'auto'} hi+lo rel err {err:.2e}")
        assert err < 2e-5


def test_linear_bf16_activations_only():
    err = _run(2048, 2048, 4, False, 0, gain=False, accumulate=False)
    print(f"single bf16 term rel err {err:.2e}")
    assert err < 1e-2  # one bf16 term: ~2^-9 per element, random-sign accumulation


def test_linear_rmsnorm_prologue_and_residual_epilogue():
    assert _run(2048, 2048, 2, True, 0, gain=True, accumulate=True) < 2e-5
    assert _run(5632, 2048, 8, True, 1, gain=True, accumulate=False) < 2e-5
