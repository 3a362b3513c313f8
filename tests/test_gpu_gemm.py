"""wgmma GEMM (through the C ABI test hook) against a plain PyTorch fp32 reference of the same op on the same
bf16-rounded operands.  Tolerance: fp32 accumulation-order noise only (rel-L2 <= 2e-5, max-abs <= 2e-3*sqrt(K/64))."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(lib, M, N, K, a_mn=0, b_mn=0, BN=0, cg=1, bias=False, residual=False, act=0, stats=False, ln=False,
         out_bf16=False, seed=0):
    from smd_b200 import lib as L
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
    B = (torch.randn(N, K, generator=g) * 0.5).to(torch.bfloat16)
    ref = A.float() @ B.float().t()
    Ad = (A.t().contiguous() if a_mn else A).cuda()
    Bd = (B.t().contiguous() if b_mn else B).cuda()
    bias_t = torch.randn(N, generator=g).cuda() if bias else None
    res_t = torch.randn(M, N, generator=g).cuda() if residual else None
    if bias:
        ref = ref + bias_t.cpu()
    if residual:
        ref = ref + res_t.cpu()
    out32 = torch.full((M, N), float("nan"), device="cuda")
    out16 = torch.zeros((M, N), dtype=torch.bfloat16, device="cuda") if (out_bf16 or ln) else None
    st = torch.zeros((M, 2), device="cuda") if stats else None
    gam = (1 + 0.1 * torch.randn(N, generator=g)).cuda() if ln else None
    bet = (0.1 * torch.randn(N, generator=g)).cuda() if ln else None
    p = lambda t: None if t is None else t.data_ptr()
    L.check(lib.smd_gemm_bf16(Ad.data_ptr(), Bd.data_ptr(), M, N, K, a_mn, b_mn, BN, cg, p(bias_t), p(res_t), act,
                              out32.data_ptr(), p(out16), p(st), p(gam), p(bet),
                              torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    got = out32.cpu()
    err = float((got - ref).norm() / ref.norm())
    assert not torch.isnan(got).any(), "unwritten / NaN outputs"
    assert err < 2e-5, f"rel-L2 {err:.3e}"
    assert float((got - ref).abs().max()) < 2e-3 * math.sqrt(K / 64)
    if stats:
        s = st.cpu()
        assert torch.allclose(s[:, 0], ref.sum(1), rtol=1e-4, atol=1e-2)
        assert torch.allclose(s[:, 1], (ref * ref).sum(1), rtol=1e-4, atol=1e-2)
    if ln:
        mu = ref.mean(1, keepdim=True)
        var = (ref * ref).mean(1, keepdim=True) - mu * mu
        expect = (ref - mu) * torch.rsqrt(var + 1e-6) * gam.cpu() + bet.cpu()
        assert float((out16.float().cpu() - expect).abs().max()) < 0.05
    elif out_bf16:
        e = ref
        if act == 1:
            e = torch.nn.functional.gelu(ref, approximate="tanh")
        elif act == 2:
            e = torch.nn.functional.silu(ref)
        assert float((out16.float().cpu() - e).abs().max()) < 0.02 * max(1.0, float(e.abs().max()))


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 256, 128), (384, 512, 2048), (4096, 2048, 2048),
                                   (1000, 2048, 128), (96, 128, 2048)])
def test_gemm_kmajor(lib, cg, M, N, K):
    _run(lib, M, N, K, cg=cg)


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("N,BN", [(42, 0), (146, 0), (384, 128), (128, 128), (512, 256)])
def test_gemm_narrow_and_ragged_n(lib, cg, N, BN):
    _run(lib, 300, N, 2048, BN=BN, cg=cg, bias=True)


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_fused_epilogues(lib, cg):
    _run(lib, 512, 2048, 128, cg=cg, bias=True, act=1, out_bf16=True)               # FFN up + GELU
    _run(lib, 512, 2048, 2048, cg=cg, bias=True, residual=True, stats=True)          # res-block GEMM + row stats
    _run(lib, 520, 128, 2048, cg=cg, bias=True, residual=True, ln=True, BN=128)      # FFN down + residual + LN
    _run(lib, 256, 2048, 2048, cg=cg, bias=True, act=2, out_bf16=True)


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("a_mn,b_mn", [(1, 1), (0, 1), (1, 0)])
def test_gemm_mn_major_operands(lib, cg, a_mn, b_mn):
    # dW = X^T G (both MN-major, reduction over tokens) and forward with un-transposed (in,out) weights
    _run(lib, 2048, 256, 1024, a_mn=a_mn, b_mn=b_mn, cg=cg, BN=256)
    _run(lib, 128, 2048, 4096, a_mn=a_mn, b_mn=b_mn, cg=cg, BN=256)
