"""The swapped-operand GEMM (gemm_bf16_wgmma_swap_kernel: N = 128, 32-token tiles in CTA pairs) against the 128 x 128
GEMM on the same operands, for every epilogue it serves: the dX kind (fp32 out, plain weight read K-major) and the
forward kind (bias + residual + fp32 out + full-row LayerNorm to bf16, (in, out) weight read MN-major), plus bias-only
fp32 and plain bf16 outputs.  The 128 x 128 GEMM runs the same product with the token operand handed over MN-major
(transposed), a layout the swapped kernel does not take.  fp32 outputs agree to 1e-5 relative L2 (accumulation order
inside a k16 step); the bf16 outputs are held to the far / not-nearest shares of the stage tests against the float64
LayerNorm of the 128 x 128 GEMM's fp32 output."""
import math

import pytest
import torch

from tests import backward_reference as R
from tests.test_gpu_backward_stages import FAR, NOT_NEAREST

pytestmark = pytest.mark.gpu
N = 128


def _gemm(lib, X, a_mn, W, b_mn, M, K, bias=None, res=None, out_bf16=False, ln=None):
    """out = X W^T (+ bias + res) through the C ABI hook; X is [M][K] (a_mn = 0: the swapped route) or [K][M]
    (a_mn = 1: the 128 x 128 route)."""
    from smd_b200 import lib as L
    out32 = torch.full((M, N), float("nan"), device="cuda")
    out16 = torch.zeros((M, N), dtype=torch.bfloat16, device="cuda") if out_bf16 else None
    p = lambda t: None if t is None else t.data_ptr()
    gam, bet = ln if ln is not None else (None, None)
    L.check(lib.smd_gemm_bf16(X.data_ptr(), W.data_ptr(), M, N, K, a_mn, b_mn, 0, 1, p(bias), p(res), 0,
                              out32.data_ptr(), p(out16), None, p(gam), p(bet),
                              torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out32, out16


def _operands(M, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    X = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    Wt = (torch.randn(N, K, generator=g) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16)   # [out][in = K]
    return g, X, Wt


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _bf16_rules(got, ref):
    ref = ref.double().cpu()
    got = got.double().cpu()
    n = ref.numel()
    f_far = int(((got - ref).abs() > R.bf16_ulp(ref)).sum()) / n
    f_nn = int((got != R.bf16_round(ref)).sum()) / n
    assert f_far <= FAR and f_nn <= NOT_NEAREST, (f_far, f_nn)


@pytest.mark.parametrize("M", [32, 96, 4096, 32000])
@pytest.mark.parametrize("K", [128, 384, 2048])
def test_swap_dx_kind_matches_128x128(lib, M, K):
    """dX: G [tokens][K] times the plain weight [128][K] (K-major), fp32 out.  (At 32 000 tokens gemm_kind keeps this
    kind on the 128 x 128 layouts: the two routes then differ only in how the token operand is read.)"""
    _, X, Wt = _operands(M, K, seed=M + K)
    W = Wt.cuda()
    new, _ = _gemm(lib, X, 0, W, 0, M, K)
    old, _ = _gemm(lib, X.t().contiguous(), 1, W, 0, M, K)
    assert not torch.isnan(new).any(), "unwritten rows"
    assert _rel(new, old) <= 1e-5


@pytest.mark.parametrize("M", [32, 96, 4096, 32000])
@pytest.mark.parametrize("K", [128, 384, 2048])
def test_swap_layernorm_kind_matches_128x128(lib, M, K):
    """Forward out-projection / FFN down: X [tokens][K] times the (in, out) weight [K][128] (MN-major), + bias +
    residual, fp32 out and LayerNorm(v) gamma + beta to bf16."""
    g, X, Wt = _operands(M, K, seed=7 * M + K)
    W = Wt.t().contiguous().cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).cuda()
    gam = (1 + 0.1 * torch.randn(N, generator=g)).cuda()
    bet = (0.1 * torch.randn(N, generator=g)).cuda()
    kw = dict(bias=bias, res=res, out_bf16=True, ln=(gam, bet))
    new32, new16 = _gemm(lib, X, 0, W, 1, M, K, **kw)
    old32, old16 = _gemm(lib, X.t().contiguous(), 1, W, 1, M, K, **kw)
    assert not torch.isnan(new32).any(), "unwritten rows"
    assert _rel(new32, old32) <= 1e-5
    v = old32.double().cpu()
    mu = v.mean(1, keepdim=True)
    var = (v * v).mean(1, keepdim=True) - mu * mu
    ref = (v - mu) * torch.rsqrt(var + 1e-6) * gam.double().cpu() + bet.double().cpu()
    _bf16_rules(new16, ref)
    _bf16_rules(old16, ref)


@pytest.mark.parametrize("M", [96, 4096])
def test_swap_bias_and_plain_bf16_outputs(lib, M):
    """bias-only fp32 out, and a bf16 copy of v without LayerNorm, both weight layouts."""
    K = 384
    for b_mn in (0, 1):
        g, X, Wt = _operands(M, K, seed=M + b_mn)
        W = (Wt.t().contiguous() if b_mn else Wt).cuda()
        bias = torch.randn(N, generator=g).cuda()
        new32, new16 = _gemm(lib, X, 0, W, b_mn, M, K, bias=bias, out_bf16=True)
        old32, _ = _gemm(lib, X.t().contiguous(), 1, W, b_mn, M, K, bias=bias, out_bf16=True)
        assert _rel(new32, old32) <= 1e-5
        _bf16_rules(new16, old32)
