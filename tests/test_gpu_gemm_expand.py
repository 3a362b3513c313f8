"""The row-resident expand GEMM (gemm_bf16_wgmma_expand_kernel: K = 128, N a multiple of 256) against the 128 x 128
GEMM on the same operands, for each epilogue it serves: FFN up (bias + tanh-GELU to bf16, with the bf16
pre-activation), its adjoint (x gelu'(pre-activation) to bf16) and the post dense (bias, fp32 out, row-statistics
partials).  The 128 x 128 GEMM runs the same product with A handed over MN-major ([K][M]), a layout the expand kernel
does not take.  Every output, the statistics partials included, is bit-identical; the fp32 outputs also agree with a
float64 product to the bounds of test_gpu_gemm (fp32 accumulation-order noise)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
K = 128
GELU = 1


def _run(lib, kind, X, a_mn, W, b_mn, M, N, bias=None, gg=None):
    from smd_b200 import lib as L
    import ctypes
    p = lambda t: None if t is None else t.data_ptr()
    o32 = o16 = pre = stats = part = None
    if kind == "post":
        o32 = torch.full((M, N), float("nan"), device="cuda")
        stats = torch.zeros(M, 2, device="cuda")
        part = torch.full((M, N // 128 * 3, 2), float("nan"), device="cuda")
    else:
        o16 = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        if kind == "up":
            pre = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    nslots = ctypes.c_int(0)
    L.check(lib.smd_gemm_bf16_epi(X.data_ptr(), W.data_ptr(), M, N, K, a_mn, b_mn, p(bias), GELU if kind == "up" else 0,
                                  p(o32), p(o16), p(pre), p(gg), p(stats), p(part), ctypes.byref(nslots),
                                  torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return {"f32": o32, "bf16": o16, "pre": pre, "part": part, "nslots": nslots.value}


def _operands(kind, M, N, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    X = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).cuda()
    if kind == "dx2":
        W = (torch.randn(N, K, generator=g) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16).cuda()   # [N][K]
        b_mn, bias = 0, None
        gg = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    else:
        W = (torch.randn(K, N, generator=g) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16).cuda()   # (in, out)
        b_mn, bias, gg = 1, torch.randn(N, generator=g).cuda(), None
    return X, W, b_mn, bias, gg


def _both(lib, kind, M, N):
    X, W, b_mn, bias, gg = _operands(kind, M, N, seed=M + N + len(kind))
    new = _run(lib, kind, X, 0, W, b_mn, M, N, bias, gg)
    old = _run(lib, kind, X.t().contiguous(), 1, W, b_mn, M, N, bias, gg)
    return X, W, b_mn, bias, new, old


@pytest.mark.parametrize("M", [4096, 4064, 104, 32000])
@pytest.mark.parametrize("N", [512, 2048])
@pytest.mark.parametrize("kind", ["up", "dx2", "post"])
def test_expand_matches_128x128_bitwise(lib, kind, M, N):
    X, W, b_mn, bias, new, old = _both(lib, kind, M, N)
    for key in ("f32", "bf16", "pre", "part"):
        if new[key] is None:
            continue
        a, b = new[key], old[key]
        if a.dtype == torch.bfloat16:
            a, b = a.view(torch.int16), b.view(torch.int16)
        else:
            a, b = a.view(torch.int32), b.view(torch.int32)
        assert torch.equal(a, b), (kind, key, int((a != b).sum()))
    if kind == "post":
        assert new["nslots"] == old["nslots"] == N // 128 * 3
        # fp32 product against float64 (test_gpu_gemm's bound)
        Wt = W.double() if b_mn else W.double().t()
        ref = X.double() @ Wt + bias.double()
        err = new["f32"].double() - ref
        assert float(err.norm() / ref.norm()) < 2e-5
        assert float(err.abs().max()) < 2e-3 * math.sqrt(K / 64)
        # the partials add up to the float64 row statistics
        s = new["part"].double().sum(1)
        torch.testing.assert_close(s[:, 0], ref.sum(1), rtol=1e-4, atol=1e-2)
        torch.testing.assert_close(s[:, 1], (ref * ref).sum(1), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("kind", ["up", "dx2", "post"])
def test_train_step_shape_runs_the_expand_kernel(lib, kind):
    """4096 tokens, N = 2048, K-major A: the expand kernel; A MN-major: the 128 x 128 kernel."""
    from torch.profiler import ProfilerActivity, profile
    M, N = 4096, 2048
    X, W, b_mn, bias, gg = _operands(kind, M, N, seed=5)
    Xt = X.t().contiguous()
    names = {}
    for a_mn, A in ((0, X), (1, Xt)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _run(lib, kind, A, a_mn, W, b_mn, M, N, bias, gg)
        names[a_mn] = [e.name for e in prof.events() if "gemm_bf16_wgmma" in e.name]
        assert names[a_mn], names
    assert all("expand_kernel" in n for n in names[0]), names[0]
    assert not any("expand_kernel" in n for n in names[1]), names[1]
