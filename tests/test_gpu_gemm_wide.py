"""The wide GEMM layout (128 x 256 tiles, BN = 256) computes the same bits as the 128-wide layouts.

Each res-block GEMM kind runs with the operand layouts the train step uses, once with BN = 256 and once with BN = 128
on the same operands.  Every output element accumulates the same k16 blocks in the same order and the epilogue applies
the same per-element operations, so fp32 and bf16 outputs must match bit for bit.  Row statistics are summed in a
different order (atomics, and per-quad partials in the wide layout) and are compared to fp32 tolerance.  Outputs are
prefilled with NaN, so a row the wide launch leaves unwritten fails the comparison."""
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 2048
# name -> (a_mn, b_mn, K, outputs)
KINDS = {
    "res-a": (0, 1, 2048, ("bias", "bf16", "stats")),          # kEpiBf16 (wide), kEpiAct (128-wide)
    "res-b": (0, 1, 2048, ("bias", "res", "f32", "stats")),    # kEpiF32Res: stays 128-wide
    "dX": (0, 0, 2048, ("bf16",)),                             # kEpiBf16 (wide), kEpiAct (128-wide)
    "dW": (1, 1, 4096, ("f32",)),                              # kEpiF32, reduction over 4096 tokens
}


def _gemm(lib, A, B, M, K, a_mn, b_mn, BN, outs, bias, res):
    from smd_b200 import lib as L
    o32 = torch.full((M, N), float("nan"), device="cuda") if "f32" in outs else None
    o16 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16) if "bf16" in outs else None
    stats = torch.zeros(M, 2, device="cuda") if "stats" in outs else None
    p = lambda t: None if t is None else t.data_ptr()
    L.check(lib.smd_gemm_bf16(A.data_ptr(), B.data_ptr(), M, N, K, a_mn, b_mn, BN, 1, p(bias), p(res), 0, p(o32),
                              p(o16), p(stats), None, None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o32, o16, stats


def _operands(kind, M):
    a_mn, b_mn, K, outs = KINDS[kind]
    g = torch.Generator(device="cuda").manual_seed(M + K + a_mn + 7)
    A = (torch.randn(*((K, M) if a_mn else (M, K)), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    B = (torch.randn(*((K, N) if b_mn else (N, K)), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g) if "bias" in outs else None
    res = torch.randn(M, N, device="cuda", generator=g) if "res" in outs else None
    return A, B, bias, res


@pytest.mark.parametrize("M", [4096, 4000, 1152])
@pytest.mark.parametrize("kind", list(KINDS))
def test_wide_tiles_match_128_wide_tiles(lib, kind, M):
    a_mn, b_mn, K, outs = KINDS[kind]
    if kind == "dW" and M == 4096:
        M = 2048                                                # dW's output rows are the 2048 input features
    A, B, bias, res = _operands(kind, M)
    wide = _gemm(lib, A, B, M, K, a_mn, b_mn, 256, outs, bias, res)
    narrow = _gemm(lib, A, B, M, K, a_mn, b_mn, 128, outs, bias, res)
    for name, got, want in zip(("f32", "bf16"), wide[:2], narrow[:2]):
        if want is None:
            continue
        assert not torch.isnan(got).any(), f"{name}: rows not written by the wide launch"
        bits = torch.int16 if name == "bf16" else torch.int32
        assert torch.equal(got.view(bits), want.view(bits)), f"{name} differs from the 128-wide launch"
    if wide[2] is not None:
        torch.testing.assert_close(wide[2], narrow[2], rtol=1e-5, atol=1e-2)


@pytest.mark.parametrize("kind", list(KINDS))
def test_bn_256_selects_the_wide_kernel_by_epilogue_kind(lib, kind):
    """BN = 256 on a long-K, multi-round launch runs gemm_bf16_wgmma_wide_kernel for the fp32 and bf16 kinds; res-b
    (fp32 residual) keeps the 128-wide dedicated-epilogue kernel, and so does every BN = 128 launch."""
    from torch.profiler import ProfilerActivity, profile
    a_mn, b_mn, K, outs = KINDS[kind]
    M = 2048 if kind == "dW" else 4096
    A, B, bias, res = _operands(kind, M)
    names = {}
    for BN in (256, 128):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _gemm(lib, A, B, M, K, a_mn, b_mn, BN, outs, bias, res)
        names[BN] = [e.name for e in prof.events() if "gemm_bf16_wgmma" in e.name]
        assert names[BN], f"no GEMM kernel in the profile of the BN = {BN} launch"
    assert any("wide_kernel" in n for n in names[256]) == (kind != "res-b"), names[256]
    assert not any("wide_kernel" in n for n in names[128]), names[128]
