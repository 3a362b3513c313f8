"""The dedicated-epilogue GEMM layout (launches of more tiles than SMs) computes the same bits as the 8-warp layout.

A tile's arithmetic does not depend on M, so a multi-round launch is compared row block by row block against
single-round launches (sized from the device's SM count, so they run the 8-warp layout) on those rows copied out
contiguously: fp32 and bf16 outputs bit for bit, row statistics (atomics, order dependent) to fp32 tolerance.
One case per converted epilogue kind, with the operand layouts the train step uses."""
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 2048
# name -> (a_mn, b_mn, K, outputs)
KINDS = {
    "res-a": (0, 1, 2048, ("bias", "bf16", "stats")),          # kEpiAct
    "res-b": (0, 1, 2048, ("bias", "res", "f32", "stats")),    # kEpiF32Res
    "dX": (0, 0, 2048, ("bf16",)),                             # kEpiAct
    "dW": (1, 1, 4096, ("f32",)),                              # kEpiF32, reduction over 4096 tokens
}


def _gemm(lib, A, B, M, K, a_mn, b_mn, outs, bias, res):
    from smd_b200 import lib as L
    o32 = torch.full((M, N), float("nan"), device="cuda") if "f32" in outs else None
    o16 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16) if "bf16" in outs else None
    stats = torch.zeros(M, 2, device="cuda") if "stats" in outs else None
    p = lambda t: None if t is None else t.data_ptr()
    L.check(lib.smd_gemm_bf16(A.data_ptr(), B.data_ptr(), M, N, K, a_mn, b_mn, 128, 1, p(bias), p(res), 0, p(o32),
                              p(o16), p(stats), None, None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o32, o16, stats


@pytest.mark.parametrize("M", [4096, 4000, 1152])
@pytest.mark.parametrize("kind", list(KINDS))
def test_multi_round_launch_matches_single_round_blocks(lib, kind, M):
    a_mn, b_mn, K, outs = KINDS[kind]
    if kind == "dW" and M == 4096:
        M = 2048                                                # dW's output rows are the 2048 input features
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    num_n = N // 128
    if ((M + 127) // 128) * num_n <= sms:
        pytest.skip(f"{M} rows fit one round on {sms} SMs")
    block = max(1, sms // num_n) * 128                          # rows of a single-round launch
    g = torch.Generator(device="cuda").manual_seed(M + K + a_mn)
    A = (torch.randn(*((K, M) if a_mn else (M, K)), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    B = (torch.randn(*((K, N) if b_mn else (N, K)), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g) if "bias" in outs else None
    res = torch.randn(M, N, device="cuda", generator=g) if "res" in outs else None
    full = _gemm(lib, A, B, M, K, a_mn, b_mn, outs, bias, res)
    for r0 in range(0, M, block):
        r1 = min(M, r0 + block)
        Ab = (A[:, r0:r1] if a_mn else A[r0:r1]).contiguous()
        part = _gemm(lib, Ab, B, r1 - r0, K, a_mn, b_mn, outs, bias, None if res is None else res[r0:r1].contiguous())
        for name, got, want in zip(("f32", "bf16"), full[:2], part[:2]):
            if want is None:
                continue
            assert not torch.isnan(got[r0:r1]).any(), f"{name} rows [{r0}, {r1}) not written"
            assert torch.equal(got[r0:r1].view(torch.int16 if name == "bf16" else torch.int32),
                               want.view(torch.int16 if name == "bf16" else torch.int32)), \
                f"{name} rows [{r0}, {r1}) differ from the single-round launch"
        if full[2] is not None:
            torch.testing.assert_close(full[2][r0:r1], part[2], rtol=1e-5, atol=1e-2)
