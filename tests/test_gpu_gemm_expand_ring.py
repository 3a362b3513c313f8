"""The expand GEMM's staging ring (gemm_bf16_wgmma_expand_kernel: each consumer warpgroup stages 64-column half-tiles
through three shared-memory slots while the bulk stores of the previous two are in flight).  Every output buffer,
the statistics partials included, starts filled with a NaN sentinel and has rows past M.  At N = 512 a CTA writes 4
half-tiles (the ring wraps once), at N = 2048 8 (4096 tokens) or 32 (32 000 tokens, one column group per row block).
Every valid element must equal the 128 x 128 route's bit for bit (which starts from a different sentinel, so nothing
can match by being left unwritten), and the rows past M must still hold the sentinel.  A slot rewritten before its
stores have read it, or a store past M, shows up here."""
import ctypes

import pytest
import torch

from .test_gpu_gemm_expand import GELU, K, _operands

pytestmark = pytest.mark.gpu
PAD = 40                                           # rows past M in every output buffer
SENTINEL = {torch.bfloat16: (0x7FC1, 0x7FC2), torch.float32: (0x7FC00001, 0x7FC00002)}


def _filled(shape, dtype, which):
    bits = torch.int16 if dtype == torch.bfloat16 else torch.int32
    return torch.full(shape, SENTINEL[dtype][which], dtype=bits, device="cuda").view(dtype)


def _run(lib, kind, A, a_mn, W, b_mn, M, N, bias, gg, which):
    from smd_b200 import lib as L
    p = lambda t: None if t is None else t.data_ptr()
    o = {}
    if kind == "post":
        o["f32"] = _filled((M + PAD, N), torch.float32, which)
        o["part"] = _filled((M + PAD, N // 128 * 3, 2), torch.float32, which)
        stats = torch.zeros(M, 2, device="cuda")
    else:
        o["bf16"] = _filled((M + PAD, N), torch.bfloat16, which)
        if kind == "up":
            o["pre"] = _filled((M + PAD, N), torch.bfloat16, which)
        stats = None
    nslots = ctypes.c_int(0)
    L.check(lib.smd_gemm_bf16_epi(A.data_ptr(), W.data_ptr(), M, N, K, a_mn, b_mn, p(bias),
                                  GELU if kind == "up" else 0, p(o.get("f32")), p(o.get("bf16")), p(o.get("pre")),
                                  p(gg), p(stats), p(o.get("part")), ctypes.byref(nslots),
                                  torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize("M,N", [(4096, 512), (4064, 512), (4096, 2048), (32000, 2048)])
@pytest.mark.parametrize("kind", ["up", "dx2", "post"])
def test_ring_writes_every_valid_byte_once_and_nothing_past_m(lib, kind, M, N):
    X, W, b_mn, bias, gg = _operands(kind, M, N, seed=3 * M + N + len(kind))
    new = _run(lib, kind, X, 0, W, b_mn, M, N, bias, gg, 0)
    old = _run(lib, kind, X.t().contiguous(), 1, W, b_mn, M, N, bias, gg, 1)
    for key, t in new.items():
        a, b = _bits(t), _bits(old[key])
        assert torch.equal(a[:M], b[:M]), (kind, key, int((a[:M] != b[:M]).sum()))
        assert bool((a[M:] == SENTINEL[t.dtype][0]).all()), (kind, key, "rows past M were written")
