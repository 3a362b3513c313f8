"""The swapped-operand GEMM (gemm_bf16_wgmma_swap_kernel, N = 128 on 32-token tiles) issues 32-wide wgmma
(HGMMA.64x32x16) only, loads the weight with multicast TMA inside its CTA pair and the token tile with plain TMA
(UTMALDG), and keeps its accumulators and epilogue out of local memory (no STL / LDL).  CPU only: cuobjdump on
libsmd.so, through the SASS table of test_sass_evidence."""
from .test_sass_evidence import _get, table  # noqa: F401  (pytest fixture)


def test_swap_gemm_uses_32_wide_wgmma_multicast_tma_and_does_not_spill(table):  # noqa: F811
    kinds = _get(table, "gemm_bf16_wgmma_swap_kernel<")
    assert len(kinds) == 2                        # the weight read MN-major (forward) and K-major (dX)
    for c in kinds:
        assert c.get("HGMMA.64x32x16", 0) > 0
        assert c.get("HGMMA", 0) == c.get("HGMMA.64x32x16", 0)
        assert c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0 and c.get("ACQBULK", 0) > 0
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0
