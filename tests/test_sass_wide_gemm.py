"""The wide GEMM layout (gemm_bf16_wgmma_wide_kernel<kind>, 128 x 256 tiles) issues 256-wide wgmma (HGMMA.64x256x16),
loads its operands with TMA (UTMALDG), moves registers from the producer to the MMA warpgroups (setmaxnreg =
USETMAXREG) and keeps its 128 accumulators per thread and the epilogue in registers: no local-memory traffic (STL /
LDL).  CPU only: cuobjdump on libsmd.so, through the SASS table of test_sass_evidence."""
from .test_sass_evidence import _get, table  # noqa: F401  (pytest fixture)

# kEpiF32, kEpiBf16 (gemm_wgmma.cuh)
WIDE_KINDS = (37, 57)


def test_wide_gemm_kernels_use_256_wide_wgmma_and_do_not_spill(table):  # noqa: F811
    for kind in WIDE_KINDS:
        (c,) = _get(table, f"gemm_bf16_wgmma_wide_kernel<{kind}u>")
        assert c.get("HGMMA.64x256x16", 0) > 0
        assert c.get("HGMMA", 0) == c.get("HGMMA.64x256x16", 0)   # no narrower wgmma in this layout
        assert c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0
        assert c.get("USETMAXREG", 0) >= 2         # the producer warpgroup gives, the MMA warpgroups take
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0
