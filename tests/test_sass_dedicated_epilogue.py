"""The dedicated-epilogue GEMM layout (gemm_bf16_wgmma_kernel<kind, 4>) really moves registers between its
warpgroups (setmaxnreg = USETMAXREG) and, with the epilogue warpgroup's larger budget, keeps every value in registers:
no local-memory traffic (STL / LDL).  CPU only: cuobjdump on libsmd.so, through the SASS table of test_sass_evidence."""
from .test_sass_evidence import _get, table  # noqa: F401  (pytest fixture)

# kEpiF32, kEpiF32Res, kEpiAct (gemm_wgmma.cuh)
DEDICATED_KINDS = (37, 39, 569)


def test_dedicated_epilogue_kernels_set_register_budgets_and_do_not_spill(table):  # noqa: F811
    for kind in DEDICATED_KINDS:
        (c,) = _get(table, f"gemm_bf16_wgmma_kernel<{kind}u, 4>")
        assert c.get("USETMAXREG", 0) >= 3          # producer and MMA warpgroups give, the epilogue warpgroup takes
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0
