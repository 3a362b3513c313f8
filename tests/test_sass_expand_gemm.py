"""The row-resident expand GEMM (gemm_bf16_wgmma_expand_kernel: K = 128, wide N) issues 128-wide wgmma, loads its
operands with TMA and mbarriers, writes its outputs with bulk copies (UBLKCP) instead of per-thread global stores, keeps
everything out of local memory, and is allocated within the 168 registers per thread that let its 384 threads start
(setmaxnreg then moves them between the producer and the consumer warpgroups).  CPU only: cuobjdump on libsmd.so."""
import re
import shutil
import subprocess

import pytest

from .test_sass_evidence import LIB, _get, table  # noqa: F401  (pytest fixture)


def test_expand_gemm_uses_wgmma_and_bulk_stores_and_does_not_spill(table):  # noqa: F811
    kinds = _get(table, "gemm_bf16_wgmma_expand_kernel<")
    assert len(kinds) == 6                        # kEpiAct / kEpiGG / kEpiF32, weight K-major and MN-major
    for c in kinds:
        assert c.get("HGMMA", 0) > 0                 # m64n128k16 only
        assert c.get("HGMMA.64x256x16", 0) == 0 and c.get("HGMMA.64x32x16", 0) == 0
        assert c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0 and c.get("UBLKCP", 0) > 0
        assert c.get("USETMAXREG", 0) > 0
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0


def test_expand_gemm_register_count_allows_one_cta_per_sm():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    regs = [int(m.group(1)) for m in re.finditer(r"Function \S*gemm_bf16_wgmma_expand_kernel\S*:\s*\n\s*REG:(\d+)", out)]
    assert len(regs) >= 6, out[:2000]
    assert max(regs) * 384 <= 65536, regs
