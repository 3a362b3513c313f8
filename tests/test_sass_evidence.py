"""The built library really contains the Hopper instructions the design claims (CPU only: cuobjdump on libsmd.so):
wgmma (HGMMA) and TMA tensor loads (UTMALDG) with mbarriers (SYNCS) in the GEMM and in the fused FFN / attention-block
kernels, mma.sync tf32 in the attention kernels (HMMA) and programmatic dependent launch (ACQBULK)."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "symbolic-music-diffusion_b200", "libsmd.so")


@pytest.fixture(scope="module")
def table():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not available")
    if not os.path.exists(LIB):
        pytest.skip("libsmd.so not built")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sass_mnemonics.py")], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    rows = {}
    for line in r.stdout.splitlines():
        if line.startswith("#") or not line.strip():
            continue
        parts = line.split("  ")
        name = parts[0].strip()
        counts = {}
        for tok in line[len(parts[0]):].split():
            if "=" in tok:
                k, v = tok.split("=")
                counts[k] = int(v)
        rows[name] = counts
    return rows


def _get(table, prefix):
    hits = [v for k, v in table.items() if k.startswith(prefix)]
    assert hits, f"no kernel named {prefix}* in the SASS table"
    return hits


def test_gemm_family_uses_wgmma_tma_and_mbarriers(table):
    for c in _get(table, "gemm_bf16_wgmma_kernel<"):
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0
        assert c.get("SYNCS", 0) > 0 and c.get("ACQBULK", 0) > 0
        assert c.get("HMMA", 0) == 0                      # no legacy mma.sync in the GEMM path


def test_fused_ffn_uses_wgmma_and_tma(table):
    for c in _get(table, "ffn_fused_kernel<"):
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0
        assert c.get("MUFU.TANH", 0) >= 64                # 64 columns of tanh-GELU per thread and chunk


def test_attention_block_uses_wgmma_gemms(table):
    for c in _get(table, "attn_block_kernel<"):
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0 and c.get("SYNCS", 0) > 0


def test_attention_kernels_use_an_mma_sync_core(table):
    for c in _get(table, "attention_mma_kernel<") + _get(table, "attention_bwd_mma_kernel<"):
        assert c.get("HMMA", 0) > 0
