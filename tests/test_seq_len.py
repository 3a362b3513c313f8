"""Sequence lengths 64 and 128 for TransformerDDPM, CPU-only checks: plans build, the parameter layout does not depend
on the length (a checkpoint trained at one length loads at another), every other length is rejected, and the attention
kernels instantiated for the new lengths keep every value in registers (no STL / LDL in their SASS)."""
import pytest

from .test_sass_evidence import _get, table  # noqa: F401  (pytest fixture)


@pytest.mark.parametrize("seq_len", [64, 128])
def test_longer_sequences_build_plans_with_the_same_layout(seq_len):
    from smd_b200 import Engine, ModelConfig
    for arch in ("TransformerDDPM", "TransformerDDPM4"):
        for training in (False, True):
            ref = Engine(ModelConfig(arch=arch), 4, training=training)
            eng = Engine(ModelConfig(arch=arch, seq_len=seq_len), 4, training=training)
            assert eng.seq_len == seq_len
            assert eng.layout == ref.layout
            assert eng.arena_floats == ref.arena_floats


@pytest.mark.parametrize("seq_len", [48, 96, 256])
def test_other_sequence_lengths_are_rejected(seq_len):
    from smd_b200 import Engine, ModelConfig
    with pytest.raises(ValueError, match=r"\{32, 64, 128\}"):
        Engine(ModelConfig(seq_len=seq_len), 4)


def test_long_sequence_attention_kernels_do_not_spill(table):  # noqa: F811
    for prefix in ("attention_kernel<", "attention_mma_kernel<", "attention_bwd_long_kernel<", "attn_block_kernel<"):
        rows = {k: v for k, v in table.items() if k.startswith(prefix) and (k.endswith(", 64>") or k.endswith(", 128>"))}
        assert rows, prefix
        for name, c in rows.items():
            assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, name
    for S in (64, 128):
        for dh in (8, 16, 32):
            (c,) = _get(table, f"attention_mma_kernel<{dh}, {S}>")
            assert c.get("HMMA", 0) > 0
