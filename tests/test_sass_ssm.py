"""The sliced-score-matching kernels (tangent LayerNorm-FiLM-swish, its second-order backward, the loss, the tangent
input cast) compile without register spills: no local-memory traffic (STL / LDL) in their SASS."""
from tests.test_sass_evidence import _get, table  # noqa: F401  (module-scoped fixture: one cuobjdump pass)

SSM_KERNELS = ("ln_film_tangent_kernel", "ssm_ln_bwd_kernel<", "ssm_loss_kernel", "tangent_input_kernel")


def test_ssm_kernels_do_not_spill(table):  # noqa: F811
    for prefix in SSM_KERNELS:
        for c in _get(table, prefix):
            assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, (prefix, c)
