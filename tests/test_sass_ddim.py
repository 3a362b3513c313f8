"""The fused DDIM update (ddim_step_kernel) compiles without register spills: no local-memory traffic (STL / LDL) in
its SASS."""
from tests.test_sass_evidence import _get, table  # noqa: F401  (module-scoped fixture: one cuobjdump pass)


def test_ddim_step_kernel_does_not_spill(table):  # noqa: F811
    for c in _get(table, "ddim_step_kernel"):
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, c
