"""The fused DPM-Solver++ update (dpm_step_kernel) compiles without register spills: no local-memory traffic (STL /
LDL) in its SASS."""
from tests.test_sass_evidence import _get, table  # noqa: F401  (module-scoped fixture: one cuobjdump pass)


def test_dpm_step_kernel_does_not_spill(table):  # noqa: F811
    for c in _get(table, "dpm_step_kernel"):
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, c
