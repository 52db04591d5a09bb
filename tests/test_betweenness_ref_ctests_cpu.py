"""The reference's betweenness C-API test programs linked against the CPU emulation build (see
tests/test_betweenness_ref_ctests_gpu.py)."""
import pytest

from tests.test_betweenness_ref_ctests_gpu import CASES, run_program


@pytest.mark.parametrize("name", sorted(CASES))
def test_betweenness_reference_c_program_emulated(name):
    run_program(name, "")
