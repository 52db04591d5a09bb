"""The reference's own C-API test programs for betweenness centrality (cpp/tests/c_api/{betweenness_centrality,
edge_betweenness_centrality}_test.c, unmodified), built by oracle/ref_ctests/build_betweenness.sh against the emulation build
(run by tests/test_betweenness_ref_ctests_cpu.py) and against the CUDA library (run here on the GPU).  Every case must report
`passed`."""
import os
import subprocess

import pytest

from tests.test_reference_c_tests_cpu import ROOT

pytestmark = pytest.mark.gpu

CASES = {
    "betweenness_centrality": ["test_betweenness_centrality_full", "test_betweenness_centrality_full_directed",
                               "test_betweenness_centrality_specific_normalized",
                               "test_betweenness_centrality_specific_unnormalized", "test_betweenness_centrality_test_endpoints",
                               "test_betweenness_centrality_full_directed_normalized_karate", "test_issue_4941",
                               "test_issue_4941_with_endpoints"],
    "edge_betweenness_centrality": ["test_edge_betweenness_centrality"],
}


def run_program(name, suffix):
    exe = os.path.join(ROOT, "oracle", "_ref", f"ref_{name}_test{suffix}")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_*_test not built (needs the reference sources at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RUNNING:")]
    assert len(lines) == len(CASES[name]), r.stdout
    for case, ln in zip(CASES[name], lines):
        assert ln.startswith(f"RUNNING: {case}...") and ln.endswith("- passed"), ln


@pytest.mark.parametrize("name", sorted(CASES))
def test_betweenness_reference_c_program_on_gpu(name):
    run_program(name, "_gpu")
