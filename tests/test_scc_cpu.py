"""Strongly connected components on the CPU: the checks of tests/test_scc_gpu.py driven through the Python surface over the
emulation build of the library (tests/emu_py.py), at sizes the emulation runs in seconds, plus the reference's own
strongly_connected_components_test.c linked against that build."""
import pytest

from tests import test_scc_gpu as t
from tests.emu_py import surface  # noqa: F401


def test_scc_goldens_emulated(surface, monkeypatch):
    t.check_goldens(monkeypatch)


def test_scc_legacy_csr_with_labels_array_emulated(surface):
    cases = [c for c in t.golden_cases().values() if "scc_comp_vertices" in c]
    assert len(cases) == 4
    for c in cases:
        t.check_legacy_csr(c)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_scc_random_both_orientations_emulated(surface, monkeypatch, seed):
    t.check_random(monkeypatch, 3000, 9000 * seed, seed=seed)


def test_scc_loops_and_multi_edges_emulated(surface, monkeypatch):
    t.check_loops_and_multi_edges(monkeypatch, 2000, 5000, seed=4)


def test_scc_both_directions_equals_wcc_emulated(surface, monkeypatch):
    t.check_both_directions_equals_wcc(monkeypatch, 3000, 2500, seed=5)


def test_scc_symmetric_graph_rejected_emulated(surface, monkeypatch):
    t.check_symmetric_rejected(monkeypatch)


def test_scc_empty_graph_and_isolated_vertices_emulated(surface, monkeypatch):
    t.check_empty_and_isolated(monkeypatch)


def test_scc_int64_ids_and_renumber_false_emulated(surface, monkeypatch):
    t.check_int64_renumber_false(monkeypatch, 2000, 8000, seed=6)


def test_scc_offs64_emulated(surface, monkeypatch):
    t.check_random(monkeypatch, 2000, 8000, seed=7, knobs=t.OFFS64)
    t.check_int64_renumber_false(monkeypatch, 1000, 4000, seed=8, knobs=t.OFFS64)


def test_scc_phase_shapes_emulated(surface, monkeypatch, capfd):
    """the chain is resolved by the trim alone, the cycle by the forward-backward step, the chain of cycles needs colouring"""
    monkeypatch.setenv("CUGRAPH_B200_SCC_TRACE", "1")
    t.check_edges(monkeypatch, *t.chain(300))
    err = capfd.readouterr().err
    assert "scc trim       rounds=150 resolved=300" in err and "scc fw-bw" not in err, err
    t.check_edges(monkeypatch, *t.cycle(300))
    err = capfd.readouterr().err
    assert "resolved=300" in err.split("scc fw-bw")[1].splitlines()[0], err
    t.check_shapes(monkeypatch, 200, 30, 4)
    assert "scc colouring" in capfd.readouterr().err


def test_scc_user_level_api_emulated(surface):
    t.check_api()


def test_reference_scc_c_test():
    t.run_reference_c_test("")
