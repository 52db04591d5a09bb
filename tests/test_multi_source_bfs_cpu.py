"""Multi-source BFS on the CPU: the checks of tests/test_multi_source_bfs_gpu.py driven through the Python surface over the
emulation build of the library (tests/emu_py.py), at sizes the emulation runs in seconds."""
import numpy as np
import pytest

from tests import test_multi_source_bfs_gpu as t
from tests.emu_py import surface  # noqa: F401


@pytest.mark.parametrize("kind", ["random", "random_sym"])
def test_rows_emulated(surface, monkeypatch, kind):
    t.check_rows(monkeypatch, kind, 300, n_sources=(1, 5, 64, 65, 130), limits=(0, 1, 3), with_oracle=True)


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_rmat_rows_emulated(surface, monkeypatch, kind):
    t.check_rows(monkeypatch, kind, 9, n_sources=(63, 65), limits=(0, 3))


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_schedules_emulated(surface, monkeypatch, capfd, kind):
    t.check_schedules(monkeypatch, capfd, kind, 9)


def test_layouts_emulated(surface, monkeypatch):
    for st in (False, True):
        for rn in (True, False):
            t.check_rows(monkeypatch, "rmat", 8, n_sources=(65,), limits=(0,), store_transposed=st, renumber=rn)
    t.check_rows(monkeypatch, "rmat_sym", 8, n_sources=(65,), limits=(0,), vertex_dtype=np.int64, renumber=False)
    t.check_rows(monkeypatch, "rmat", 8, n_sources=(65,), limits=(0, 2), knobs=t.OFFS64, store_transposed=True)
    t.check_rows(monkeypatch, "rmat_sym", 8, n_sources=(65,), limits=(0,), knobs=t.OFFS64, vertex_dtype=np.int64)


def test_inputs_emulated(surface, monkeypatch):
    t.check_inputs(monkeypatch, size=200)


def test_errors_and_extract_paths_emulated(surface, monkeypatch):
    t.check_errors(monkeypatch, size=200)


def test_api_emulated(surface):
    t.check_api(size=200)
