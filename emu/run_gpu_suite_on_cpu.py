"""Run the `-m gpu` test suite against the CPU emulation build of the library (tests/emu_py.py): the tests' Python logic
and the kernels' LOGIC at the test sizes, without a GPU.  Multi-GPU (NCCL) tests are left out; the RMAT-24 certificates
run at CUGRAPH_B200_FULL_SCALE (default here: 10).  Not a substitute for the GPU run — timing, memory ordering and
scheduling only exist there — but it finds everything else first.
    python emu/run_gpu_suite_on_cpu.py [pytest args]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUGRAPH_B200_FULL_SCALE", "10")

import pytest  # noqa: E402
from tests.emu_py import emulated_python_surface  # noqa: E402

with emulated_python_surface():
    sys.exit(pytest.main([os.path.join(ROOT, "tests"), "-q", "-m", "gpu", "--deselect", "tests/test_mg_gpu.py",
                          "--deselect", "tests/test_reference_c_tests_gpu.py",
                          "--deselect", "tests/test_zz_late_additions_gpu.py::test_reference_c_test_program_on_gpu",
                          # SCC at GPU sizes (RMAT-16/18, 10^5-vertex chains and cycles); tests/test_scc_cpu.py runs the same checks smaller
                          *[a for t in ("rmat", "rmat_scrambled_int64_and_renumber_false", "random_both_orientations", "offs64",
                                        "loops_multi_edges_and_wcc", "inputs", "phase_shapes") for a in ("--deselect", f"tests/test_scc_gpu.py::test_scc_{t}_gpu")],
                          "--deselect", "tests/test_scc_gpu.py::test_reference_scc_c_test_gpu",
                          # SSSP on every shape, weight family, cutoff and knob set (hundreds of traversals);
                          # tests/test_traversal_shapes_cpu.py runs the same checks on fewer cases
                          "--deselect", "tests/test_traversal_shapes_gpu.py::test_sssp_shapes",
                          # multi-GPU SCC at GPU sizes (RMAT-14/16 on four grids); tests/test_mg_scc_cpu.py runs the same checks smaller
                          *[a for t in ("simulated", "phases", "edge_cases", "offs64", "weighted_blocks")
                            for a in ("--deselect", f"tests/test_mg_scc_gpu.py::test_mg_scc_{t}_on_one_gpu")],
                          "-p", "no:cacheprovider"] + sys.argv[1:]))
