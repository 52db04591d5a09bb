"""ctypes binding of the C-ABI in include/cugraph_c/*.h (what the reference binds through Cython's
`cdef extern` in python/pylibcugraph/pylibcugraph/_cugraph_c/*.pxd)."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcugraph_c.so")

# cugraph_data_type_id_t (types.h)
INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, SIZE_T, BOOL = range(12)

# cugraph_error_code_t (error.h)
SUCCESS, UNKNOWN_ERROR, INVALID_HANDLE, ALLOC_ERROR, INVALID_INPUT, NOT_IMPLEMENTED, UNSUPPORTED_TYPE_COMBINATION = range(7)


class GraphPropertiesStruct(C.Structure):
    _fields_ = [("is_symmetric", C.c_int), ("is_multigraph", C.c_int)]


_lib = None


def _sig(fn, res, args):
    fn.restype = res
    fn.argtypes = args


def emulated():
    """True when the CPU emulation build of the library is loaded (tests/emu_py.py): test infrastructure only"""
    return os.path.basename(LIB_PATH).startswith("libcugraph_c_emu")


def lib():
    """Load libcugraph_c.so (fails loudly: there is no CPU fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -m cugraph_b200.build` "
            "(nvcc, sm_90a). cugraph_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, sz, i32, dbl = C.c_void_p, C.c_size_t, C.c_int, C.c_double
    pvp = C.POINTER(C.c_void_p)
    _sig(L.cugraph_error_message, C.c_char_p, [vp])
    _sig(L.cugraph_error_free, None, [vp])
    _sig(L.cugraph_create_resource_handle, vp, [vp])
    _sig(L.cugraph_free_resource_handle, None, [vp])
    _sig(L.cugraph_resource_handle_get_rank, i32, [vp])
    _sig(L.cugraph_resource_handle_get_comm_size, i32, [vp])
    _sig(L.cugraph_type_erased_device_array_create, i32, [vp, sz, i32, pvp, pvp])
    _sig(L.cugraph_type_erased_device_array_create_from_view, i32, [vp, vp, pvp, pvp])
    _sig(L.cugraph_type_erased_device_array_free, None, [vp])
    _sig(L.cugraph_type_erased_device_array_view, vp, [vp])
    _sig(L.cugraph_type_erased_device_array_view_as_type, i32, [vp, i32, pvp, pvp])
    _sig(L.cugraph_type_erased_device_array_view_create, vp, [vp, sz, i32])
    _sig(L.cugraph_type_erased_device_array_view_free, None, [vp])
    _sig(L.cugraph_type_erased_device_array_view_size, sz, [vp])
    _sig(L.cugraph_type_erased_device_array_view_type, i32, [vp])
    _sig(L.cugraph_type_erased_device_array_view_pointer, vp, [vp])
    _sig(L.cugraph_type_erased_host_array_create, i32, [vp, sz, i32, pvp, pvp])
    _sig(L.cugraph_type_erased_host_array_free, None, [vp])
    _sig(L.cugraph_type_erased_host_array_view, vp, [vp])
    _sig(L.cugraph_type_erased_host_array_view_create, vp, [vp, sz, i32])
    _sig(L.cugraph_type_erased_host_array_view_free, None, [vp])
    _sig(L.cugraph_type_erased_host_array_size, sz, [vp])
    _sig(L.cugraph_type_erased_host_array_type, i32, [vp])
    _sig(L.cugraph_type_erased_host_array_pointer, vp, [vp])
    _sig(L.cugraph_type_erased_host_array_view_copy, i32, [vp, vp, vp, pvp])
    _sig(L.cugraph_type_erased_device_array_view_copy_from_host, i32, [vp, vp, vp, pvp])
    _sig(L.cugraph_type_erased_device_array_view_copy_to_host, i32, [vp, vp, vp, pvp])
    _sig(L.cugraph_type_erased_device_array_view_copy, i32, [vp, vp, vp, pvp])
    gp = C.POINTER(GraphPropertiesStruct)
    _sig(L.cugraph_graph_create_sg, i32, [vp, gp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, pvp, pvp])
    _sig(L.cugraph_graph_create_with_times_sg, i32,
         [vp, gp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, pvp, pvp])
    _sig(L.cugraph_graph_create_sg_from_csr, i32, [vp, gp, vp, vp, vp, vp, vp, i32, i32, i32, i32, pvp, pvp])
    _sig(L.cugraph_graph_create_mg, i32, [vp, gp, pvp, pvp, pvp, pvp, pvp, pvp, i32, sz, i32, i32, i32, i32, pvp, pvp])
    _sig(L.cugraph_graph_create_with_times_mg, i32,
         [vp, gp, pvp, pvp, pvp, pvp, pvp, pvp, pvp, pvp, i32, sz, i32, i32, i32, i32, pvp, pvp])
    _sig(L.cugraph_graph_free, None, [vp])
    _sig(L.cugraph_centrality_result_get_vertices, vp, [vp])
    _sig(L.cugraph_centrality_result_get_values, vp, [vp])
    _sig(L.cugraph_centrality_result_get_num_iterations, sz, [vp])
    _sig(L.cugraph_centrality_result_converged, i32, [vp])
    _sig(L.cugraph_centrality_result_free, None, [vp])
    pr = [vp, vp, vp, vp, vp, vp, dbl, dbl, sz, i32, pvp, pvp]
    ppr = [vp, vp, vp, vp, vp, vp, vp, vp, dbl, dbl, sz, i32, pvp, pvp]
    _sig(L.cugraph_pagerank, i32, pr)
    _sig(L.cugraph_pagerank_allow_nonconvergence, i32, pr)
    _sig(L.cugraph_personalized_pagerank, i32, ppr)
    _sig(L.cugraph_personalized_pagerank_allow_nonconvergence, i32, ppr)
    _sig(L.cugraph_paths_result_get_vertices, vp, [vp])
    _sig(L.cugraph_paths_result_get_distances, vp, [vp])
    _sig(L.cugraph_paths_result_get_predecessors, vp, [vp])
    _sig(L.cugraph_paths_result_free, None, [vp])
    _sig(L.cugraph_bfs, i32, [vp, vp, vp, i32, sz, i32, i32, pvp, pvp])
    _sig(L.cugraph_b200_multi_source_bfs, i32, [vp, vp, vp, sz, i32, pvp, pvp])
    _sig(L.cugraph_sssp, i32, [vp, vp, sz, dbl, i32, i32, pvp, pvp])
    _sig(L.cugraph_extract_paths, i32, [vp, vp, vp, vp, vp, pvp, pvp])
    _sig(L.cugraph_extract_paths_result_get_max_path_length, sz, [vp])
    _sig(L.cugraph_extract_paths_result_get_paths, vp, [vp])
    _sig(L.cugraph_extract_paths_result_free, None, [vp])
    for f in ("cugraph_in_degrees", "cugraph_out_degrees", "cugraph_degrees"):
        _sig(getattr(L, f), i32, [vp, vp, vp, i32, pvp, pvp])
    for f in ("vertices", "in_degrees", "out_degrees"):
        _sig(getattr(L, f"cugraph_degrees_result_get_{f}"), vp, [vp])
    _sig(L.cugraph_degrees_result_free, None, [vp])
    _sig(L.cugraph_katz_centrality, i32, [vp, vp, vp, dbl, dbl, dbl, sz, i32, pvp, pvp])
    _sig(L.cugraph_eigenvector_centrality, i32, [vp, vp, dbl, sz, i32, pvp, pvp])
    _sig(L.cugraph_hits, i32, [vp, vp, dbl, sz, vp, vp, i32, i32, pvp, pvp])
    for f in ("vertices", "hubs", "authorities"):
        _sig(getattr(L, f"cugraph_hits_result_get_{f}"), vp, [vp])
    _sig(L.cugraph_hits_result_get_hub_score_differences, dbl, [vp])
    _sig(L.cugraph_hits_result_get_number_of_iterations, sz, [vp])
    _sig(L.cugraph_hits_result_free, None, [vp])
    _sig(L.cugraph_weakly_connected_components, i32, [vp, vp, i32, pvp, pvp])
    _sig(L.cugraph_strongly_connected_components, i32, [vp, vp, i32, pvp, pvp])
    _sig(L.cugraph_labeling_result_get_vertices, vp, [vp])
    _sig(L.cugraph_labeling_result_get_labels, vp, [vp])
    _sig(L.cugraph_labeling_result_free, None, [vp])
    # extensions (b200_ext.h)
    _sig(L.cugraph_b200_version, C.c_char_p, [])
    _sig(L.cugraph_b200_handle_stream, vp, [vp])
    _sig(L.cugraph_b200_handle_launch_count, sz, [vp])
    _sig(L.cugraph_b200_time_pull_spmv, i32, [vp, vp, sz, C.POINTER(dbl), C.POINTER(dbl), pvp])
    _sig(L.cugraph_b200_create_resource_handle_on_stream, vp, [vp])
    _sig(L.cugraph_b200_padded_elems, sz, [sz, sz])
    _sig(L.cugraph_b200_block_create, i32, [vp, sz, sz, vp, vp, vp, pvp, pvp])
    _sig(L.cugraph_b200_block_stage_edges, i32, [vp, sz, sz, vp, vp, vp, vp, i32, i32, C.POINTER(sz), pvp])
    _sig(L.cugraph_b200_block_degrees, i32, [vp, vp, vp, vp, pvp])
    _sig(L.cugraph_b200_block_free, None, [vp])
    _sig(L.cugraph_b200_block_span, sz, [vp])
    _sig(L.cugraph_b200_block_pull_sweep, i32, [vp, vp, vp, vp, dbl, pvp])
    _sig(L.cugraph_b200_generate_rmat_edgelist, i32, [vp, sz, sz, dbl, dbl, dbl, C.c_uint64, i32, i32, vp, vp, pvp])
    _sig(L.cugraph_b200_generate_uniform, i32, [vp, C.c_uint64, dbl, dbl, vp, pvp])
    _sig(L.cugraph_b200_generate_rmat_edgelist_at, i32,
         [vp, sz, C.c_uint64, sz, dbl, dbl, dbl, C.c_uint64, i32, i32, vp, vp, pvp])
    _sig(L.cugraph_b200_generate_uniform_at, i32, [vp, C.c_uint64, C.c_uint64, dbl, dbl, vp, pvp])
    _sig(L.cugraph_b200_block_bfs_pull, i32, [vp, vp, vp, vp, sz, i32, i32, vp, pvp])
    _sig(L.cugraph_b200_block_bfs_push, i32, [vp, vp, vp, vp, sz, i32, i32, vp, pvp])
    _sig(L.cugraph_b200_bfs_bottom_up, i32, [vp, i32, sz, sz, sz, sz, sz])
    _sig(L.cugraph_b200_block_ms_bfs_push, i32, [vp, vp, vp, vp, i32, vp, pvp])
    _sig(L.cugraph_b200_block_ms_bfs_pull, i32, [vp, vp, vp, vp, i32, vp, pvp])
    _sig(L.cugraph_b200_block_ms_bfs_pred, i32, [vp, vp, vp, vp, sz, i32, i32, sz, vp, pvp])
    _sig(L.cugraph_b200_ms_bfs_owner_step, i32, [vp, vp, i32, sz, sz, i32, i32, vp, vp, vp, vp, vp, vp, pvp])
    _sig(L.cugraph_b200_ms_bfs_owner_pred, i32, [vp, vp, vp, sz, i32, vp, pvp])
    _sig(L.cugraph_b200_block_sssp_relax, i32, [vp, vp, vp, dbl, sz, i32, i32, vp, pvp])
    _sig(L.cugraph_b200_block_sssp_pred, i32, [vp, vp, vp, vp, sz, i32, i32, vp, pvp])
    _sig(L.cugraph_b200_block_wcc_min, i32, [vp, vp, vp, vp, pvp])
    _sig(L.cugraph_b200_block_check_paths, i32, [vp, vp, vp, vp, vp, dbl, sz, i32, i32, vp, vp, C.POINTER(C.c_uint64), pvp])
    _sig(L.cugraph_b200_block_scc_push, i32, [vp, vp, i32, i32, vp, vp, vp, sz, i32, i32, i32, i32, vp, pvp])
    _sig(L.cugraph_b200_paths_answer, i32, [vp, vp, vp, vp, sz, vp, pvp])
    _sig(L.cugraph_b200_paths_advance, i32, [vp, vp, vp, vp, vp, sz, sz, i32, vp, vp, vp, vp, pvp])
    _sig(L.cugraph_b200_pagerank_vertex_step, i32, [vp, vp, vp, vp, vp, sz, dbl, dbl, i32, vp, vp, pvp])
    _sig(L.cugraph_b200_pagerank_personalized_vertex_step, i32, [vp, vp, vp, vp, vp, vp, sz, dbl, dbl, i32, vp, vp, pvp])
    _sig(L.cugraph_b200_block_sweep, i32, [vp, vp, i32, i32, vp, vp, dbl, pvp])
    _sig(L.cugraph_b200_katz_step, i32, [vp, vp, vp, sz, dbl, vp, pvp])
    _sig(L.cugraph_b200_eigenvector_add_step, i32, [vp, vp, vp, sz, vp, pvp])
    _sig(L.cugraph_b200_eigenvector_scale_step, i32, [vp, vp, vp, sz, vp, vp, pvp])
    _sig(L.cugraph_b200_hits_max_step, i32, [vp, vp, vp, sz, vp, pvp])
    _sig(L.cugraph_b200_hits_scale_step, i32, [vp, vp, vp, vp, sz, vp, vp, pvp])
    _sig(L.cugraph_b200_vertex_sum, i32, [vp, vp, sz, i32, vp, pvp])
    _sig(L.cugraph_b200_vertex_scale, i32, [vp, vp, sz, dbl, pvp])
    _lib = L
    return L


class CugraphError(Exception):
    """Base of the errors raised for a non-success C return code.  `code` is the cugraph_error_code_t; the concrete class
    also derives from the builtin exception the reference raises for that code (utils.pyx:40-83), so callers written
    against the reference (`except ValueError`, `pytest.raises(RuntimeError)`) keep working."""

    def __init__(self, code, message, where):
        self.code = code
        super().__init__(f"non-success value returned from {where}: {_CODE_NAMES.get(code, 'unknown error code')} {message}")


class CugraphRuntimeError(CugraphError, RuntimeError):
    pass


class CugraphValueError(CugraphError, ValueError):
    pass


class CugraphMemoryError(CugraphError, MemoryError):
    pass


class CugraphNotImplementedError(CugraphError, NotImplementedError):
    pass


_CODE_NAMES = {UNKNOWN_ERROR: "CUGRAPH_UNKNOWN_ERROR", INVALID_HANDLE: "CUGRAPH_INVALID_HANDLE", ALLOC_ERROR: "CUGRAPH_ALLOC_ERROR",
               INVALID_INPUT: "CUGRAPH_INVALID_INPUT", NOT_IMPLEMENTED: "CUGRAPH_NOT_IMPLEMENTED",
               UNSUPPORTED_TYPE_COMBINATION: "CUGRAPH_UNSUPPORTED_TYPE_COMBINATION"}
_CODE_CLASS = {UNKNOWN_ERROR: CugraphRuntimeError, INVALID_HANDLE: CugraphValueError, ALLOC_ERROR: CugraphMemoryError,
               INVALID_INPUT: CugraphValueError, NOT_IMPLEMENTED: CugraphNotImplementedError,
               UNSUPPORTED_TYPE_COMBINATION: CugraphValueError}


def check(code, err_ptr, where):
    """assert_success of python/pylibcugraph/pylibcugraph/utils.pyx:40-83: same exception type per error code."""
    if code == SUCCESS:
        return
    msg = ""
    if err_ptr and err_ptr.value:
        m = lib().cugraph_error_message(err_ptr)
        msg = m.decode() if m else ""
        lib().cugraph_error_free(err_ptr)
    raise _CODE_CLASS.get(code, CugraphRuntimeError)(code, msg, where)
