/* Labeling algorithms: weakly and strongly connected components.
 * Replaces cpp/include/cugraph_c/labeling_algorithms.h:20-95 (cpp/src/c_api/weakly_connected_components.cpp,
 * cpp/src/c_api/strongly_connected_components.cpp, cpp/src/c_api/labeling_result.cpp). */
#pragma once
#include <cugraph_c/array.h>
#include <cugraph_c/error.h>
#include <cugraph_c/export.h>
#include <cugraph_c/graph.h>
#include <cugraph_c/resource_handle.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int32_t align_; } cugraph_labeling_result_t;

CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_labeling_result_get_vertices(cugraph_labeling_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_labeling_result_get_labels(cugraph_labeling_result_t* result);
CUGRAPH_EXPORT void cugraph_labeling_result_free(cugraph_labeling_result_t* result);

/* Every vertex gets the label of its component (vertex dtype; two vertices share a label iff an undirected path joins them;
 * the label is the id of one vertex of the component).  The graph must be symmetric
 * (weakly_connected_components_impl.cuh:287-289). */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_weakly_connected_components(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, bool_t do_expensive_check,
  cugraph_labeling_result_t** result, cugraph_error_t** error);

/* Every vertex gets the label of its strongly connected component (vertex dtype; two vertices share a label iff each can
 * reach the other along directed edges; the label is the id of one vertex of the component).  Edge weights are ignored.
 * The graph must not be symmetric: use cugraph_weakly_connected_components there (strongly_connected_components_impl.cuh:
 * 2013-2015, CUGRAPH_UNKNOWN_ERROR). */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_strongly_connected_components(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, bool_t do_expensive_check,
  cugraph_labeling_result_t** result, cugraph_error_t** error);

#ifdef __cplusplus
}
#endif
