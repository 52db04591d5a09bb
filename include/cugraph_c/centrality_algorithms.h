/*
 * PageRank family + its result object.  Replaces cpp/include/cugraph_c/centrality_algorithms.h:
 * result accessors :37-75, cugraph_pagerank :114, cugraph_pagerank_allow_nonconvergence :169 (the
 * entry pylibcugraph.pagerank binds, pagerank.pyx:196-208), cugraph_personalized_pagerank :228,
 * cugraph_personalized_pagerank_allow_nonconvergence :285.
 *
 * Semantics preserved from cpp/src/link_analysis/pagerank_impl.cuh:224-329 and
 * cpp/src/c_api/pagerank.cpp:89-376: convergence test is sum|delta| < epsilon (not scaled by V),
 * checked after the iteration counter is incremented; converged == (iterations < max_iterations);
 * the non-"allow" entry points return CUGRAPH_UNKNOWN_ERROR "PageRank failed to converge.";
 * result rows are (external vertex id, score) ; an unweighted graph yields FLOAT32 scores.
 */
#pragma once
#include <cugraph_c/error.h>
#include <cugraph_c/export.h>
#include <cugraph_c/graph.h>
#include <cugraph_c/resource_handle.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int32_t align_; } cugraph_centrality_result_t;

CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_centrality_result_get_vertices(
  cugraph_centrality_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_centrality_result_get_values(
  cugraph_centrality_result_t* result);
CUGRAPH_EXPORT size_t cugraph_centrality_result_get_num_iterations(cugraph_centrality_result_t* result);
CUGRAPH_EXPORT bool_t cugraph_centrality_result_converged(cugraph_centrality_result_t* result);
CUGRAPH_EXPORT void cugraph_centrality_result_free(cugraph_centrality_result_t* result);

CUGRAPH_EXPORT cugraph_error_code_t cugraph_pagerank(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  double alpha, double epsilon, size_t max_iterations, bool_t do_expensive_check,
  cugraph_centrality_result_t** result, cugraph_error_t** error);

CUGRAPH_EXPORT cugraph_error_code_t cugraph_pagerank_allow_nonconvergence(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  double alpha, double epsilon, size_t max_iterations, bool_t do_expensive_check,
  cugraph_centrality_result_t** result, cugraph_error_t** error);

CUGRAPH_EXPORT cugraph_error_code_t cugraph_personalized_pagerank(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  const cugraph_type_erased_device_array_view_t* personalization_vertices,
  const cugraph_type_erased_device_array_view_t* personalization_values,
  double alpha, double epsilon, size_t max_iterations, bool_t do_expensive_check,
  cugraph_centrality_result_t** result, cugraph_error_t** error);

CUGRAPH_EXPORT cugraph_error_code_t cugraph_personalized_pagerank_allow_nonconvergence(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  const cugraph_type_erased_device_array_view_t* personalization_vertices,
  const cugraph_type_erased_device_array_view_t* personalization_values,
  double alpha, double epsilon, size_t max_iterations, bool_t do_expensive_check,
  cugraph_centrality_result_t** result, cugraph_error_t** error);

/* ---- sibling algorithms on the same primitive (SURVEY.md §8 f3) ----
 * Katz centrality: cpp/include/cugraph_c/centrality_algorithms.h:328-364, cpp/src/c_api/katz.cpp,
 * cpp/src/centrality/katz_centrality_impl.cuh:34-196.  x <- alpha * A^T x + beta until sum |x_new - x_old| < epsilon, then
 * divided by its L2 norm; `betas` is accepted and — as in the reference's C entry point — not used. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_katz_centrality(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, const cugraph_type_erased_device_array_view_t* betas,
  double alpha, double beta, double epsilon, size_t max_iterations, bool_t do_expensive_check,
  cugraph_centrality_result_t** result, cugraph_error_t** error);

/* Eigenvector centrality: centrality_algorithms.h:297-326, cpp/src/c_api/eigenvector_centrality.cpp,
 * cpp/src/centrality/eigenvector_centrality_impl.cuh:34-150.  x <- (A^T x + x) / ||.||_2 until sum |x_new - x_old| < V * epsilon. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_eigenvector_centrality(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, double epsilon, size_t max_iterations,
  bool_t do_expensive_check, cugraph_centrality_result_t** result, cugraph_error_t** error);

/* HITS: centrality_algorithms.h:488-591, cpp/src/c_api/hits.cpp, cpp/src/link_analysis/hits_impl.cuh:29-206. */
typedef struct { int32_t align_; } cugraph_hits_result_t;
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_vertices(cugraph_hits_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_hubs(cugraph_hits_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_authorities(cugraph_hits_result_t* result);
CUGRAPH_EXPORT double cugraph_hits_result_get_hub_score_differences(cugraph_hits_result_t* result);
CUGRAPH_EXPORT size_t cugraph_hits_result_get_number_of_iterations(cugraph_hits_result_t* result);
CUGRAPH_EXPORT void cugraph_hits_result_free(cugraph_hits_result_t* result);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_hits(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, double epsilon, size_t max_iterations,
  const cugraph_type_erased_device_array_view_t* initial_hubs_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_hubs_guess_values, bool_t normalize, bool_t do_expensive_check,
  cugraph_hits_result_t** result, cugraph_error_t** error);

/* Betweenness centrality: centrality_algorithms.h:366-486, cpp/src/c_api/betweenness_centrality.cpp,
 * cpp/src/centrality/betweenness_centrality_impl.cuh.  Brandes' algorithm over batches of up to 64 sources on the multi-source
 * BFS levels (betweenness.cu); shortest paths are counted by hops and edge weights are not used.  vertex_list == NULL: every
 * vertex is a source; else its vertices are the sources (cugraph_select_random_vertices draws such a list).  Values have the
 * graph's weight type (FLOAT32 on an unweighted graph), scaled as the reference scales them.  A source that is not a vertex
 * gives CUGRAPH_INVALID_INPUT. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_betweenness_centrality(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, const cugraph_type_erased_device_array_view_t* vertex_list,
  bool_t normalized, bool_t include_endpoints, bool_t do_expensive_check, cugraph_centrality_result_t** result,
  cugraph_error_t** error);

/* Edge betweenness: one value per edge of the graph, multi-edges each with their own.  Edge ids are not stored by this
 * library (graph creation validates and drops them), so get_edge_ids returns NULL, as the reference's result of a graph
 * created without edge ids holds none. */
typedef struct { int32_t align_; } cugraph_edge_centrality_result_t;
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_src_vertices(
  cugraph_edge_centrality_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_dst_vertices(
  cugraph_edge_centrality_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_edge_ids(
  cugraph_edge_centrality_result_t* result);
CUGRAPH_EXPORT cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_values(
  cugraph_edge_centrality_result_t* result);
CUGRAPH_EXPORT void cugraph_edge_centrality_result_free(cugraph_edge_centrality_result_t* result);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_edge_betweenness_centrality(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, const cugraph_type_erased_device_array_view_t* vertex_list,
  bool_t normalized, bool_t do_expensive_check, cugraph_edge_centrality_result_t** result, cugraph_error_t** error);

#ifdef __cplusplus
}
#endif
