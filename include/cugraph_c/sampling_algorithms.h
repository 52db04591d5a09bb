/*
 * Sampling (the reference's cpp/include/cugraph_c/sampling_algorithms.h): only cugraph_select_random_vertices, which
 * draws the sources of sampled betweenness centrality.  The two opaque types are declared because the reference's
 * prototypes of the other sampling entry points name them; those entry points are not provided.
 */
#pragma once
#include <cugraph_c/error.h>
#include <cugraph_c/export.h>
#include <cugraph_c/graph.h>
#include <cugraph_c/random.h>
#include <cugraph_c/resource_handle.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int32_t align_; } cugraph_sample_result_t;
typedef struct { int32_t align_; } cugraph_sampling_options_t;

/* num_vertices distinct vertices of the graph (external ids, the graph's vertex type), drawn uniformly without replacement:
 * every vertex gets a key from the state's counter-based stream and the vertices with the num_vertices smallest keys are
 * returned in ascending key order.  num_vertices == the number of vertices returns every vertex.  The stream is not the
 * reference's, so the drawn vertices differ from the reference's for the same seed. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_select_random_vertices(const cugraph_resource_handle_t* handle,
                                                                   const cugraph_graph_t* graph, cugraph_rng_state_t* rng_state,
                                                                   size_t num_vertices, cugraph_type_erased_device_array_t** vertices,
                                                                   cugraph_error_t** error);

#ifdef __cplusplus
}
#endif
