/*
 * Random number generator state (the reference's cpp/include/cugraph_c/random.h).  The state is a seed and a counter:
 * every draw (cugraph_select_random_vertices) reads the counter-based stream from the counter on and advances it, so
 * two states created with the same seed draw the same sequence of results.
 */
#pragma once
#include <cugraph_c/error.h>
#include <cugraph_c/export.h>
#include <cugraph_c/resource_handle.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int32_t align_; } cugraph_rng_state_t;

CUGRAPH_EXPORT cugraph_error_code_t cugraph_rng_state_create(const cugraph_resource_handle_t* handle, uint64_t seed,
                                                             cugraph_rng_state_t** state, cugraph_error_t** error);
CUGRAPH_EXPORT void cugraph_rng_state_free(cugraph_rng_state_t* p);

#ifdef __cplusplus
}
#endif
