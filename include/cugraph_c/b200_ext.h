/*
 * Extensions that have no counterpart in the reference ABI (prefixed cugraph_b200_).
 *
 *  - multi-GPU: the reference receives NCCL communicators inside a raft::handle_t built by raft-dask / MPI
 *    (python/pylibcugraph/pylibcugraph/comms/comms_wrapper.pyx:10-32, cpp/tests/utilities/mg_utilities.cpp:37-55) and keeps
 *    the 2D-partitioned blocks inside graph_t.  raft is not part of this build: cugraph_graph_create_mg and the multi-GPU
 *    algorithm entry points return CUGRAPH_NOT_IMPLEMENTED; multi-GPU PageRank, BFS, extract_paths, SSSP, WCC, SCC, Katz,
 *    eigenvector centrality and HITS are driven by the launcher (cugraph_b200/mg.py, one process per GPU over torch.distributed / NCCL) on top of
 *    the cugraph_b200_block_* and owner-step device pieces declared below.
 *  - profiling hooks used by bench.py to time the dominant kernel on the handle's stream.
 */
#pragma once
#include <cugraph_c/algorithms.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Library version string and the CUDA stream of a handle (as an integer, for event timing). */
CUGRAPH_EXPORT const char* cugraph_b200_version(void);
CUGRAPH_EXPORT void* cugraph_b200_handle_stream(const cugraph_resource_handle_t* handle);

/* Number of kernels this library launched through the handle since it was created. */
CUGRAPH_EXPORT size_t cugraph_b200_handle_launch_count(const cugraph_resource_handle_t* handle);

/*
 * Benchmark hook: run `iterations` pull-SpMV sweeps (the PageRank inner kernel set, no vertex pass)
 * on the graph's pull orientation and return the average time of ONE sweep in milliseconds,
 * measured with CUDA events on the handle's stream.  x is refreshed from a fixed vector; results
 * are written to an internal buffer.  Used for roofline.achieved in bench.py.
 */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_time_pull_spmv(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, size_t iterations,
  double* ms_per_sweep, double* algorithmic_bytes_per_sweep, cugraph_error_t** error);

/*
 * ---- multi-GPU building blocks (orchestrated by cugraph_b200/mg.py over torch.distributed) ----
 * The reference keeps its 2D-partitioned edge blocks inside graph_t and runs the exchange inside the
 * prims (update_edge_src_property / per_v_transform_reduce_e MG paths).  Here the launcher owns the
 * process groups; the library provides the device pieces.  Every call below only enqueues work on
 * the handle's stream (create the handle on the caller's stream so that collectives and kernels
 * are ordered without host synchronisation).
 */
typedef struct { int32_t align_; } cugraph_b200_block_t;

CUGRAPH_EXPORT cugraph_resource_handle_t* cugraph_b200_create_resource_handle_on_stream(void* cuda_stream);
CUGRAPH_EXPORT size_t cugraph_b200_padded_elems(size_t n, size_t elem_size);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_create(
  const cugraph_resource_handle_t* handle, size_t n_rows, size_t n_cols,
  const cugraph_type_erased_device_array_view_t* rows, const cugraph_type_erased_device_array_view_t* cols,
  const cugraph_type_erased_device_array_view_t* weights, cugraph_b200_block_t** block, cugraph_error_t** error);
/* Staging of this GPU's share of a multi-GPU edge list before cugraph_b200_block_create: the rules of single-GPU staging
 * (drop_multi_edges, symmetrize of cugraph_graph_create_sg) applied to the n edges (rows[i], cols[i]) in the block's slot
 * coordinates, rows[i] < n_rows and cols[i] < n_cols (else CUGRAPH_INVALID_INPUT), with optional FLOAT32 / FLOAT64 weights.
 *   drop_multi_edges: one edge per (row, col, reversed flag) is kept, the one of MINIMUM weight.
 *   symmetrize: reversed (one byte per edge, nonzero = a reversed copy; NULL = none) marks the copies u -> v of edges v -> u
 *   that the caller has shuffled to the position (row = v, col = u) of the original u -> v (none for a self-loop).  Per
 *   position, the i-th lightest original is paired with the i-th lightest reversed copy and becomes one edge of weight
 *   (W)((a + b) / 2); unpaired edges keep their weight.  Only this position's orientation is emitted: the position of the
 *   reversed pair sees the same group from the other side and emits the other one, with a bit-identical weight.  Without
 *   symmetrize the flags are ignored.
 * The staged edges are written in place into the first *n_out entries of rows, cols and weights (*n_out <= n), ordered by
 * (row, col).  Symmetrize needs 2n < 2^31 (single-GPU staging's bound, kept although this pass has no 32-bit output
 * positions), weights n < 2^32 (32-bit permutations).  Synchronises the handle's stream. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_stage_edges(
  const cugraph_resource_handle_t* handle, size_t n_rows, size_t n_cols, cugraph_type_erased_device_array_view_t* rows,
  cugraph_type_erased_device_array_view_t* cols, const cugraph_type_erased_device_array_view_t* reversed,
  cugraph_type_erased_device_array_view_t* weights, bool_t drop_multi_edges, bool_t symmetrize, size_t* n_out,
  cugraph_error_t** error);
/* The block's edge counts: row_counts[row slot] (INT64, at least n_rows) = the edges of that row, col_counts[column slot]
 * (INT64, at least n_cols) = the edges of that column; the first n_rows / n_cols entries are overwritten.  Summed over the
 * row group (rows) and the column group (columns) they are the in- and out-degrees of the owned vertices.  Asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_degrees(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, cugraph_type_erased_device_array_view_t* row_counts,
  cugraph_type_erased_device_array_view_t* col_counts, cugraph_error_t** error);
CUGRAPH_EXPORT void cugraph_b200_block_free(cugraph_b200_block_t* block);
CUGRAPH_EXPORT size_t cugraph_b200_block_span(const cugraph_b200_block_t* block);
/* y[row] = alpha * sum over the block's edges (row, col) of x[col] * w; rows without edges get 0.  The FIRST sweep of a block
 * into a given y array writes every row slot; later sweeps into the same array may rewrite only the rows that have edges (in a
 * 2D block most row slots are empty) — the caller must leave the other entries alone, or pass a zero-initialised array.
 * x holds cugraph_b200_padded_elems(span) elements: x[col] for the columns, ZERO from index `span` on (whole slices of x are
 * copied, and padding entries read a column at or behind the span); a column that no edge reads may hold anything, NaN
 * included.  x and y must not overlap: rows are written band by band while later bands still read x. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_pull_sweep(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* x, cugraph_type_erased_device_array_view_t* y, double alpha,
  cugraph_error_t** error);
/* The block sweep in either orientation.  transposed = FALSE, use_weights = TRUE is cugraph_b200_block_pull_sweep.
 * transposed = TRUE: y[col] = alpha * sum over the block's edges (row, col) of x[row] * w for every column slot; x is indexed by
 * row slot.  use_weights = FALSE sums plain neighbour values (w = 1) on a weighted block.  The rules of
 * cugraph_b200_block_pull_sweep hold for both orientations: x holds cugraph_b200_padded_elems(span) elements, zero from
 * `span` on, anything (NaN included) where no edge reads; y holds `span` elements; x and y do not overlap; the first sweep
 * of an orientation into a given y writes every slot, later sweeps of that orientation into the same y only the slots that
 * have edges (the two orientations keep this state apart; a sweep into an array the other orientation last swept writes it
 * whole again).  The transposed sweep runs the same kernels over the block's column-major copy; the first transposed call
 * on a block builds that copy (shared with cugraph_b200_block_sssp_relax / _wcc_min) when no earlier call did, together with
 * its sweep layout and accumulators, and synchronises once.  Otherwise asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_sweep(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, bool_t transposed, bool_t use_weights,
  const cugraph_type_erased_device_array_view_t* x, cugraph_type_erased_device_array_view_t* y, double alpha,
  cugraph_error_t** error);
/* Owner steps of multi-GPU Katz, eigenvector centrality and HITS (the launcher cugraph_b200/mg.py runs them between its
 * collectives).  Each passes once over this rank's first n_local elements, which all arrays must hold, and ADDS its fp64
 * partials into the caller's device doubles (max partials are merged with an atomic max), to be all-reduced by the launcher.
 * All arrays share one FLOAT32 / FLOAT64 type.  The arithmetic is that of the single-GPU cugraph_katz_centrality /
 * _eigenvector_centrality / cugraph_hits: scaling as (T)((double)v * inv), differences and norms in fp64.  Asynchronous.
 *   katz_step:              x_new = (T)(y + beta); partial[0] += sum |x_new - x|, partial[1] += sum x_new^2; x = x_new.
 *   eigenvector_add_step:   y += x; partial[0] += sum y^2.
 *   eigenvector_scale_step: y = y / sqrt(sumsq[0]) (sumsq: the all-reduced sum of the add step, read on the device);
 *                           partial[0] += sum |y - x|; x = y.
 *   hits_max_step:          max_out[0] = max(max_out[0], max hubs), max_out[1] = max(max_out[1], max authorities); the values
 *                           must be non-negative and max_out starts at 0.
 *   hits_scale_step:        hubs /= max[0], authorities /= max[1] (the all-reduced maxima, read on the device);
 *                           partial[0] += sum |hubs - prev_hubs|.
 *   vertex_sum:             partial[0] += sum v^2 (squares = TRUE) or sum v.
 *   vertex_scale:           v = (T)(v * inv). */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_katz_step(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* y,
  cugraph_type_erased_device_array_view_t* x, size_t n_local, double beta, double* partial_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_eigenvector_add_step(
  const cugraph_resource_handle_t* handle, cugraph_type_erased_device_array_view_t* y,
  const cugraph_type_erased_device_array_view_t* x, size_t n_local, double* partial_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_eigenvector_scale_step(
  const cugraph_resource_handle_t* handle, cugraph_type_erased_device_array_view_t* y,
  cugraph_type_erased_device_array_view_t* x, size_t n_local, const double* sumsq_device, double* partial_out_device,
  cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_hits_max_step(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* hubs,
  const cugraph_type_erased_device_array_view_t* authorities, size_t n_local, double* max_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_hits_scale_step(
  const cugraph_resource_handle_t* handle, cugraph_type_erased_device_array_view_t* hubs,
  cugraph_type_erased_device_array_view_t* authorities, const cugraph_type_erased_device_array_view_t* prev_hubs,
  size_t n_local, const double* max_device, double* partial_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_vertex_sum(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* v, size_t n_local, bool_t squares,
  double* partial_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_vertex_scale(
  const cugraph_resource_handle_t* handle, cugraph_type_erased_device_array_view_t* v, size_t n_local, double inv,
  cugraph_error_t** error);
/* Owner step of one multi-GPU PageRank iteration over this rank's first n_local vertices (y: the reduce-scattered sweep
 * output, alpha applied; pr: the ranks, updated in place; out_w: out-weight sums, 0 = dangling; x: pr / out_w for the next
 * sweep, pr where out_w is 0).  All arrays share one FLOAT32 / FLOAT64 type and hold at least n_local elements.  With
 * base = totals_prev[1] * alpha + 1 - alpha (totals_prev: the all-reduced partials of the previous step, read on the device):
 *   pagerank_vertex_step:              pr = (T)(y + base / n_vertices_global)
 *   pagerank_personalized_vertex_step: pr = (T)(y + base * ((double)pers / pers_sum)), pers dense over the owned slice
 *                                      (0 for the vertices not personalized), pers_sum > 0 the global sum of its values —
 *                                      the single-GPU personalized rule (cugraph_personalized_pagerank), divided in fp64.
 * first = TRUE keeps pr as it is and reads no totals_prev (the prologue that derives x and the dangling sum of the start
 * vector).  Both then ADD partial_out[0] += sum |pr_new - pr_old| and partial_out[1] += sum of pr_new over the dangling
 * vertices, to be all-reduced by the launcher.  n_local = 0 is a no-op.  Asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_pagerank_vertex_step(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* y,
  cugraph_type_erased_device_array_view_t* pr, const cugraph_type_erased_device_array_view_t* out_w,
  cugraph_type_erased_device_array_view_t* x, size_t n_local, double alpha, double n_vertices_global, bool_t first,
  const double* totals_prev_device, double* partial_out_device, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_pagerank_personalized_vertex_step(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* y,
  cugraph_type_erased_device_array_view_t* pr, const cugraph_type_erased_device_array_view_t* out_w,
  cugraph_type_erased_device_array_view_t* x, const cugraph_type_erased_device_array_view_t* pers, size_t n_local,
  double alpha, double pers_sum, bool_t first, const double* totals_prev_device, double* partial_out_device,
  cugraph_error_t** error);

/* RMAT edge list written into caller-allocated INT32 arrays (the role of cugraph_generate_rmat_edgelist,
 * cpp/include/cugraph_c/graph_generators.h, without its rng_state / coo objects): the reference's sampling rule, clip-and-flip
 * and id scramble (generate_rmat_edgelist.cuh:66-108, scramble.cuh:44-67) over a counter-based uniform stream, so that
 * the same (scale, seed) gives the same edges on any grid size — restated in numpy by oracle/rmat.py for the parity test. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_generate_rmat_edgelist(
  const cugraph_resource_handle_t* handle, size_t scale, size_t num_edges, double a, double b, double c, uint64_t seed,
  bool_t clip_and_flip, bool_t scramble_vertex_ids, cugraph_type_erased_device_array_view_t* src,
  cugraph_type_erased_device_array_view_t* dst, cugraph_error_t** error);

/* Uniform values for synthetic edge weights / types (what cugraph_generate_edge_weights / _edge_types draw from raft's RNG):
 * out[i] = lo + u_i * (hi - lo), u_i from a 64-bit mix of (seed, i); INT32 arrays get integers in [lo, hi). */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_generate_uniform(const cugraph_resource_handle_t* handle, uint64_t seed, double lo,
                                                                  double hi, cugraph_type_erased_device_array_view_t* out,
                                                                  cugraph_error_t** error);

/* Slices of the same two streams.  Both are counter-based (edge e draws from mix64(seed ^ (64 e + bit)), value i from
 * mix64(seed ^ i)), so edges [first_edge, first_edge + num_edges) of the RMAT stream, and values [first, first + size(out))
 * of the uniform stream, are written to elements 0, 1, ... of the arrays: the concatenation of consecutive slices is the
 * output of one call over their union, bit for bit.  cugraph_b200_generate_rmat_edgelist / _uniform are the slices at 0;
 * arguments and checks are theirs. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_generate_rmat_edgelist_at(
  const cugraph_resource_handle_t* handle, size_t scale, uint64_t first_edge, size_t num_edges, double a, double b, double c,
  uint64_t seed, bool_t clip_and_flip, bool_t scramble_vertex_ids, cugraph_type_erased_device_array_view_t* src,
  cugraph_type_erased_device_array_view_t* dst, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_generate_uniform_at(const cugraph_resource_handle_t* handle, uint64_t seed,
                                                                     uint64_t first, double lo, double hi,
                                                                     cugraph_type_erased_device_array_view_t* out,
                                                                     cugraph_error_t** error);

/* Breadth-first search from each of the n sources separately (not from their union, as cugraph_bfs does).  The result's
   distances and predecessors hold n x V entries, source-major: entry s*V + i belongs to sources[s] and to vertices[i].
   Row s equals what cugraph_bfs returns for the single source sources[s] with the same depth_limit: the distances in the
   graph's vertex type (INT32_MAX / INT64_MAX unreached), predecessors in external ids (-1 for the source and unreached
   vertices), a parent being any in-neighbour one level closer.  Out-edges are followed on any graph, symmetric or not;
   weights are ignored.  compute_predecessors = FALSE: predecessors has size 0.  Duplicate sources give identical rows.
   The sources run in batches of 64, each one pass over the graph per level, in either direction (Beamer's rule with
   CUGRAPH_B200_BFS_ALPHA / _BETA; the result does not depend on it).  cugraph_extract_paths accepts a result of one row
   only.  Errors as cugraph_bfs: NULL result or sources, a source type that is not the graph's, a source that is not a
   vertex (CUGRAPH_INVALID_INPUT). */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_multi_source_bfs(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* sources, size_t depth_limit, bool_t compute_predecessors,
  cugraph_paths_result_t** result, cugraph_error_t** error);

/* One level of multi-GPU BFS on this GPU's edge block (pull direction; the role of the bottom-up step of
 * cpp/src/traversal/bfs_impl.cuh:593-869 on one edge partition).  frontier_cols / visited_rows: byte flags over the block's
 * column (source) / row (destination) slots, gathered by the launcher inside the column / row group.  cand (INT64, one per row
 * slot) receives, for every unvisited row with a source in the frontier, that source's global code
 * ((col / maxpart) * grid_cols + grid_c) * maxpart + col % maxpart  (= owner rank * maxpart + local id), else -1. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_bfs_pull(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* frontier_cols, const cugraph_type_erased_device_array_view_t* visited_rows,
  size_t maxpart, int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* cand, cugraph_error_t** error);

/* The same level in the push direction (the role of the top-down step of cpp/src/traversal/bfs_impl.cuh on one edge
 * partition).  Same arguments and the same checks as cugraph_b200_block_bfs_pull.  cand is first filled with -1; then the
 * frontier columns are queued through the block's column-major copy (shared with cugraph_b200_block_sssp_relax / _wcc_min /
 * _scc_push / the transposed sweep, built by the first of these calls on the block and kept), and every edge (row, col) of a
 * frontier column into an unvisited row raises cand[row] to col's global code (atomic max).  cand[row] is therefore the
 * LARGEST code among the row's frontier sources, whatever order the edges are visited in.  Asynchronous, apart from one
 * read-back of the number of frontier columns and their edge count. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_bfs_push(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* frontier_cols, const cugraph_type_erased_device_array_view_t* visited_rows,
  size_t maxpart, int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* cand, cugraph_error_t** error);

/* The direction of one level of a direction-optimising BFS (Beamer's rule, as single-GPU cugraph_bfs decides it, with the
 * handle's CUGRAPH_B200_BFS_ALPHA / _BETA), given the direction of the last level (bottom_up_now):
 *   top-down -> bottom-up when m_f * alpha > m_u and n_f >= prev_n_f;
 *   bottom-up -> top-down when n_f * beta < n_unvisited and n_f < prev_n_f;
 *   otherwise the direction stays.
 * n_f, m_f: vertices and out-edges of the current frontier; prev_n_f: vertices of the previous frontier (0 at the first
 * level); m_u: edges into the unvisited vertices; n_unvisited: vertices not visited yet.  Returns TRUE for bottom-up.  A NULL
 * handle returns bottom_up_now.  Host only, no device work. */
CUGRAPH_EXPORT bool_t cugraph_b200_bfs_bottom_up(const cugraph_resource_handle_t* handle, bool_t bottom_up_now, size_t n_f,
                                                 size_t prev_n_f, size_t m_f, size_t m_u, size_t n_unvisited);

/* One level of a multi-GPU multi-source BFS batch on this GPU's edge block (MGGraph.multi_source_bfs).  Bit j of a 64-bit word
 * stands for source j of a batch of n_sources (1 to 64).  cur_cols (INT64, one word per column slot, gathered by the launcher
 * inside the column group): the sources that reached each column at this level.  seen_rows (INT64, one per row slot,
 * gathered inside the row group): the sources that have reached each row.  next_rows (INT64, one per row slot) is first
 * zeroed, then receives for every row slot the OR of cur_cols[col] & ~seen_rows[row] over the row's columns, limited to the
 * batch's bits; the launcher ORs the row group's words at the owners.  No distance is written here.
 *   _push queues the columns with a non-zero word through the block's column-major copy (shared with
 *     cugraph_b200_block_bfs_push and the others, built by the first of these calls and kept) and ORs each edge's bits with
 *     an atomic.  Asynchronous, apart from one read-back of the number of such columns and their edge count.
 *   _pull scans every row slot that still wants a bit over its own columns, and stops once it has them all (a warp per row of
 *     degree >= 32, a thread per other row).  Asynchronous.
 * Both take the same arguments, with the same checks: INT64 arrays no shorter than the block's slots, n_sources in [1, 64]. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_ms_bfs_push(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, const cugraph_type_erased_device_array_view_t* cur_cols,
  const cugraph_type_erased_device_array_view_t* seen_rows, int n_sources, cugraph_type_erased_device_array_view_t* next_rows,
  cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_ms_bfs_pull(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, const cugraph_type_erased_device_array_view_t* cur_cols,
  const cugraph_type_erased_device_array_view_t* seen_rows, int n_sources, cugraph_type_erased_device_array_view_t* next_rows,
  cugraph_error_t** error);

/* The predecessors of a level of a multi-source BFS batch on this GPU's edge block.  cur_cols: the level's frontier words, as
 * given to the level step; new_rows (INT64, one per row slot, gathered inside the row group): the bits the owners accepted at
 * this level.  For every row slot with new bits b and every bit j of b, the entry of (row, j) receives the largest code
 * ((col / maxpart) * grid_cols + grid_c) * maxpart + col % maxpart over the row's columns with bit j in cur_cols[col], or -1
 * when this block has none.  The entries are laid out as grid_cols owner segments of seg entries (pairs: INT64, at least
 * grid_cols * seg, filled with -1 first): row slot r lies in segment k = r / maxpart, and (r, j) sits at
 * k * seg + (the new bits of the row slots k * maxpart .. r - 1) + (the bits of b below j).  seg must be at least the new
 * bits of every segment; entries past it are dropped.  A MAX reduce-scatter of pairs in the row group then gives every owner
 * its own segment.  The block must have at most grid_cols * maxpart row slots.  Asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_ms_bfs_pred(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, const cugraph_type_erased_device_array_view_t* cur_cols,
  const cugraph_type_erased_device_array_view_t* new_rows, size_t maxpart, int grid_cols, int grid_c, size_t seg,
  cugraph_type_erased_device_array_view_t* pairs, cugraph_error_t** error);

/* The owners' update of one level of a multi-source BFS batch, over the n_local owned slots.  recv (INT64, parts * maxpart
 * words): the row group's partial next words for the owned slots, one slice of maxpart per member.  For every owned slot v:
 * new = (OR of the parts slices at v) & ~seen[v] (batch bits only), seen[v] |= new, cur[v] = new, and
 * distances[j * n_local + v] = level (INT32) for every bit j of new.  counts (INT64, 5 entries, overwritten) = the slots with
 * new bits, their deg_out sum, the slots whose seen word became the whole batch, their deg_in sum, and the new bits in all.
 * deg_out / deg_in (INT64, n_local entries) may both be NULL: their sums are then 0.  Asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_ms_bfs_owner_step(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* recv, int parts, size_t maxpart,
  size_t n_local, int n_sources, int level, cugraph_type_erased_device_array_view_t* seen,
  cugraph_type_erased_device_array_view_t* cur, cugraph_type_erased_device_array_view_t* distances,
  const cugraph_type_erased_device_array_view_t* deg_out, const cugraph_type_erased_device_array_view_t* deg_in,
  cugraph_type_erased_device_array_view_t* counts, cugraph_error_t** error);

/* The owners' side of the predecessor step: new_words (INT64, n_local) are the level's new bits, pairs (INT64) the owner's
 * segment of cugraph_b200_block_ms_bfs_pred's buffer after the MAX reduce-scatter.  predecessors[j * n_local + v] (INT64)
 * = the entry of (v, j) for every bit j of new_words[v], at (the new bits of the slots before v) + (the bits below j);
 * entries past the end of pairs are skipped.  Asynchronous. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_ms_bfs_owner_pred(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* new_words,
  const cugraph_type_erased_device_array_view_t* pairs, size_t n_local, int n_sources,
  cugraph_type_erased_device_array_view_t* predecessors, cugraph_error_t** error);

/* One relaxation round of multi-GPU SSSP on this GPU's edge block (push direction; the role of the MG relaxation of
 * cpp/src/traversal/sssp_impl.cuh:301-375 on one edge partition).  The block must have been created with weights.
 * dist_cols (the block's weight type, one value per column slot, gathered by the launcher inside the column group) holds the
 * tentative distance of every source in the frontier and +inf for all others.  For every edge (row, col) of an active column
 * with nd = dist_cols[col] + w < cutoff, cand_rows[row] (INT64, one per row slot) is lowered with an atomic min to a key:
 *   FLOAT32 blocks: (float bits of nd) << 32 | code(col)   -> the smallest distance, among equal ones the smallest code
 *   FLOAT64 blocks: the bit pattern of nd                   (non-negative doubles order like their int64 bit patterns)
 * code(col) = ((col / maxpart) * grid_cols + grid_c) * maxpart + col % maxpart, as in cugraph_b200_block_bfs_pull.  Row slots
 * without a proposal hold INT64_MAX.  FLOAT32 keys need every code to fit in 32 bits (R * grid_cols * maxpart < 2^32 with
 * R = ceil(n_cols / maxpart)), else CUGRAPH_INVALID_INPUT.  The cutoff is rounded to the weight type as cugraph_sssp does.
 * The first call on a block builds its column-major (push) copy and keeps it; blocks that never run SSSP do not pay for it.
 * Asynchronous, apart from one read-back of the number of active columns and their edge count. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_sssp_relax(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* dist_cols, double cutoff, size_t maxpart, int grid_cols, int grid_c,
  cugraph_type_erased_device_array_view_t* cand_rows, cugraph_error_t** error);

/* Predecessors of a FLOAT64 relaxation round.  win_rows (the block's weight type, one per row slot; +inf = not asked) holds
 * the distance a row accepted in this round.  code_rows[row] (INT64) receives the smallest code(col) over the active columns
 * of dist_cols with dist_cols[col] + w == win_rows[row] (the sum is recomputed exactly as the relaxation formed it), else
 * INT64_MAX.  Arguments and asynchrony as in cugraph_b200_block_sssp_relax. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_sssp_pred(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* dist_cols, const cugraph_type_erased_device_array_view_t* win_rows,
  size_t maxpart, int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* code_rows, cugraph_error_t** error);

/* The edge rules of a BFS / SSSP certificate on this GPU's edge block (MGGraph.validate_bfs / validate_sssp).  One push
 * round over the block's column-major copy (shared with cugraph_b200_block_sssp_relax and the others).
 *   dist_cols (one per column slot, gathered by the launcher inside the column group) and dist_rows (one per row slot,
 *     gathered inside the row group) are INT32 BFS levels with unit steps (weights ignored; INT32_MAX = unreached), or the
 *     weight type of a weighted block (SSSP; the unreached columns must hold +inf so that they are not queued).
 *   pred_rows (INT64, one per row slot): the predecessor code of every row slot (owner rank * maxpart + local id, as
 *     cugraph_b200_block_bfs_pull gives them), -1 = none.
 * For every edge (row, col) of a reached column with nd < cutoff, where nd = dist_cols[col] + w in the weight type (the
 * sum of cugraph_b200_block_sssp_relax, cutoff rounded as there) or dist_cols[col] + 1 in 64-bit integers (unit steps;
 * pass depth_limit + 1, or +inf for none):
 *   violations[0] (INT64, zeroed first) counts the edges with dist_rows[row] > nd or NaN;
 *   flag_rows[row] (byte flags, zeroed first) = 1 when pred_rows[row] is the column's code and dist_rows[row] == nd, 2
 *     when besides dist_cols[col] == dist_rows[row] (a flat step).
 * *edges_from_reached (host) = the number of edges of the reached columns, self-loops and multi-edges included.  NULL
 * arguments, other dtypes, short arrays and a bad grid position return CUGRAPH_INVALID_INPUT.  Asynchronous, apart from
 * one read-back of the number of reached columns and their edge count. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_check_paths(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, const cugraph_type_erased_device_array_view_t* dist_cols,
  const cugraph_type_erased_device_array_view_t* dist_rows, const cugraph_type_erased_device_array_view_t* pred_rows,
  double cutoff, size_t maxpart, int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* flag_rows,
  cugraph_type_erased_device_array_view_t* violations, uint64_t* edges_from_reached, cugraph_error_t** error);

/* One round of multi-GPU weakly connected components on this GPU's edge block (min-label propagation).  The block may be
 * unweighted or weighted; weights are ignored.  label_cols (INT64, at least one per column slot, gathered by the launcher
 * inside the column group) holds the label of every source that changed in the last round and INT64_MAX for all others.
 * cand_rows (INT64, at least one per row slot) receives, for every row slot, the smallest label among the row's sources,
 * INT64_MAX when none is active.  The active columns' edges are pushed with atomicMin through the block's column-major copy,
 * built by the first SSSP or WCC call on the block and kept.  Asynchronous, apart from one read-back of the number of
 * active columns and their edge count. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_wcc_min(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
  const cugraph_type_erased_device_array_view_t* label_cols,
  cugraph_type_erased_device_array_view_t* cand_rows, cugraph_error_t** error);

/* One round of multi-GPU strongly connected components on this GPU's edge block (any phase of Multistep: trim, reach,
 * colouring).  The block may be unweighted or weighted; weights are ignored.
 *   transposed = FALSE (forward, along u -> v): sources are the column slots (key_src, val_src: at least n_cols entries),
 *     destinations the row slots (key_dst, out_dst: at least n_rows); the edges are pushed through the block's column-major
 *     copy (shared with cugraph_b200_block_sssp_relax / _wcc_min / the transposed sweep).
 *   transposed = TRUE (backward, along v -> u): sources are the row slots, destinations the column slots; the edges are
 *     pushed through the block's own rows, with a queue built by the first backward call and kept.
 * All arrays are INT64.  out_dst is first filled with INT64_MIN (mode 0, max) or 0 (mode 1, count).  Then, for every edge
 * whose source is active (val_src[src] != INT64_MIN), whose two ends are different vertices (the codes of the column slot,
 * ((col / maxpart) * grid_cols + grid_c) * maxpart + col % maxpart, and of the row slot,
 * (grid_r * grid_cols + row / maxpart) * maxpart + row % maxpart, differ) and with key_src[src] == key_dst[dst]:
 *   mode 0: out_dst[dst] = max(out_dst[dst], val_src[src]);   mode 1: out_dst[dst] += 1  (multi-edges count once each).
 * NULL arguments, other dtypes, short arrays, a grid position outside grid_rows x grid_cols and other modes return
 * CUGRAPH_INVALID_INPUT.  Asynchronous, apart from one read-back of the number of active sources and their edge count. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_block_scc_push(
  const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block, bool_t transposed, int mode,
  const cugraph_type_erased_device_array_view_t* key_src, const cugraph_type_erased_device_array_view_t* val_src,
  const cugraph_type_erased_device_array_view_t* key_dst, size_t maxpart, int grid_rows, int grid_cols, int grid_r,
  int grid_c, cugraph_type_erased_device_array_view_t* out_dst, cugraph_error_t** error);

/* One position round of multi-GPU extract_paths (the role of the gather rounds of
 * cpp/src/traversal/extract_bfs_paths_impl.cuh:129-238).  An entry (row, pos, code) of a requester asks the owner of the
 * vertex code (owner rank * maxpart + local id, as in cugraph_b200_block_bfs_pull) for that vertex's external id, written at
 * paths[row][pos], and for its predecessor's code, which continues the walk at pos - 1.  The launcher sends the local ids to
 * their owners and brings the answers back in request order.
 *   paths_answer (owner side): for every local id lids[i] (INT32), answers[2i] = vertices[lids[i]] (INT32 / INT64 external
 *     ids, widened) and answers[2i + 1] = pred_codes[lids[i]] (INT64, -1 = none); (-1, -1) for an id outside [0, n_local).
 *     vertices and pred_codes hold at least n_local entries, answers (INT64) at least 2 * len(lids).
 *   paths_advance (requester side): entry i is (rows[i], positions[i]) (INT32, equal sizes) with answers[2i], answers[2i + 1]
 *     as above.  paths (INT32 / INT64, whole rows of max_path_length entries) gets paths[row][pos] = answers[2i] for every
 *     entry inside it; entries outside it are dropped.  An entry with pos > 0 and a code >= 0 of a rank q < world goes on as
 *     (local id = code - q * maxpart, row, pos - 1) into next_lids / next_rows / next_positions (INT32, at least as many
 *     entries as rows), grouped by q in rank order, and counts[q] (INT64, at least world entries, overwritten) receives the
 *     size of group q.  One pass over the entries counts the groups, a second writes the paths and appends every entry to
 *     its group at a per-rank cursor (warp-aggregated atomics); the order inside a group is not fixed.
 * Both are asynchronous; wrong types or sizes return CUGRAPH_INVALID_INPUT. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_paths_answer(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* lids,
  const cugraph_type_erased_device_array_view_t* vertices, const cugraph_type_erased_device_array_view_t* pred_codes,
  size_t n_local, cugraph_type_erased_device_array_view_t* answers, cugraph_error_t** error);
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_paths_advance(
  const cugraph_resource_handle_t* handle, const cugraph_type_erased_device_array_view_t* answers,
  const cugraph_type_erased_device_array_view_t* rows, const cugraph_type_erased_device_array_view_t* positions,
  cugraph_type_erased_device_array_view_t* paths, size_t max_path_length, size_t maxpart, int world,
  cugraph_type_erased_device_array_view_t* next_lids, cugraph_type_erased_device_array_view_t* next_rows,
  cugraph_type_erased_device_array_view_t* next_positions, cugraph_type_erased_device_array_view_t* counts,
  cugraph_error_t** error);

/* Debug hook: one sweep as PageRank would run it on this graph (the shared-memory piece stream when the graph has one)
 * against the plain sweep (an independent implementation) on the same pseudo-random x.  out[0..3] = degree >= 32 rows
 * {max relative difference, its row, that row's degree, rows above 1e-5}; out[4..7] = the same for the degree < 32 rows. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_debug_compare_sweeps(const cugraph_resource_handle_t* handle,
                                                                     cugraph_graph_t* graph, double* out,
                                                                     cugraph_error_t** error);

/* Host-only planner of the sweep's work structure (chunks, phases, per-CTA phase ranges) from the piece counts per
 * (block, kind); the function graph staging itself uses.  Needs no GPU: exposed so that the host logic is testable on CPU
 * (tests/test_sweep_plan_cpu.py).  class_start has n_blocks * 11 + 1 entries (kinds S, Q, H, F1..F8).
 * Outputs: totals[3] = {step-rows, row slots, CTAs}; chunks / fills / phases are 4 x int32 records
 * ({sr_begin,row_begin,n_groups,kind}, {piece_begin,piece_end,block,0}, {block,chunk_begin,chunk_end,0});
 * cta_phase has totals[2] + 1 entries.  Returns CUGRAPH_INVALID_INPUT when a capacity is too small. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_debug_plan_sweep(const int32_t* class_start, int n_blocks, int sm_count,
                                                                 int64_t* totals, int32_t* chunks, int32_t* fills,
                                                                 size_t chunks_capacity, size_t* n_chunks, int32_t* phases,
                                                                 size_t phases_capacity, size_t* n_phases, int32_t* cta_phase,
                                                                 size_t cta_capacity, cugraph_error_t** error);

/* The same planner over n_bands row bands: class_start has n_bands * n_blocks * 11 + 1 entries, key (band * n_blocks +
 * block) * 11 + kind.  Bands are planned one after the other over the same totals[2] CTAs: cta_phase has
 * n_bands * totals[2] + 1 entries (entry band * totals[2] + c starts CTA c of that band) and band_phase n_bands + 1
 * (the phases of band b are [band_phase[b], band_phase[b+1])).  n_bands = 1 is cugraph_b200_debug_plan_sweep. */
CUGRAPH_EXPORT cugraph_error_code_t cugraph_b200_debug_plan_sweep_bands(const int32_t* class_start, int n_bands, int n_blocks,
                                                                       int sm_count, int64_t* totals, int32_t* chunks,
                                                                       int32_t* fills, size_t chunks_capacity, size_t* n_chunks,
                                                                       int32_t* phases, size_t phases_capacity, size_t* n_phases,
                                                                       int32_t* cta_phase, size_t cta_capacity,
                                                                       int32_t* band_phase, cugraph_error_t** error);

#ifdef __cplusplus
}
#endif
