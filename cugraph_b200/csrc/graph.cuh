// Graph data model on one GPU: the graph_view_t / edge_partition_device_view_t role
// (reference cpp/include/cugraph/graph_view.hpp:840-1122, edge_partition_device_view.cuh:912-1215),
// laid out for the kernels in spmv.cuh / traverse.cu.  The pull sweep's own layout of a csx (the piece stream) is private to
// the sweep (sweep_layout.cuh); this header only declares the sweep's entry points.
//
// Three id spaces:
//   external : whatever the caller passed (int32 or int64)
//   rank     : dense 0..V-1 in ascending external-id order (or == external when renumber=false)
//   internal : 0..V-1 in DESCENDING degree of the primary orientation's rows, ties by rank.
// Kernels only see internal ids (always int32: V < 2^31).  The ordering *is* the degree binning:
// rows with degree >= 32 form a prefix whose edges form a prefix of `indices`
// (the role of the reference's segment offsets, graph_view.hpp:242-254 / renumber_edgelist_impl.cuh:740-828).
#pragma once
#include "common.cuh"

#include <memory>
#include <vector>

namespace b200 {

// degree thresholds that delimit the row bins (descending); bin k holds rows with
// kSegThreshold[k] <= degree < kSegThreshold[k-1].
constexpr int kNumSeg                = 7;
constexpr int kSegThreshold[kNumSeg] = {32, 16, 8, 4, 2, 1, 0};

// edges per warp / per CTA in the edge-balanced kernel for the degree>=32 prefix
constexpr int kWarpChunk  = 1024;
constexpr int kWarpsPerCta = 8;

// the pull sweep's layouts of one csx, built on first use (sweep_layout.cuh)
struct sweep_cache_t;

// One orientation: compressed rows over `n_rows` physical rows.
// row_vertex == nullptr  -> physical row r is vertex r (rows are degree-descending by construction)
// row_vertex != nullptr  -> physical row r is vertex row_vertex[r] (a lazily built transpose whose
//                           rows were re-sorted by ITS degree so that the same kernels apply)
struct csx_t {
  int32_t n_rows{0};
  int64_t nnz{0};
  bool offs64{false};
  dbuf offsets;     // (n_rows+1) x int32|int64
  dbuf indices;     // nnz x int32, ascending within a row
  dbuf weights;     // nnz x float|double, or empty
  dbuf row_vertex;  // n_rows x int32, or empty
  bool degree_sorted{true};  // rows in descending degree (binning valid)
  int32_t seg[kNumSeg + 1]{};  // seg[k] = #rows with degree >= kSegThreshold[k]; seg[kNumSeg]=n_rows
  int64_t nnz_hi{0};           // edges in rows with degree >= 32 (= offsets[seg[0]])
  // per-warp-chunk metadata for the edge-balanced kernel over [0, nnz_hi)
  int32_t n_chunks{0};
  dbuf chunk_first_row;  // n_chunks+1 x int32 : row that contains edge c*kWarpChunk
  int32_t n_split{0};
  dbuf split_rows;  // n_split x int32 : rows that straddle a chunk boundary (each listed once)
  // lazily built pull-sweep layouts and cached out-weight sums
  mutable std::unique_ptr<sweep_cache_t> sweep;
  mutable dbuf out_w;  // n_vertices x T : per-source sum of edge weights (or out-degree), T = weight type
  csx_t();   // both in sweep_layout.cu, where sweep_cache_t is complete
  ~csx_t();
};

struct graph_impl {
  cugraph_data_type_id_t vertex_type{INT32};
  cugraph_data_type_id_t edge_type{INT32};
  cugraph_data_type_id_t weight_type{FLOAT32};
  bool weighted{false};
  bool is_symmetric{false};
  bool is_multigraph{false};
  bool store_transposed{false};
  bool renumbered{true};
  int32_t n_vertices{0};
  int64_t n_edges{0};
  int device{0};

  // id maps
  dbuf ext_of_int;    // V x vertex_type : external id of internal vertex i   (the "number_map")
  dbuf sorted_ext;    // V x vertex_type : external ids ascending (renumber=true only)
  dbuf int_of_rank;   // V x int32       : internal id of rank r
  // renumber=false: reported order is external order; results are permuted through int_of_rank.

  std::unique_ptr<csx_t> primary;    // orientation requested at creation (degree-sorted, identity rows)
  std::unique_ptr<csx_t> pull_alt;   // lazily built CSC with re-sorted rows (PageRank on a CSR graph)
  std::unique_ptr<csx_t> push_alt;   // lazily built CSR in vertex order (BFS/SSSP on a CSC graph)
  std::unique_ptr<csx_t> out_alt;    // lazily built CSR with rows re-sorted by out-degree (HITS' hub sweep on a CSC graph)
  std::unique_ptr<csx_t> in_alt;     // lazily built CSC in vertex order (SCC's backward advances on a CSR graph)
};

inline graph_impl* G(cugraph_graph_t* g)
{
  B200_EXPECTS(g != nullptr, CUGRAPH_INVALID_INPUT, "graph is NULL");
  return reinterpret_cast<graph_impl*>(g);
}

// Accessors that build the missing orientation on demand (graph_build.cu).
csx_t const& pull_view(handle_impl const& h, graph_impl& g);  // rows = destinations, indices = sources
csx_t const& push_view(handle_impl const& h, graph_impl& g);  // rows = sources, vertex-indexed offsets
csx_t const& in_view(handle_impl const& h, graph_impl& g);    // rows = destinations, vertex-indexed offsets
csx_t const& out_sweep_view(handle_impl const& h, graph_impl& g);  // rows = sources, binned for the sweep kernels (HITS)

// ---- the pull sweep (sweep.cu): y[row] = init + alpha * sum_{(col -> row)} x[col] * w(col, row) for every row of a csx
// device-resident loop state of one PageRank run (no per-iteration host round trip); a sweep is a no-op once `done` is set
struct pr_state_t {
  double diff;        // sum |pr_new - pr_old| of the iteration being computed
  double dangling;    // sum of pr_new over vertices without out-edges
  double init;        // unvarying part added to every row in the CURRENT sweep
  double pers_scale;  // (dangling*alpha + 1-alpha) for the personalization scatter
  double last_diff;
  int iter;
  int done;
};
// what sweeps over one csx need besides x and y: fp64 accumulators, zero between sweeps, and the device pr_state_t
struct sweep_scratch_t {
  dbuf acc, state;
  void init(handle_impl const& h, csx_t const& c);   // zero accumulators for c's rows; a state of zeros (init 0, not done)
  void set_init(handle_impl const& h, double init);  // the unvarying term the sweep adds to every row
  pr_state_t* st() const { return state.as<pr_state_t>(); }
};
// elements an x buffer needs: whole slices are TMA-copied and everything behind n_vertices must read 0
size_t padded_x_elems(int32_t n_vertices, size_t elem_size);
// an x buffer of padded_x_elems() elements, zero-filled; only [0, n_vertices) is to be written afterwards
template <typename T>
dbuf make_sweep_x(handle_impl const& h, int32_t n_vertices);
// PageRank's vertex pass, done by the sweep where it writes each row (x_next == nullptr: none).  For the value `val` of vertex
// v: x_next[v] = val / out_w[v] (val where out_w[v] is 0), st->dangling += val where out_w[v] is 0, and with y_old
// st->diff += |val - y_old[v]|.  The sums are fp64 partials added with one atomic per warp, read by a later launch.
// x_next is a second buffer from make_sweep_x: the sweep still reads x while it writes rows.  With an epilogue y may be
// nullptr: the sweep then writes x_next alone (PageRank at epsilon = 0, whose y is read only after the last iteration).
template <typename T>
struct sweep_epilogue_t {
  T const* out_w{nullptr};
  T* x_next{nullptr};
  T const* y_old{nullptr};
};
// The piece stream (sweep.cuh) when the graph has one, else the plain sweep (spmv.cuh).  x holds padded_x_elems() elements
// and does not overlap y.  use_weights = false: plain neighbour sums on a weighted graph (HITS).  covered_rows_only: the
// rows without edges may keep what y holds (multi-GPU blocks, whose unvarying term is 0).
template <typename T>
void pull_sweep(handle_impl const& h, csx_t const& c, int32_t n_vertices, T const* x, T* y, sweep_scratch_t& sc, double alpha,
                bool use_weights = true, bool covered_rows_only = false, sweep_epilogue_t<T> const& epi = {});
// build now what pull_sweep would build on its first call for elements of `elem_size` bytes (the piece stream, if c gets one)
void prepare_pull_sweep(handle_impl const& h, csx_t const& c, int32_t n_vertices, size_t elem_size);

// ---- multi-source BFS (traverse.cu): one batch of nb <= 64 sources (internal ids), bit j of a vertex's 64-bit word for
// sources[j].  dist / pred (each may be null) get nb rows of V entries.  After the seed (level 0) and after every level d
// that reached something, sink->level(d, words, queue, n) sees the frontier: the n vertices that gained bits at level d and,
// in words[v] (V entries), exactly those bits.  queue lists the n vertices, or is null after a bottom-up level (then the
// vertices are those with a non-zero word).  Both are only valid during the call; the sink may enqueue work on h.stream.
struct ms_level_sink {
  virtual void level(int d, unsigned long long const* words, int32_t const* queue, int n) = 0;
 protected:
  ~ms_level_sink() = default;
};
void multi_source_bfs_batch(handle_impl const& h, graph_impl& g, int32_t const* sources, int nb, int depth_limit, int32_t* dist,
                            int32_t* pred, int batch, ms_level_sink* sink);

// external <-> internal id helpers (graph_build.cu)
// out[i] = internal id of ext[i], or -1 if ext[i] is not a vertex.
void ext_to_int(handle_impl const& h, graph_impl const& g, void const* ext, size_t n, int32_t* out);
// in-place/out-of-place: ext_out[i] = external id of internal id in[i] (in[i] < 0 stays -1)
void int_to_ext(handle_impl const& h, graph_impl const& g, int32_t const* in, size_t n, void* ext_out);
// vertices array (external ids) in reported order
dbuf reported_vertices(handle_impl const& h, graph_impl const& g);
// permute a per-vertex result from internal order into reported order (no-op copy when renumbered)
dbuf to_reported_order(handle_impl const& h, graph_impl const& g, void const* internal_vals, size_t elem_size);
// the same into out (V elements, not overlapping internal_vals)
void to_reported_order_into(handle_impl const& h, graph_impl const& g, void const* internal_vals, size_t elem_size, void* out);

// (vertex, value) pairs with external ids -> dense internal-order vector, missing = fill
template <typename T>
dbuf collect_vertex_values(handle_impl const& h, graph_impl const& g,
                           device_array_view_impl const* verts, device_array_view_impl const* vals,
                           T fill);

std::unique_ptr<csx_t> build_binned_rows(handle_impl const& h, int32_t const* major, int32_t const* minor, void const* w,
                                         cugraph_data_type_id_t wtype, int64_t n, int32_t nv);
// the vertex (row_vertex, or the physical row) of every edge of a csx, in edge order
dbuf expand_majors(handle_impl const& h, csx_t const& c);
// multi-GPU staging of one edge block (cugraph_b200_block_stage_edges): the n edges (rows, cols[, reversed][, w]) in
// slot coordinates, rewritten in place; returns how many are left
int64_t stage_block_edges(handle_impl const& h, int32_t n_rows, int32_t n_cols, int32_t* rows, int32_t* cols,
                          uint8_t const* reversed, void* w, cugraph_data_type_id_t wtype, int64_t n, bool drop_multi_edges,
                          bool symmetrize);

}  // namespace b200
