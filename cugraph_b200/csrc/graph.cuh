// Graph data model on one GPU: the graph_view_t / edge_partition_device_view_t role
// (reference cpp/include/cugraph/graph_view.hpp:840-1122, edge_partition_device_view.cuh:912-1215),
// laid out for the kernels in spmv.cu / traverse.cu.
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

#include <algorithm>
#include <cstdlib>
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

// ---------------------------------------------------------------------------------------------
// Column-blocked "piece stream" of the rows [0, n_str) for the shared-memory pull sweep (sweep.cuh).  n_str is a degree-bin
// bound: on large graphs the rows of in-degree < kSweepTailDegree (the TAIL) leave the stream and are swept by a row
// kernel instead (k_sweep_tail); on smaller graphs the stream covers every non-empty row.
// The source (column) space is cut into B blocks of W vertices (W * sizeof(T) = 192 KiB minus 64 zero columns: the slice of
// x a persistent CTA keeps in shared memory).  Rows keep their neighbours sorted by source id, so a row's adjacency is
// already partitioned by block; every (row, block) SEGMENT is cut into PIECES of <= 64 entries.  A piece is stored with
// 16-bit local column ids in one of 11 KINDS: S / Q / H = 1 / 2 / <= 4 entries (2 / 4 / 8 bytes of ids), F1..F8 = 1..8 lane
// slots of 8 entries (16 bytes each; short pieces are padded with a column that reads 0).  The stream rows are split into
// BANDS of consecutive rows (a multiple of kBandRowAlign each, sized so that a band's fp64 accumulators stay in the L2) and
// pieces are ordered by (band, block, kind): the sweep runs band after band.  The unit every kernel step works on is a
// STEP-ROW = 32 lanes x 16 bytes of ids (one 128-bit load per lane, 512 contiguous bytes per warp): it holds 256 S pieces, 128 Q pieces, 64 H pieces, or one of the c slots of 32 Fc
// pieces (a GROUP of kind Fc is c consecutive step-rows, lane = piece).  Row ids (int32, -1 = unused piece) are stored per
// group so that a lane's rows are contiguous: 8 / 4 / 2 / 1 per lane.
// ---------------------------------------------------------------------------------------------
constexpr int kHotSliceBytes = 192 * 1024;  // x slice a CTA keeps in shared memory
constexpr int kHotZeroPad    = 64;          // trailing elements of the slice that hold zeros (padding target)
constexpr int kHotSlot       = 8;           // entries per lane slot

constexpr int kBandRowAlign = 512;  // band bounds: a multiple of the finish kernel's rows per warp (k_sweep_finish)

// Tail of the piece stream: a row of small in-degree has its few edges in different column blocks, so the stream pays one
// fp64 RED per edge for it, and such rows are most of the rows (their accumulators decide how many bands are needed).
// Rows of in-degree < kSweepTailDegree are gathered by k_sweep_tail instead, on graphs of at least kSweepTailMinEdges edges.
// A kSegThreshold value.  Measured on an H100 80GB HBM3 at 700 W, RMAT-24 PageRank step, with the row-per-thread tail kernel
// of before: 86.3 ms without a tail, 78.8 / 73.4 / 72.7 / 74.5 ms with bounds 4 / 8 / 16 / 32 (DESIGN.md §3.2); from 8 on the
// stream needs one band.  With the tail layout below, at 400 W: 73.1 / 68.3-70.6 / 69.1 ms with bounds 8 / 16 / 32 (sweep
// 0.660 / 0.635-0.642 / 0.612 ms): 32 is not yet separated from 16 by more than the run-to-run spread.
constexpr int kSweepTailDegree         = 16;
constexpr long long kSweepTailMinEdges = 1ll << 24;

constexpr int kNumKinds = 11;  // S, Q, H, F1..F8
constexpr int kKindS = 0, kKindQ = 1, kKindH = 2, kKindF1 = 3;
__host__ __device__ __forceinline__ int kind_steps(int kind) { return kind < kKindF1 ? 1 : kind - 2; }  // step-rows per group
__host__ __device__ __forceinline__ int kind_pieces(int kind) { return kind == kKindS ? 256 : (kind == kKindQ ? 128 : (kind == kKindH ? 64 : 32)); }
// groups per chunk (a chunk = consecutive groups of one kind in one block = what a warp loads into its registers at once:
// at most 8 x 128 bits of ids / rows + 2 row words, chunk_regs_t in sweep.cuh)
__host__ __device__ __forceinline__ int kind_chunk_groups(int kind)
{
  return kind == kKindS ? 2 : (kind == kKindQ ? 4 : (kind == kKindH ? 4 : (kind == kKindF1 ? 6 : (kind == kKindF1 + 1 ? 3 : (kind <= kKindF1 + 3 ? 2 : 1)))));
}

struct sweep_chunk_t {  // 16 bytes
  int32_t sr_begin;   // first step-row
  int32_t row_begin;  // first row slot
  int32_t n_groups;   // 1 .. kind_chunk_groups(kind)
  int32_t kind;
};
struct sweep_phase_t {  // consecutive chunks of one block inside one CTA's range; its cursor is phase-indexed
  int32_t block;
  int32_t chunk_begin;
  int32_t chunk_end;
  int32_t pad;
};

// ---------------------------------------------------------------------------------------------
// Tail layout of the rows [n_str, n_cov) for k_sweep_tail (sweep.cuh).  Rows are degree-descending, so the tail is made of
// RUNS of rows of one in-degree d (< kSweepTailDegree <= 32).  A run is cut into TILES of 32 consecutive rows, lane l = row
// first_row + 32 * t + l; entry k of lane l of tile t of a run sits at tail_ids[id_off + t * 32 * d + k * 32 + l] (int32 source
// id, a row's entries in ascending source order: hubs first).  No offsets and no padding inside a run: every warp-wide load
// of ids is one 128-byte line; only the last tile of a run has lanes without a row, whose entries read column n_vertices (x
// is zero there).  A WORK UNIT is tail_unit_tiles(d) consecutive tiles of one run (the last one of a run may be shorter):
// about kTailUnitEntries entries per lane whatever d, consecutive in tail_ids.
// ---------------------------------------------------------------------------------------------
constexpr int kTailTile        = 32;  // rows per tile (= lanes)
constexpr int kTailUnitEntries = 24;  // entries per lane in a work unit, at least one tile (ids held in registers, twice)
constexpr int kTailMaxDegree   = 31;  // kSegThreshold[0] - 1: the largest bound leaves rows of in-degree <= 31 in the tail
__host__ __device__ constexpr int tail_unit_tiles(int d) { return d >= kTailUnitEntries ? 1 : kTailUnitEntries / d; }

struct tail_run_t {   // 24 bytes; a run table ends with a sentinel that holds the totals (first_row = n_cov)
  int32_t degree;
  int32_t first_row;
  int32_t first_tile;
  int32_t first_unit;
  int64_t id_off;     // first entry in tail_ids
};

struct sweep_layout_t {
  int W{0};               // source columns per block (= slice elements - kHotZeroPad)
  int B{0};               // blocks
  int32_t n_cov{0};       // rows [0, n_cov) are covered = every non-empty row (rows are degree-descending)
  int32_t n_str{0};       // rows [0, n_str) are in the piece stream (a degree-bin bound <= n_cov); [n_str, n_cov) is the tail
  int64_t nnz{0};         // edges of the graph (the stream holds the first offsets[n_str] of them)
  bool bank_order{false};  // entries inside the F slots ordered by shared-memory bank (4-byte values)
  int64_t n_steprows{0};
  int64_t n_rowslots{0};
  int64_t n_pieces{0};
  dbuf ids;        // n_steprows x 32 x uint4 (8 x uint16: column - block * W; padding -> one of the zero columns)
  dbuf w;          // n_steprows x 32 x 8 x T, padding 0; or empty
  dbuf rows;       // n_rowslots x int32
  dbuf chunks;     // n_chunks x sweep_chunk_t
  dbuf phases;     // n_phases x sweep_phase_t
  dbuf cta_phase;  // (n_bands * n_cta + 1) x int32: in band b, CTA c owns phases [cta_phase[b * n_cta + c], the next entry)
                   // (cost-balanced, contiguous chunks)
  dbuf cursor;     // n_phases + 1 x int: next chunk of the phase (relative), then the tail's next work unit; reset by the
                   // finish kernel (the tail's by the last band's, which runs after the previous sweep's tail)
  int32_t n_chunks{0};
  int32_t n_phases{0};
  int n_cta{0};
  int n_bands{1};
  std::vector<int32_t> band_row;    // n_bands + 1: band b holds rows [band_row[b], band_row[b+1]); band_row[n_bands] = n_str
  std::vector<int32_t> band_phase;  // n_bands + 1: the phases of band b are [band_phase[b], band_phase[b+1])
  // the tail (rows [n_str, n_cov)), when there is one
  int n_tail_runs{0};
  std::vector<tail_run_t> tail_runs;  // n_tail_runs + 1 (sentinel), on the host
  dbuf tail_run;                      // the same on the device
  dbuf tail_ids;                      // tail_runs[n_tail_runs].id_off x int32
  dbuf tail_w;                        // the same x T, padding 0; or empty
};

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
  // lazily built column-blocked copies (float / double element width) and cached out-weight sums
  mutable std::unique_ptr<sweep_layout_t> hot4, hot8;
  mutable bool hot4_tried{false}, hot8_tried{false};
  mutable dbuf out_w;  // n_vertices x T : per-source sum of edge weights (or out-degree), T = weight type
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

  // multi-GPU (mg.cu): this rank's blocks of the 2D partition
  void* mg{nullptr};
};

inline graph_impl* G(cugraph_graph_t* g)
{
  B200_EXPECTS(g != nullptr, CUGRAPH_INVALID_INPUT, "graph is NULL");
  return reinterpret_cast<graph_impl*>(g);
}

// Accessors that build the missing orientation on demand (graph_build.cu).
csx_t const& pull_view(handle_impl const& h, graph_impl& g);  // rows = destinations, indices = sources
// piece stream for elements of `elem_size` bytes, or nullptr when the graph is too small for it or has 64-bit offsets
sweep_layout_t const* sweep_layout(handle_impl const& h, csx_t const& c, int32_t n_vertices, size_t elem_size);
csx_t const& push_view(handle_impl const& h, graph_impl& g);  // rows = sources, vertex-indexed offsets
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
// The piece stream (sweep.cuh) when the graph has one, else the plain sweep (spmv.cuh).  x holds padded_x_elems() elements
// and does not overlap y.  use_weights = false: plain neighbour sums on a weighted graph (HITS).  covered_rows_only: the
// rows without edges may keep what y holds (multi-GPU blocks, whose unvarying term is 0).
template <typename T>
void pull_sweep(handle_impl const& h, csx_t const& c, int32_t n_vertices, T const* x, T* y, sweep_scratch_t& sc, double alpha,
                bool use_weights = true, bool covered_rows_only = false);

// external <-> internal id helpers (graph_build.cu)
// out[i] = internal id of ext[i], or -1 if ext[i] is not a vertex.
void ext_to_int(handle_impl const& h, graph_impl const& g, void const* ext, size_t n, int32_t* out);
// in-place/out-of-place: ext_out[i] = external id of internal id in[i] (in[i] < 0 stays -1)
void int_to_ext(handle_impl const& h, graph_impl const& g, int32_t const* in, size_t n, void* ext_out);
// vertices array (external ids) in reported order
dbuf reported_vertices(handle_impl const& h, graph_impl const& g);
// permute a per-vertex result from internal order into reported order (no-op copy when renumbered)
dbuf to_reported_order(handle_impl const& h, graph_impl const& g, void const* internal_vals, size_t elem_size);

// (vertex, value) pairs with external ids -> dense internal-order vector, missing = fill
template <typename T>
dbuf collect_vertex_values(handle_impl const& h, graph_impl const& g,
                           device_array_view_impl const* verts, device_array_view_impl const* vals,
                           T fill);

std::unique_ptr<csx_t> build_binned_rows(handle_impl const& h, int32_t const* major, int32_t const* minor, void const* w,
                                         cugraph_data_type_id_t wtype, int64_t n, int32_t nv);
// the vertex (row_vertex, or the physical row) of every edge of a csx, in edge order
dbuf expand_majors(handle_impl const& h, csx_t const& c);

// ---- multi-GPU hooks (mg.cu) ----
struct mg_pr_args {
  double alpha;
  double epsilon;
  size_t max_iterations;
};
void attach_comm(handle_impl* h, void* comm);
void free_mg_graph(graph_impl* g);
void mg_pagerank(handle_impl const& h, graph_impl& g, mg_pr_args const& a, centrality_result_impl& res);

}  // namespace b200
