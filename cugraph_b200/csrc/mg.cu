// Multi-GPU building blocks (one process per GPU).  The 2D edge partition, the vertex -> GPU map and
// the collectives (all-gather of x over the column group, reduce-scatter of partial y over the row
// group — the roles of update_edge_src_property's grouped ncclBroadcast and
// per_v_transform_reduce_e's grouped ncclReduce, update_edge_src_dst_property.cuh:550-579 /
// per_v_transform_reduce_e.cuh:3389-3407) are orchestrated by cugraph_b200/mg.py over
// torch.distributed (NCCL on NVLink 5 / NVSwitch).  This file provides the device-side pieces behind
// the C ABI (the resource handle bound to the caller's CUDA stream is made in capi_basic.cu): rectangular edge blocks with the
// same binned / column-blocked layout as the single-GPU graph, the block pull sweep and the fused
// per-iteration vertex step, the transposed block sweep, the owner steps of Katz, eigenvector centrality and HITS, the BFS
// pull and push steps, the multi-source BFS level, predecessor and owner steps, the SSSP push relaxation, the WCC min-label round and the two sides of an extract_paths round.  All calls only ENQUEUE work on the handle's stream (the
// push calls of BFS, SSSP, WCC and SCC read back one queue size; the first transposed sweep of a block builds its column-major copy).
#include "advance.cuh"
#include "centrality_ops.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <initializer_list>
#include <limits>
#include <type_traits>

namespace b200 {

// the column-major copy of a block (built by the first BFS push, SSSP, WCC, SCC or transposed sweep call on the block): physical rows are
// the block's column slots in descending out-degree (row_vertex = column slot), neighbours are row slots
struct block_push_t {
  std::unique_ptr<csx_t> csx;
  int32_t n_ne{0};     // physical rows with at least one edge (a prefix)
  dbuf queue, q_deg;   // active physical rows and their degrees (q_deg has one element more: advance() reads n + 1)
  dbuf counts;         // block_queue_counts_t
  advance_scratch_t adv;
  sweep_scratch_t scratch;  // the transposed sweep's (a pull sweep over this copy), made by its first call
  bool sweep_ready{false};
};

// a queue over the block's own physical rows (row slots as sources: the backward push of multi-GPU SCC), built on first use
struct block_rows_queue_t {
  int32_t n_ne{0};     // physical rows with at least one edge (a prefix)
  dbuf queue, q_deg;   // as in block_push_t
  dbuf counts;         // block_queue_counts_t
  advance_scratch_t adv;
};

struct block_impl {
  std::unique_ptr<csx_t> csx;
  std::unique_ptr<block_push_t> push;  // lazily built (multi-GPU BFS push steps, SSSP, WCC, SCC and transposed sweeps)
  std::unique_ptr<block_rows_queue_t> rows_queue;  // lazily built (multi-GPU SCC's backward push)
  int32_t n_rows{0}, n_cols{0}, n_span{0};
  bool weighted{false};
  cugraph_data_type_id_t wtype{FLOAT32};
  sweep_scratch_t scratch;  // init = 0
  // per orientation (0 = pull, 1 = transposed): the y array whose slots WITHOUT edges this block has already written (0):
  // later sweeps of that orientation into the same array only finish the slots that have edges — in a 2D block more than
  // half of the slots are empty (the caller must not write them either)
  void const* y_complete[2]{nullptr, nullptr};
};

namespace {

// owner slice, one PageRank iteration (pagerank_impl.cuh:225-251, 311-318 fused):
//   init    = (dangling_prev * alpha + 1 - alpha) / V        (dangling_prev from totals_prev[1])
//   pr_new  = first ? pr : y + init                          (kPersonalized = false, pers unused)
//   pr_new  = first ? pr : y + (dangling_prev * alpha + 1 - alpha) * (pers / pers_sum)
//                                                            (kPersonalized: k_finalize + k_personalize of pagerank.cu,
//                                                             pers = 0 for the vertices not personalized)
//   diff += |pr_new - pr| ; dangling += pr_new where out_w == 0 ; x = pr_new / (out_w or 1) ; pr = pr_new
// The personalization is a compile-time flag so that the plain float instantiation keeps its 32 registers: a runtime
// branch took it to 40, which fits 6 instead of the launched 8 CTAs of 256 per SM, and the step on 8.87 M owned vertices
// went from 66.0 to 75.6 us (H100 80GB HBM3, 700 W).
template <typename T, bool kPersonalized>
__global__ void __launch_bounds__(256)
k_mg_vertex_step(T const* __restrict__ y, T* __restrict__ pr, T const* __restrict__ out_w, T* __restrict__ x,
                 T const* __restrict__ pers, int32_t n, double alpha, double n_vertices_global, double pers_sum, int first,
                 double const* __restrict__ totals_prev, double* __restrict__ partial_out)
{
  __shared__ double smem[8];
  const double base = kPersonalized && !first ? totals_prev[1] * alpha + (1.0 - alpha) : 0.0;
  const double init = kPersonalized || first ? 0.0 : (totals_prev[1] * alpha + (1.0 - alpha)) / n_vertices_global;
  double diff = 0.0, dang = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T old = pr[i];
    T nv;
    if constexpr (kPersonalized) {
      // a vertex without personalization keeps y, which is what y + base * (0 / pers_sum) gives: skip the fp64 divide
      const T pv = first ? (T)0 : pers[i];
      nv         = first ? old : pv == (T)0 ? y[i] : (T)((double)y[i] + base * ((double)pv / pers_sum));
    } else {
      nv = first ? old : (T)((double)y[i] + init);
    }
    const T ow  = out_w[i];
    diff += fabs((double)nv - (double)old);
    if (ow == (T)0) dang += (double)nv;
    x[i]  = (ow == (T)0) ? nv : nv / ow;
    pr[i] = nv;
  }
  diff = block_sum(diff, smem);
  dang = block_sum(dang, smem);
  if (threadIdx.x == 0) {
    atomicAdd(partial_out + 0, diff);
    atomicAdd(partial_out + 1, dang);
  }
}

// the global code of a column slot: (owner rank) * maxpart + local id, owner rank = (col / maxpart) * grid_cols + grid_c
__device__ __forceinline__ long long column_code(int col, long long maxpart, int grid_cols, int grid_c)
{
  return ((long long)(col / maxpart) * grid_cols + grid_c) * maxpart + (col % maxpart);
}

// ---- one level of multi-GPU BFS on this GPU's edge block, pull direction (the MG form of k_bfs_bottomup, traverse.cu;
// reference: the bottom-up step of bfs_impl.cuh:593-869 on an edge partition, with the frontier arriving through
// fill_edge_dst_property-style broadcasts, fill_edge_src_dst_property.cuh:1368).  The block stores its edges by destination
// slot (rows) with the source slots as neighbours (columns, ascending).  frontier[col] / visited[row] are byte flags over
// the block's column / row slots (the launcher all-gathers them inside the column / row group); every unvisited row scans
// its sources until it meets one in the frontier and reports it as cand[row] = GLOBAL code of that source (column_code),
// else -1.  Rows of degree >= 32
// (the prefix of the degree-ordered physical rows) take a warp each with a ballot early exit, the others a thread each.

template <typename O>
__global__ void __launch_bounds__(256)
k_block_bfs_pull_hi(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t n_hi,
                    uint8_t const* __restrict__ frontier, uint8_t const* __restrict__ visited, long long maxpart, int grid_cols,
                    int grid_c, long long* __restrict__ cand)
{
  const int lane = threadIdx.x & 31;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < n_hi; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    if (visited[slot]) continue;
    const long long e1 = (long long)off[r + 1];
    int found          = -1;
    for (long long e = (long long)off[r] + lane; __any_sync(0xffffffffu, e < e1); e += 32) {
      const int col = e < e1 ? idx[e] : -1;
      const bool hit = col >= 0 && frontier[col] != 0;
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (m) {
        found = __shfl_sync(0xffffffffu, col, __ffs((int)m) - 1);
        break;
      }
    }
    if (lane == 0 && found >= 0) cand[slot] = column_code(found, maxpart, grid_cols, grid_c);
  }
}

template <typename O>
__global__ void __launch_bounds__(256)
k_block_bfs_pull_low(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t r0,
                     int32_t r1, uint8_t const* __restrict__ frontier, uint8_t const* __restrict__ visited, long long maxpart,
                     int grid_cols, int grid_c, long long* __restrict__ cand)
{
  for (long long r = r0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; r < r1; r += (long long)gridDim.x * blockDim.x) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    if (visited[slot]) continue;
    const long long e1 = (long long)off[r + 1];
    for (long long e = (long long)off[r]; e < e1; ++e) {
      const int col = idx[e];
      if (frontier[col]) {
        cand[slot] = column_code(col, maxpart, grid_cols, grid_c);
        break;
      }
    }
  }
}

template <typename O>
void block_bfs_pull(handle_impl const& h, csx_t const& c, uint8_t const* frontier, uint8_t const* visited, long long maxpart,
                    int grid_cols, int grid_c, long long* cand, int32_t n_row_slots)
{
  B200_LAUNCH(h, k_fill<long long>, grid_for(n_row_slots, 1, h.sm_count * 8), kBlock, 0, cand, (int64_t)n_row_slots, -1ll);
  const int32_t n_hi = c.degree_sorted ? c.seg[0] : 0;
  const int32_t n_ne = c.degree_sorted ? c.seg[kNumSeg - 2] : c.n_rows;  // rows with at least one edge
  if (n_hi > 0)
    B200_LAUNCH(h, (k_block_bfs_pull_hi<O>), grid_for((int64_t)n_hi * 32, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, frontier, visited, maxpart, grid_cols, grid_c, cand);
  if (n_ne > n_hi)
    B200_LAUNCH(h, (k_block_bfs_pull_low<O>), grid_for(n_ne - n_hi, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, n_ne, frontier, visited, maxpart, grid_cols, grid_c, cand);
}

// ---- one relaxation round of multi-GPU SSSP on this GPU's edge block, push direction (the MG form of the SSSP rounds of
// traverse.cu; reference: the multi_gpu branches of sssp_impl.cuh:301-375, whose frontier arrives through
// update_edge_src_property).  The launcher gathers the distances of the frontier sources over the block's column slots
// (+inf = not in the frontier); the block's column-major copy (block_push_t) turns the active columns into a queue of its
// physical rows, and the same merge-path advance as on one GPU (advance.cuh) relaxes their edges into one INT64 key per row
// slot, reduced to the owners by a MIN reduce-scatter.
struct block_queue_counts_t {
  int n;                     // active physical rows appended to the queue
  int pad;
  unsigned long long edges;  // their degree sum
};

// whether a column takes part in a round: a finite SSSP distance, a WCC label other than INT64_MAX
__device__ __forceinline__ bool column_active(float v) { return v < INFINITY; }
__device__ __forceinline__ bool column_active(double v) { return v < INFINITY; }
__device__ __forceinline__ bool column_active(long long v) { return v != LLONG_MAX; }
__device__ __forceinline__ bool column_active(uint8_t f) { return f != 0; }  // a BFS frontier flag
__device__ __forceinline__ bool column_active(int32_t d) { return d != INT_MAX; }  // a reached BFS distance
__device__ __forceinline__ bool column_active(unsigned long long w) { return w != 0ull; }  // a multi-source BFS frontier word

// physical rows r < n_ne of the push copy whose column slot row_vertex[r] is active, with their degrees
template <typename O, typename T>
__global__ void __launch_bounds__(kBlock)
k_block_active_rows(O const* __restrict__ off, int32_t const* __restrict__ row_vertex, int32_t n_ne, T const* __restrict__ dist_cols,
                    int32_t* __restrict__ q, int32_t* __restrict__ q_deg, block_queue_counts_t* __restrict__ cnt)
{
  unsigned long long edges = 0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n_ne; r += gridDim.x * blockDim.x) {
    if (column_active(dist_cols[row_vertex[r]])) {
      const int32_t d = (int32_t)((long long)off[r + 1] - (long long)off[r]);
      const int pos   = warp_append(&cnt->n);
      q[pos]          = r;
      q_deg[pos]      = d;
      edges += (unsigned long long)d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) edges += __shfl_xor_sync(0xffffffffu, edges, o);
  if ((threadIdx.x & 31) == 0 && edges) atomicAdd(&cnt->edges, edges);
}

// one key orders the proposals to a row: float (distance bits, code) — the smallest distance, among equal distances the
// smallest code; double: the distance bits alone (non-negative doubles order like their int64 bit patterns)
__device__ __forceinline__ long long sssp_key(float nd, long long code)
{
  return (long long)(((unsigned long long)__float_as_uint(nd) << 32) | (unsigned long long)code);
}
__device__ __forceinline__ long long sssp_key(double nd, long long) { return __double_as_longlong(nd); }

template <typename T>
struct block_relax_op {
  int32_t const* col_of;  // column slot of a physical row of the push copy
  T const* w;
  T const* dist;          // over column slots, +inf = not in the frontier
  T cutoff;
  long long maxpart;
  int grid_cols, grid_c;
  long long* cand;        // over row slots
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const int col = col_of[src];
    const T nd    = dist[col] + w[e];
    if (!(nd < cutoff)) return;
    const long long key = sssp_key(nd, column_code(col, maxpart, grid_cols, grid_c));
    if (key < cand[nbr]) atomicMin(cand + nbr, key);  // a stale read is larger than the current value: never skips a win
  }
};

// the smallest code among the frontier columns whose sum reproduces the distance a row accepted (double runs)
template <typename T>
struct block_pred_op {
  int32_t const* col_of;
  T const* w;
  T const* dist;
  T const* win;           // over row slots, +inf = not asked
  long long maxpart;
  int grid_cols, grid_c;
  long long* code;        // over row slots
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const T want = win[nbr];
    if (!(want < (T)INFINITY)) return;
    const int col = col_of[src];
    if (dist[col] + w[e] != want) return;
    const long long k = column_code(col, maxpart, grid_cols, grid_c);
    if (k < code[nbr]) atomicMin(code + nbr, k);
  }
};

// ---- the edge part of the BFS / SSSP certificate (MGGraph.validate_bfs / validate_sssp) on this GPU's edge block.  The
// launcher gathers the given distances over the column slots (unreached: INT32_MAX for BFS, +inf for SSSP, so that only
// the reached columns are queued) and over the row slots (as given), and the predecessor codes over the row slots.  For
// every stored edge u -> v of a reached column whose step is allowed (nd = d[u] + w, or d[u] + 1 with unit steps, below the
// cutoff, in the arithmetic of block_relax_op) the op counts an `edge` violation when d[v] > nd (or is NaN), and marks
// the row when the row's predecessor is this column at exactly d[v] = nd: 1, or 2 for a flat step (d[u] = d[v]).
// Unit steps (T = int32_t) add in 64 bits, so the cutoff d[u] < depth_limit reads nd < depth_limit + 1.
template <typename T>
struct block_check_op {
  using A = std::conditional_t<std::is_same<T, int32_t>::value, long long, T>;
  int32_t const* col_of;     // column slot of a physical row of the push copy
  T const* w;                // nullptr: unit steps
  T const* dist_cols;        // over column slots, unreached = inactive
  T const* dist_rows;        // over row slots
  long long const* pred_rows;  // over row slots: predecessor code, -1 = none
  A cutoff;
  long long maxpart;
  int grid_cols, grid_c;
  uint8_t* flag_rows;        // over row slots
  unsigned long long* violations;
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const int col = col_of[src];
    const A du    = (A)dist_cols[col];
    const A nd    = w ? (A)(dist_cols[col] + w[e]) : du + (A)1;
    const bool allowed = nd < cutoff;
    const A dv         = (A)dist_rows[nbr];
    const bool bad     = allowed && !(dv <= nd);
    if (allowed && dv == nd && pred_rows[nbr] == column_code(col, maxpart, grid_cols, grid_c))
      flag_rows[nbr] = du == dv ? 2 : 1;  // every match of a row writes the same value: d[u] is the predecessor's
    const unsigned mask = __activemask();
    const unsigned n    = (unsigned)__popc(__ballot_sync(mask, bad));
    if (n && (threadIdx.x & 31) == __ffs(mask) - 1) atomicAdd(violations, (unsigned long long)n);
  }
};

// ---- one level of multi-GPU BFS on this GPU's edge block, push direction (the MG form of bfs_topdown_op, traverse.cu;
// reference: the top-down step of bfs_impl.cuh on an edge partition).  The frontier columns (byte flags, gathered as for
// the pull step) are queued through the push copy, and every edge into an unvisited row offers the global code of its
// source; the row keeps the largest, so a level's candidate does not depend on the order of the atomics.
struct block_bfs_push_op {
  int32_t const* col_of;   // column slot of a physical row of the push copy
  uint8_t const* visited;  // over row slots
  long long maxpart;
  int grid_cols, grid_c;
  long long* cand;         // over row slots, -1 = no frontier source
  __device__ __forceinline__ void edge(int src, long long, int nbr) const
  {
    if (visited[nbr]) return;
    const long long code = column_code(col_of[src], maxpart, grid_cols, grid_c);
    if (code > cand[nbr]) atomicMax(cand + nbr, code);  // a stale read is smaller than the current value: never skips a win
  }
};

// argument checks shared by the two BFS block calls
void check_bfs_block_args(block_impl const& b, device_array_view_impl const* fv, device_array_view_impl const* vv,
                          device_array_view_impl const* cv, size_t maxpart, int grid_cols, int grid_c)
{
  B200_EXPECTS(dtype_size(fv->type) == 1 && dtype_size(vv->type) == 1, CUGRAPH_INVALID_INPUT, "frontier / visited are byte flags");
  B200_EXPECTS(cv->type == INT64, CUGRAPH_INVALID_INPUT, "cand must be INT64");
  B200_EXPECTS(fv->size >= (size_t)b.n_cols && vv->size >= (size_t)b.n_rows && cv->size >= (size_t)b.n_rows,
               CUGRAPH_INVALID_INPUT, "flag / candidate arrays shorter than the block's slots");
  B200_EXPECTS(maxpart > 0 && grid_cols > 0 && grid_c >= 0 && grid_c < grid_cols, CUGRAPH_INVALID_INPUT, "bad grid position");
}

// the column-major copy of the block, built on first use (the mirror image of pull_view / out_sweep_view, graph_build.cu)
block_push_t& push_copy(handle_impl const& h, block_impl& b)
{
  if (!b.push) {
    auto p         = std::make_unique<block_push_t>();
    csx_t const& c = *b.csx;
    dbuf maj       = expand_majors(h, c);  // row slot of every edge
    p->csx = build_binned_rows(h, c.indices.as<int32_t>(), maj.as<int32_t>(), b.weighted ? c.weights.data() : nullptr, b.wtype,
                               c.nnz, b.n_span);
    csx_t const& pc = *p->csx;
    p->n_ne         = pc.degree_sorted ? pc.seg[kNumSeg - 2] : pc.n_rows;
    p->queue        = make_dbuf<int32_t>((size_t)std::max(pc.n_rows, 1), h.stream);
    p->q_deg        = make_dbuf<int32_t>((size_t)pc.n_rows + 1, h.stream);
    p->counts       = make_dbuf<block_queue_counts_t>(1, h.stream);
    p->adv.init(h, pc.n_rows, pc.nnz);
    sync(h);
    b.push = std::move(p);
  }
  return *b.push;
}

// a pull sweep of the block (transposed = false) or of its column-major copy (transposed = true: y over column slots,
// x over row slots) — the copy is binned like the block, so the same sweep and the same layouts apply to it
void block_sweep(handle_impl const& h, block_impl& b, bool transposed, bool use_weights, device_array_view_impl const* xv,
                 device_array_view_impl const* yv, double alpha)
{
  const bool f32 = b.wtype == FLOAT32;
  B200_EXPECTS(xv->type == b.wtype && yv->type == b.wtype, CUGRAPH_INVALID_INPUT, "x / y dtype must match the block");
  B200_EXPECTS(xv->size >= padded_x_elems(b.n_span, f32 ? 4 : 8), CUGRAPH_INVALID_INPUT,
               "x must hold cugraph_b200_padded_elems(span) elements");
  B200_EXPECTS(yv->size >= (size_t)b.n_span, CUGRAPH_INVALID_INPUT, "y must hold `span` elements");
  const size_t es = f32 ? 4 : 8;
  auto const* x0  = static_cast<const char*>(xv->data);
  auto const* y0  = static_cast<const char*>(yv->data);
  B200_EXPECTS(y0 + yv->size * es <= x0 || x0 + xv->size * es <= y0, CUGRAPH_INVALID_INPUT, "x and y must not overlap");
  csx_t const* c      = b.csx.get();
  sweep_scratch_t* sc = &b.scratch;
  if (transposed) {
    block_push_t& p = push_copy(h, b);
    if (!p.sweep_ready) {  // the layout is built here rather than inside the first sweep, as cugraph_b200_block_create does
      p.scratch.init(h, *p.csx);
      prepare_pull_sweep(h, *p.csx, b.n_span, es);
      sync(h);
      p.sweep_ready = true;
    }
    c  = p.csx.get();
    sc = &p.scratch;
  }
  const int o             = transposed ? 1 : 0;
  const bool covered_only = b.y_complete[o] == yv->data;  // the empty slots of this y hold their zeros from an earlier sweep
  if (f32) pull_sweep<float>(h, *c, b.n_span, (float const*)xv->data, (float*)yv->data, *sc, alpha, use_weights, covered_only);
  else pull_sweep<double>(h, *c, b.n_span, (double const*)xv->data, (double*)yv->data, *sc, alpha, use_weights, covered_only);
  b.y_complete[o] = yv->data;
  if (b.y_complete[1 - o] == yv->data) b.y_complete[1 - o] = nullptr;  // this sweep wrote the other orientation's empty slots
}

// f(float{}) for FLOAT32, else f(double{}): the launchers' dispatch on the floating type of their (checked) arrays
template <typename F>
void by_float_type(cugraph_data_type_id_t t, F&& f)
{
  if (t == FLOAT32) f(float{});
  else f(double{});
}

// The frame of the owner steps (Katz, eigenvector, HITS, vertex sums and scaling; their kernels, in centrality_ops.cuh,
// are those of the single-GPU drivers).  Checks in this order: `partial` is not NULL; the arrays `vs` are not NULL, share
// one FLOAT32 / FLOAT64 type and hold n_local elements; the device scalars `ins` are not NULL.  Then, for n_local > 0,
// launch(h, T{}, n_local, grid) and the check of the launch.
template <typename F>
cugraph_error_code_t owner_step(cugraph_error_t** error, const char* what, const cugraph_resource_handle_t* handle,
                                std::initializer_list<device_array_view_impl const*> vs, size_t n_local, void const* partial,
                                std::initializer_list<void const*> ins, F&& launch)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(partial != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    const cugraph_data_type_id_t t = (*vs.begin()) ? (*vs.begin())->type : FLOAT32;
    for (auto const* v : vs) {
      B200_EXPECTS(v != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
      B200_EXPECTS(v->type == t && (t == FLOAT32 || t == FLOAT64), CUGRAPH_INVALID_INPUT, "arrays must share one FLOAT32 / FLOAT64 type");
      B200_EXPECTS(v->size >= n_local, CUGRAPH_INVALID_INPUT, "arrays shorter than n_local");
    }
    for (void const* p : ins) B200_EXPECTS(p != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    if (n_local == 0) return;
    by_float_type(t, [&](auto z) { launch(h, z, (int32_t)n_local, grid_for((int64_t)n_local, 1, h.sm_count * 8)); });
    check_last(what);
  });
}

// active rows -> queue (one read-back of its size and edge count) -> advance with `op`; returns the queue's counts
template <typename O, typename T, typename Op>
block_queue_counts_t block_push_round(handle_impl const& h, block_push_t& p, T const* dist_cols, Op op)
{
  csx_t const& pc = *p.csx;
  auto* cnt       = p.counts.as<block_queue_counts_t>();
  CUDA_TRY(cudaMemsetAsync(cnt, 0, sizeof(block_queue_counts_t), h.stream));
  if (p.n_ne > 0)
    B200_LAUNCH(h, (k_block_active_rows<O, T>), grid_for(p.n_ne, 1, h.sm_count * 8), kBlock, 0,
                pc.offsets.as<O>(), pc.row_vertex.as<int32_t>(), p.n_ne, dist_cols, p.queue.as<int32_t>(), p.q_deg.as<int32_t>(),
                cnt);
  const block_queue_counts_t hc = read_back(h, cnt);
  advance<O>(h, p.adv, pc.offsets.as<O>(), pc.indices.as<int32_t>(), p.queue.as<int32_t>(), hc.n, hc.edges, op,
             p.q_deg.as<int32_t>());
  return hc;
}

// out[row slot] = INT64_MAX (no proposal), then one push round of `op` over the columns active in `active_cols`
template <typename T, typename Op>
void block_push_min(handle_impl const& h, block_impl const& b, block_push_t& p, long long* out, T const* active_cols, Op op)
{
  B200_LAUNCH(h, k_fill<long long>, grid_for(b.n_rows, 1, h.sm_count * 8), kBlock, 0, out, (int64_t)b.n_rows, LLONG_MAX);
  if (p.csx->offs64) block_push_round<int64_t>(h, p, active_cols, op);
  else block_push_round<int32_t>(h, p, active_cols, op);
}

// ---- multi-GPU multi-source BFS (MGGraph.multi_source_bfs): one BFS per source of a batch of up to 64, bit j of a 64-bit
// word standing for source j (the words of single GPU's multi-source BFS, traverse.cu).  The launcher gathers the owners'
// `cur` words (the sources that reached a vertex at this level) over the block's column slots and their `seen` words over
// its row slots.  A level step, push or pull (the same arrays in and out), writes a partial `next` word per row slot; the
// launcher ORs the row group's partials at the owners (one all-to-all) and the owner step keeps the new bits and writes the
// distances.  The predecessor step is separate, so that push and pull share it and a run without predecessors skips it.
using u64 = unsigned long long;

inline u64 batch_mask(int n_sources) { return n_sources >= 64 ? ~0ull : (1ull << n_sources) - 1ull; }

// push: for every edge col -> row of a frontier column, the sources that reached col at this level and have not reached row
// (the MG form of ms_topdown_op, traverse.cu)
struct block_ms_push_op {
  int32_t const* col_of;  // column slot of a physical row of the push copy
  u64 const* cur;         // over column slots
  u64 const* seen;        // over row slots
  u64 mask;
  u64* next;              // over row slots, zeroed first
  __device__ __forceinline__ void edge(int src, long long, int nbr) const
  {
    const u64 bits = cur[col_of[src]] & ~seen[nbr] & mask;
    if (bits & ~next[nbr]) atomicOr(next + nbr, bits);  // next only gains bits during the step: a stale read costs an atomic
  }
};

__device__ __forceinline__ u64 warp_or_u64(u64 v)
{
  const unsigned lo = __reduce_or_sync(0xffffffffu, (unsigned)v);
  const unsigned hi = __reduce_or_sync(0xffffffffu, (unsigned)(v >> 32));
  return ((u64)hi << 32) | lo;
}

// pull: every row slot ORs cur over its columns into the bits it still wants (want = ~seen & mask) and stops once it has
// them all.  Rows of degree >= 32 (the prefix of the degree-ordered physical rows) take a warp each, 32 edges per step.
template <typename O>
__global__ void __launch_bounds__(256)
k_block_ms_pull_hi(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t n_hi,
                   u64 const* __restrict__ cur, u64 const* __restrict__ seen, u64 mask, u64* __restrict__ next)
{
  const int lane = threadIdx.x & 31;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < n_hi; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    const u64 want = ~seen[slot] & mask;
    if (!want) continue;  // warp-uniform
    const long long e1 = (long long)off[r + 1];
    u64 found          = 0;
    for (long long e0 = (long long)off[r]; e0 < e1; e0 += 32) {
      const long long e = e0 + lane;
      found |= warp_or_u64(e < e1 ? cur[idx[e]] & want : 0ull);
      if (found == want) break;
    }
    if (lane == 0 && found) next[slot] = found;
  }
}

template <typename O>
__global__ void __launch_bounds__(256)
k_block_ms_pull_low(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t r0,
                    int32_t r1, u64 const* __restrict__ cur, u64 const* __restrict__ seen, u64 mask, u64* __restrict__ next)
{
  for (long long r = r0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; r < r1; r += (long long)gridDim.x * blockDim.x) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    const u64 want = ~seen[slot] & mask;
    if (!want) continue;
    u64 found          = 0;
    const long long e1 = (long long)off[r + 1];
    for (long long e = (long long)off[r]; e < e1 && found != want; ++e) found |= cur[idx[e]] & want;
    if (found) next[slot] = found;
  }
}

template <typename O>
void block_ms_pull(handle_impl const& h, csx_t const& c, u64 const* cur, u64 const* seen, u64 mask, u64* next, int32_t n_row_slots)
{
  CUDA_TRY(cudaMemsetAsync(next, 0, sizeof(u64) * (size_t)n_row_slots, h.stream));
  const int32_t n_hi = c.degree_sorted ? c.seg[0] : 0;
  const int32_t n_ne = c.degree_sorted ? c.seg[kNumSeg - 2] : c.n_rows;  // rows with at least one edge
  if (n_hi > 0)
    B200_LAUNCH(h, (k_block_ms_pull_hi<O>), grid_for((int64_t)n_hi * 32, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, cur, seen, mask, next);
  if (n_ne > n_hi)
    B200_LAUNCH(h, (k_block_ms_pull_low<O>), grid_for(n_ne - n_hi, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, n_ne, cur, seen, mask, next);
}

// out[i] = popc(words[i])
__global__ void __launch_bounds__(kBlock) k_ms_popc(u64 const* __restrict__ words, long long n, long long* __restrict__ out)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __popcll(words[i]);
}

// scan[i] = the set bits of words[0, i): where the bits of word i start in a list of (word, bit) pairs
dbuf popc_scan(handle_impl const& h, u64 const* words, int64_t n)
{
  dbuf cnt = make_dbuf<long long>((size_t)std::max<int64_t>(n, 1), h.stream);
  dbuf scan = make_dbuf<long long>((size_t)std::max<int64_t>(n, 1), h.stream);
  if (n == 0) return scan;
  B200_LAUNCH(h, k_ms_popc, grid_for(n, 1, h.sm_count * 8), kBlock, 0, words, (long long)n, cnt.as<long long>());
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt.as<long long>(), scan.as<long long>(), n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, cnt.as<long long>(), scan.as<long long>(), n, h.stream));
  h.launches += 2;
  return scan;
}

// write `code` for every bit j of `win` at base + (the bits of b below j)
__device__ __forceinline__ void ms_write_pairs(u64 win, u64 b, long long base, long long lim, long long code, long long* pairs)
{
  while (win) {
    const int j         = __ffsll((long long)win) - 1;
    const long long pos = base + __popcll(b & ((1ull << j) - 1ull));
    if (pos < lim) pairs[pos] = code;
    win &= win - 1;
  }
}

// predecessors: for every row slot with new bits b and every bit j of b, the largest code of a column with bit j in cur.
// A row lists its columns in ascending slot order (build_binned_rows sorts by (row, column)) and the code grows with the slot,
// so a scan from the row's end that stops once every bit of b is found gives the maxima without atomics.  The pair of (row
// slot, bit j) goes to k * seg + (scan[slot] - scan[k * maxpart]) + popc(b below j), k = slot / maxpart: owner segment k,
// padded to seg entries; entries past seg are dropped.
struct ms_pairs_at {
  long long const* scan;
  long long maxpart, seg;
  __device__ __forceinline__ long long base(int slot) const
  {
    const long long k = slot / maxpart;
    return k * seg + scan[slot] - scan[k * maxpart];
  }
  __device__ __forceinline__ long long lim(int slot) const { return (slot / maxpart + 1) * seg; }
};

template <typename O>
__global__ void __launch_bounds__(256)
k_block_ms_pred_hi(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t n_hi,
                   u64 const* __restrict__ cur, u64 const* __restrict__ new_rows, ms_pairs_at at, int grid_cols, int grid_c,
                   long long* __restrict__ pairs)
{
  const int lane = threadIdx.x & 31;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < n_hi; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    const u64 b    = new_rows[slot];
    if (!b) continue;  // warp-uniform
    const long long base = at.base(slot), lim = at.lim(slot), e0 = (long long)off[r];
    u64 left             = b;
    // 32 edges per step from the row's end: lane 0 holds the largest column, so bit j goes to the lowest lane that has it
    for (long long e1 = (long long)off[r + 1]; e1 > e0 && left; e1 -= 32) {
      const long long e = e1 - 1 - lane;
      const int col     = e >= e0 ? idx[e] : 0;
      const u64 mine    = e >= e0 ? cur[col] & left : 0ull;
      u64 incl          = mine;  // inclusive prefix OR over the lanes
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const u64 t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl |= t;
      }
      const u64 before = __shfl_up_sync(0xffffffffu, incl, 1);
      const u64 win    = lane ? mine & ~before : mine;
      if (win) ms_write_pairs(win, b, base, lim, column_code(col, at.maxpart, grid_cols, grid_c), pairs);
      left &= ~__shfl_sync(0xffffffffu, incl, 31);
    }
  }
}

template <typename O>
__global__ void __launch_bounds__(256)
k_block_ms_pred_low(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t r0,
                    int32_t r1, u64 const* __restrict__ cur, u64 const* __restrict__ new_rows, ms_pairs_at at, int grid_cols,
                    int grid_c, long long* __restrict__ pairs)
{
  for (long long r = r0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; r < r1; r += (long long)gridDim.x * blockDim.x) {
    const int slot = row_vertex ? row_vertex[r] : (int)r;
    const u64 b    = new_rows[slot];
    if (!b) continue;
    const long long base = at.base(slot), lim = at.lim(slot), e0 = (long long)off[r];
    u64 left             = b;
    for (long long e = (long long)off[r + 1] - 1; e >= e0 && left; --e) {
      const int col = idx[e];
      const u64 win = cur[col] & left;
      if (!win) continue;
      ms_write_pairs(win, b, base, lim, column_code(col, at.maxpart, grid_cols, grid_c), pairs);
      left &= ~win;
    }
  }
}

template <typename O>
void block_ms_pred(handle_impl const& h, csx_t const& c, u64 const* cur, u64 const* new_rows, int32_t n_row_slots, long long maxpart,
                   int grid_cols, int grid_c, long long seg, long long* pairs)
{
  B200_LAUNCH(h, k_fill<long long>, grid_for(std::max<long long>(grid_cols * seg, 1), 1, h.sm_count * 8), kBlock, 0, pairs,
              (int64_t)grid_cols * seg, -1ll);
  if (n_row_slots == 0 || seg == 0) return;
  dbuf scan = popc_scan(h, new_rows, n_row_slots);
  const ms_pairs_at at{scan.as<long long>(), maxpart, seg};
  const int32_t n_hi = c.degree_sorted ? c.seg[0] : 0;
  const int32_t n_ne = c.degree_sorted ? c.seg[kNumSeg - 2] : c.n_rows;
  if (n_hi > 0)
    B200_LAUNCH(h, (k_block_ms_pred_hi<O>), grid_for((int64_t)n_hi * 32, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, cur, new_rows, at, grid_cols, grid_c, pairs);
  if (n_ne > n_hi)
    B200_LAUNCH(h, (k_block_ms_pred_low<O>), grid_for(n_ne - n_hi, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, n_ne, cur, new_rows, at, grid_cols, grid_c, pairs);
}

// owner step over the owned slots: next = OR of the `parts` received partials, new = next & ~seen, seen |= new, cur = new,
// dist[j][v] = level for every bit j of new; counts += (vertices with new bits, their out-degree sum, vertices whose seen
// became the whole batch, their in-degree sum, the new bits)
__global__ void __launch_bounds__(kBlock)
k_ms_owner_step(u64 const* __restrict__ recv, int parts, long long maxpart, int32_t n_local, u64 mask, int32_t level, u64* __restrict__ seen,
                u64* __restrict__ cur, int32_t* __restrict__ dist, long long const* __restrict__ deg_out,
                long long const* __restrict__ deg_in, unsigned long long* __restrict__ counts)
{
  u64 c_n = 0, c_m = 0, c_full = 0, c_in = 0, c_bits = 0;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_local; v += gridDim.x * blockDim.x) {
    u64 nxt = 0;
    for (int k = 0; k < parts; ++k) nxt |= recv[k * maxpart + v];
    const u64 s  = seen[v];
    const u64 nw = nxt & ~s & mask;
    cur[v]       = nw;
    if (!nw) continue;
    seen[v] = s | nw;
    for (u64 w = nw; w; w &= w - 1) dist[(long long)(__ffsll((long long)w) - 1) * n_local + v] = level;
    c_n += 1;
    c_bits += (u64)__popcll(nw);
    if (deg_out) c_m += (u64)deg_out[v];
    if ((s | nw) == mask) {
      c_full += 1;
      if (deg_in) c_in += (u64)deg_in[v];
    }
  }
  const u64 c[5] = {warp_sum_u64(c_n), warp_sum_u64(c_m), warp_sum_u64(c_full), warp_sum_u64(c_in), warp_sum_u64(c_bits)};
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 5; ++i)
      if (c[i]) atomicAdd(counts + i, c[i]);
}

// pred[j][v] = pairs[scan[v] + popc(new[v] below j)] for every bit j of new[v] (the owner's segment of the pair buffer)
__global__ void __launch_bounds__(kBlock)
k_ms_owner_pred(u64 const* __restrict__ nw, long long const* __restrict__ scan, int32_t n_local, long long const* __restrict__ pairs,
                long long n_pairs, long long* __restrict__ pred)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_local; v += gridDim.x * blockDim.x) {
    const u64 b = nw[v];
    for (u64 w = b; w; w &= w - 1) {
      const int j         = __ffsll((long long)w) - 1;
      const long long pos = scan[v] + __popcll(b & ((1ull << j) - 1ull));
      if (pos < n_pairs) pred[(long long)j * n_local + v] = pairs[pos];
    }
  }
}

// argument checks shared by the multi-source push and pull steps
void check_ms_bfs_block_args(block_impl const& b, device_array_view_impl const* cv, device_array_view_impl const* sv,
                             device_array_view_impl const* nv, int n_sources)
{
  B200_EXPECTS(cv->type == INT64 && sv->type == INT64 && nv->type == INT64, CUGRAPH_INVALID_INPUT,
               "cur_cols / seen_rows / next_rows must be INT64");
  B200_EXPECTS(cv->size >= (size_t)b.n_cols && sv->size >= (size_t)b.n_rows && nv->size >= (size_t)b.n_rows,
               CUGRAPH_INVALID_INPUT, "word arrays shorter than the block's slots");
  B200_EXPECTS(n_sources >= 1 && n_sources <= 64, CUGRAPH_INVALID_INPUT, "n_sources must be in [1, 64]");
}

template <typename T>
T rounded_cutoff(double cutoff)  // as cugraph_sssp rounds it (traverse.cu, sssp_windows)
{
  const T unreached = std::numeric_limits<T>::max();
  return cutoff >= (double)unreached ? unreached : (T)cutoff;
}

// argument checks shared by the two SSSP block calls; `dv` over column slots, `out` (INT64) over row slots
void check_sssp_block_args(block_impl const& b, device_array_view_impl const* dv, device_array_view_impl const* out, size_t maxpart,
                           int grid_cols, int grid_c)
{
  B200_EXPECTS(b.weighted, CUGRAPH_INVALID_INPUT, "SSSP requires a weighted block");
  B200_EXPECTS(dv->type == b.wtype, CUGRAPH_INVALID_INPUT, "dist_cols dtype must match the block's weights");
  B200_EXPECTS(out->type == INT64, CUGRAPH_INVALID_INPUT, "cand_rows / code_rows must be INT64");
  B200_EXPECTS(dv->size >= (size_t)b.n_cols && out->size >= (size_t)b.n_rows, CUGRAPH_INVALID_INPUT,
               "distance / candidate arrays shorter than the block's slots");
  B200_EXPECTS(maxpart > 0 && grid_cols > 0 && grid_c >= 0 && grid_c < grid_cols, CUGRAPH_INVALID_INPUT, "bad grid position");
}

// ---- one round of multi-GPU weakly connected components on this GPU's edge block (min-label propagation).  The launcher
// gathers the labels of the vertices that changed in the last round (INT64_MAX for all others) over the block's column
// slots; the push copy turns the active columns into a queue and the merge-path advance offers every active column's
// label to its rows with atomicMin, reduced to the owners by a MIN reduce-scatter.  A dense pull over the block's rows
// without atomics lost every round to this push on RMAT-24 and was removed (DESIGN §6).
struct block_wcc_op {
  int32_t const* col_of;  // column slot of a physical row of the push copy
  long long const* label;  // over column slots, INT64_MAX = inactive
  long long* cand;         // over row slots
  __device__ __forceinline__ void edge(int src, long long, int nbr) const
  {
    const long long l = label[col_of[src]];
    if (l < cand[nbr]) atomicMin(cand + nbr, l);  // a stale read is larger than the current value: never skips a win
  }
};

// ---- one round of multi-GPU strongly connected components on this GPU's edge block (MGGraph.strongly_connected_components).
// Forward (along u -> v) the sources are the column slots, and the push copy advances the active ones into row slots.
// Backward (along v -> u) the sources are the row slots, and the block's own rows (rows = destinations, neighbours =
// sources) advance the active ones into column slots.  An edge counts when its source is active (value != INT64_MIN), its
// two ends are different vertices (their global codes differ: self-loops are never live edges) and the source's key equals
// the destination's (subproblem or colour).  It then raises out[dst] to the source's value (max) or adds one to it (count).
constexpr int kSccPushMax = 0, kSccPushCount = 1;

// an SCC push value over the source slots; INT64_MIN = inactive (the launcher's values use the whole range above it)
struct scc_value_t {
  long long v;
};
__device__ __forceinline__ bool column_active(scc_value_t x) { return x.v != LLONG_MIN; }

struct block_scc_op {
  int32_t const* src_of;     // source slot of a physical row (column slot forward, row slot backward)
  long long const* key_src;  // over source slots
  long long const* val_src;
  long long const* key_dst;  // over destination slots
  int maxpart;                // < 2^31: 32-bit divisions (a 64-bit one is a call, whose frame spilled)
  int grid_cols, grid_r, grid_c;
  bool transposed;
  int mode;
  long long* out;            // over destination slots
  __device__ __forceinline__ void edge(int r, long long, int nbr) const
  {
    const int s = src_of[r];
    if (key_src[s] != key_dst[nbr]) return;
    const int col = transposed ? nbr : s, row = transposed ? s : nbr;
    // equal codes = equal owner ranks ((col / maxpart) * grid_cols + grid_c for the column, grid_r * grid_cols +
    // row / maxpart for the row, as column_code) and equal local ids
    const int cq = col / maxpart, rq = row / maxpart;
    if (col - cq * maxpart == row - rq * maxpart && (long long)cq * grid_cols + grid_c == (long long)grid_r * grid_cols + rq)
      return;
    if (mode == kSccPushCount) {
      atomicAdd((unsigned long long*)(out + nbr), 1ull);
    } else {
      const long long v = val_src[s];
      if (v > out[nbr]) atomicMax(out + nbr, v);  // a stale read is smaller than the current value: never skips a win
    }
  }
};

// the queue over the block's own rows, built on first use (block_push_t's queue, for the primary rows)
block_rows_queue_t& rows_queue(handle_impl const& h, block_impl& b)
{
  if (!b.rows_queue) {
    auto q         = std::make_unique<block_rows_queue_t>();
    csx_t const& c = *b.csx;
    q->n_ne        = c.degree_sorted ? c.seg[kNumSeg - 2] : c.n_rows;
    q->queue       = make_dbuf<int32_t>((size_t)std::max(c.n_rows, 1), h.stream);
    q->q_deg       = make_dbuf<int32_t>((size_t)c.n_rows + 1, h.stream);
    q->counts      = make_dbuf<block_queue_counts_t>(1, h.stream);
    q->adv.init(h, c.n_rows, c.nnz);
    sync(h);
    b.rows_queue = std::move(q);
  }
  return *b.rows_queue;
}

// active rows of the block itself -> queue (one read-back of its size and edge count) -> advance with `op` (the mirror of
// block_push_round over the primary rows)
template <typename O>
void block_rows_round(handle_impl const& h, csx_t const& c, block_rows_queue_t& q, scc_value_t const* vals, block_scc_op op)
{
  auto* cnt = q.counts.as<block_queue_counts_t>();
  CUDA_TRY(cudaMemsetAsync(cnt, 0, sizeof(block_queue_counts_t), h.stream));
  if (q.n_ne > 0)
    B200_LAUNCH(h, (k_block_active_rows<O, scc_value_t>), grid_for(q.n_ne, 1, h.sm_count * 8), kBlock, 0, c.offsets.as<O>(),
                c.row_vertex.as<int32_t>(), q.n_ne, vals, q.queue.as<int32_t>(), q.q_deg.as<int32_t>(), cnt);
  const block_queue_counts_t hc = read_back(h, cnt);
  advance<O>(h, q.adv, c.offsets.as<O>(), c.indices.as<int32_t>(), q.queue.as<int32_t>(), hc.n, hc.edges, op,
             q.q_deg.as<int32_t>());
}

// the block's edge counts per row slot (from the offsets, through row_vertex) and per column slot (a histogram)
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_block_degrees(O const* __restrict__ off, int32_t const* __restrict__ row_vertex, int32_t n_phys, int32_t const* __restrict__ idx,
                long long nnz, long long* __restrict__ row_deg, long long* __restrict__ col_deg)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz || i < n_phys; i += (long long)gridDim.x * blockDim.x) {
    if (i < n_phys) {
      const long long d = (long long)off[i + 1] - (long long)off[i];
      if (d) row_deg[row_vertex[i]] = d;   // a row slot with edges lies below n_rows
    }
    if (i < nnz) atomicAdd((unsigned long long*)(col_deg + idx[i]), 1ull);
  }
}

// ---- one position round of multi-GPU extract_paths (the MG walk of k_paths_walk, traverse.cu; reference: the gather rounds
// of extract_bfs_paths_impl.cuh:129-238).  An entry (row, pos, code) asks the owner of `code` (owner rank * maxpart + local
// id) for that vertex's external id, to be written at paths[row][pos], and for its predecessor's code, which continues the
// walk at pos - 1.  The launcher sends the requests' local ids to their owners and brings the answers back in request order.

// owner side: answers[2i] = external id, answers[2i + 1] = predecessor code (-1 = none) of local id lids[i]; (-1, -1) for a
// local id outside [0, n_local)
template <typename V>
__global__ void __launch_bounds__(kBlock)
k_paths_answer(int32_t const* __restrict__ lids, long long n, V const* __restrict__ vertices, long long const* __restrict__ pred_code,
               int32_t n_local, long long* __restrict__ answers)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t l = lids[i];
    const bool ok   = l >= 0 && l < n_local;
    answers[2 * i]     = ok ? (long long)vertices[l] : -1ll;
    answers[2 * i + 1] = ok ? pred_code[l] : -1ll;
  }
}

// whether an entry lies inside the paths matrix (entries outside it are dropped unwritten)
__device__ __forceinline__ bool paths_in_matrix(int32_t row, int32_t pos, long long n_paths_rows, long long len)
{
  return row >= 0 && row < n_paths_rows && pos >= 0 && pos < len;
}

// the owner rank of the request that follows an answered entry, -1 when its walk ends here: the position is 0, there is no
// predecessor, or the code names no rank
__device__ __forceinline__ int paths_next_rank(long long code, int32_t pos, long long maxpart, int world)
{
  if (pos <= 0 || code < 0) return -1;
  const long long q = code / maxpart;
  return q < world ? (int)q : -1;
}

// requester side, first pass: counts[q] = the next requests that go to rank q
__global__ void __launch_bounds__(kBlock)
k_paths_count(long long const* __restrict__ answers, int32_t const* __restrict__ rows, int32_t const* __restrict__ pos, long long n,
              long long n_paths_rows, long long len, long long maxpart, int world, long long* __restrict__ counts)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t p = pos[i];
    if (!paths_in_matrix(rows[i], p, n_paths_rows, len)) continue;
    const int q = paths_next_rank(answers[2 * i + 1], p, maxpart, world);
    if (q >= 0) atomicAdd((unsigned long long*)(counts + q), 1ull);
  }
}

// warp-aggregated append to one of several counters: the active lanes with the same key claim consecutive slots of it
__device__ __forceinline__ int warp_append_keyed(int* counters, int key)
{
  const unsigned peers = __match_any_sync(__activemask(), key);
  const int leader     = __ffs((int)peers) - 1;
  const int lane       = threadIdx.x & 31;
  int base             = 0;
  if (lane == leader) base = atomicAdd(counters + key, __popc(peers));
  base = __shfl_sync(peers, base, leader);
  return base + __popc(peers & ((1u << lane) - 1u));
}

// requester side, second pass: paths[row][pos] = the answered external id; the entries that go on are placed in rank
// order (bucket q starts at counts[0] + ... + counts[q - 1]; cursor[q] starts at 0) as (local id, row, pos - 1)
template <typename V>
__global__ void __launch_bounds__(kBlock)
k_paths_advance(long long const* __restrict__ answers, int32_t const* __restrict__ rows, int32_t const* __restrict__ pos, long long n,
                V* __restrict__ paths, long long n_paths_rows, long long len, long long maxpart, int world,
                long long const* __restrict__ counts, int* __restrict__ cursor, int32_t* __restrict__ next_lid,
                int32_t* __restrict__ next_row, int32_t* __restrict__ next_pos)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t r = rows[i], p = pos[i];
    if (!paths_in_matrix(r, p, n_paths_rows, len)) continue;
    const long long code = answers[2 * i + 1];
    paths[r * len + p]   = (V)answers[2 * i];
    const int q          = paths_next_rank(code, p, maxpart, world);
    if (q < 0) continue;
    long long at = 0;
    for (int k = 0; k < q; ++k) at += counts[k];
    at += warp_append_keyed(cursor, q);
    next_lid[at] = (int32_t)(code - (long long)q * maxpart);
    next_row[at] = r;
    next_pos[at] = p - 1;
  }
}

// the two PageRank owner-step entry points: argument checks and the launch (pv == nullptr: uniform teleport)
void pagerank_vertex_step(handle_impl const& h, device_array_view_impl const* yv, device_array_view_impl const* pv,
                          device_array_view_impl const* ov, device_array_view_impl const* xv,
                          device_array_view_impl const* persv, size_t n_local, double alpha, double n_vertices_global,
                          double pers_sum, bool_t first, double const* totals_prev, double* partial_out)
{
  B200_EXPECTS(pv->type == yv->type && ov->type == yv->type && xv->type == yv->type && (!persv || persv->type == yv->type),
               CUGRAPH_INVALID_INPUT, "dtype mismatch");
  B200_EXPECTS(yv->size >= n_local && pv->size >= n_local && ov->size >= n_local && xv->size >= n_local &&
                 (!persv || persv->size >= n_local),
               CUGRAPH_INVALID_INPUT, "arrays shorter than n_local");
  if (n_local == 0) return;
  by_float_type(yv->type, [&](auto z) {
    using T = decltype(z);
    auto* kernel = persv ? k_mg_vertex_step<T, true> : k_mg_vertex_step<T, false>;
    B200_LAUNCH(h, kernel, grid_for((int64_t)n_local, 1, h.sm_count * 8), kBlock, 0, (T const*)yv->data, (T*)pv->data, (T const*)ov->data, (T*)xv->data,
                persv ? (T const*)persv->data : nullptr, (int32_t)n_local, alpha, n_vertices_global, pers_sum,
                first == TRUE ? 1 : 0, totals_prev, partial_out);
  });
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t cugraph_b200_padded_elems(size_t n, size_t elem_size) { return padded_x_elems((int32_t)n, elem_size); }

cugraph_error_code_t cugraph_b200_block_create(const cugraph_resource_handle_t* handle, size_t n_rows, size_t n_cols,
                                               const cugraph_type_erased_device_array_view_t* rows,
                                               const cugraph_type_erased_device_array_view_t* cols,
                                               const cugraph_type_erased_device_array_view_t* weights,
                                               cugraph_b200_block_t** block, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && rows && cols, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* r = V(rows);
    auto const* c = V(cols);
    auto const* w = V(weights);
    B200_EXPECTS(r->type == INT32 && c->type == INT32 && r->size == c->size, CUGRAPH_INVALID_INPUT,
                 "block rows / cols must be INT32 arrays of equal size");
    B200_EXPECTS(w == nullptr || ((w->type == FLOAT32 || w->type == FLOAT64) && w->size == r->size), CUGRAPH_INVALID_INPUT,
                 "block weights must be FLOAT32 / FLOAT64 with one value per edge");
    B200_EXPECTS(n_rows < (1u << 31) && n_cols < (1u << 31), CUGRAPH_INVALID_INPUT, "block too large");
    auto b     = std::make_unique<block_impl>();
    b->n_rows  = (int32_t)n_rows;
    b->n_cols  = (int32_t)n_cols;
    b->n_span  = (int32_t)std::max(n_rows, n_cols);
    b->wtype   = w ? w->type : FLOAT32;
    b->weighted = w != nullptr;
    b->csx     = build_binned_rows(h, (int32_t const*)r->data, (int32_t const*)c->data, w ? w->data : nullptr, b->wtype,
                                   (int64_t)r->size, b->n_span);
    b->scratch.init(h, *b->csx);
    // build the column-blocked copy now (it is lazily created otherwise, inside the first timed sweep)
    prepare_pull_sweep(h, *b->csx, b->n_span, b->wtype == FLOAT64 ? 8 : 4);
    sync(h);
    *block = reinterpret_cast<cugraph_b200_block_t*>(b.release());
  });
}

cugraph_error_code_t cugraph_b200_block_stage_edges(const cugraph_resource_handle_t* handle, size_t n_rows, size_t n_cols,
                                                    cugraph_type_erased_device_array_view_t* rows,
                                                    cugraph_type_erased_device_array_view_t* cols,
                                                    const cugraph_type_erased_device_array_view_t* reversed,
                                                    cugraph_type_erased_device_array_view_t* weights, bool_t drop_multi_edges,
                                                    bool_t symmetrize, size_t* n_out, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(rows && cols && n_out, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* r = V(rows);
    auto const* c = V(cols);
    auto const* f = V(reversed);
    auto const* w = V(weights);
    B200_EXPECTS(r->type == INT32 && c->type == INT32 && r->size == c->size, CUGRAPH_INVALID_INPUT,
                 "block rows / cols must be INT32 arrays of equal size");
    B200_EXPECTS(f == nullptr || (dtype_size(f->type) == 1 && f->size == r->size), CUGRAPH_INVALID_INPUT,
                 "reversed must hold one byte flag per edge");
    B200_EXPECTS(w == nullptr || ((w->type == FLOAT32 || w->type == FLOAT64) && w->size == r->size), CUGRAPH_INVALID_INPUT,
                 "block weights must be FLOAT32 / FLOAT64 with one value per edge");
    B200_EXPECTS(n_rows < (1u << 31) && n_cols < (1u << 31), CUGRAPH_INVALID_INPUT, "block too large");
    *n_out = (size_t)stage_block_edges(h, (int32_t)n_rows, (int32_t)n_cols, (int32_t*)r->data, (int32_t*)c->data,
                                       f ? (uint8_t const*)f->data : nullptr, w ? w->data : nullptr, w ? w->type : FLOAT32,
                                       (int64_t)r->size, drop_multi_edges == TRUE, symmetrize == TRUE);
  });
}

cugraph_error_code_t cugraph_b200_block_degrees(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                cugraph_type_erased_device_array_view_t* row_counts,
                                                cugraph_type_erased_device_array_view_t* col_counts, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && row_counts && col_counts, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* b  = reinterpret_cast<block_impl const*>(block);
    auto const* rv = V(row_counts);
    auto const* cv = V(col_counts);
    B200_EXPECTS(rv->type == INT64 && cv->type == INT64, CUGRAPH_INVALID_INPUT, "row_counts / col_counts must be INT64");
    B200_EXPECTS(rv->size >= (size_t)b->n_rows && cv->size >= (size_t)b->n_cols, CUGRAPH_INVALID_INPUT,
                 "count arrays shorter than the block's slots");
    CUDA_TRY(cudaMemsetAsync(rv->data, 0, (size_t)b->n_rows * sizeof(long long), h.stream));
    CUDA_TRY(cudaMemsetAsync(cv->data, 0, (size_t)b->n_cols * sizeof(long long), h.stream));
    csx_t const& c   = *b->csx;
    const long long n = std::max<long long>(c.nnz, c.n_rows);
    if (n == 0) return;
    const int grid = grid_for(n, 1, h.sm_count * 8);
    if (c.offs64)
      B200_LAUNCH(h, k_block_degrees<int64_t>, grid, kBlock, 0, c.offsets.as<int64_t>(), c.row_vertex.as<int32_t>(), c.n_rows,
                  c.indices.as<int32_t>(), (long long)c.nnz, (long long*)rv->data, (long long*)cv->data);
    else
      B200_LAUNCH(h, k_block_degrees<int32_t>, grid, kBlock, 0, c.offsets.as<int32_t>(), c.row_vertex.as<int32_t>(), c.n_rows,
                  c.indices.as<int32_t>(), (long long)c.nnz, (long long*)rv->data, (long long*)cv->data);
    check_last("block_degrees");
  });
}

void cugraph_b200_block_free(cugraph_b200_block_t* block)
{
  if (block) delete reinterpret_cast<block_impl*>(block);
}

size_t cugraph_b200_block_span(const cugraph_b200_block_t* block)
{
  return block ? (size_t) reinterpret_cast<block_impl const*>(block)->n_span : 0;
}

// y[row] = alpha * sum_{edges (row, col)} x[col] * w ; rows without edges get 0.  Asynchronous.
cugraph_error_code_t cugraph_b200_block_pull_sweep(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                   const cugraph_type_erased_device_array_view_t* x,
                                                   cugraph_type_erased_device_array_view_t* y, double alpha,
                                                   cugraph_error_t** error)
{
  return cugraph_b200_block_sweep(handle, block, FALSE, TRUE, x, y, alpha, error);
}

// transposed = FALSE: y[row] = alpha * sum_{edges (row, col)} x[col] * w ; TRUE: y[col] = alpha * sum_{edges (row, col)} x[row] * w
// (w = 1 when use_weights is FALSE).  Asynchronous, apart from the first transposed sweep of a block.
cugraph_error_code_t cugraph_b200_block_sweep(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                              bool_t transposed, bool_t use_weights,
                                              const cugraph_type_erased_device_array_view_t* x,
                                              cugraph_type_erased_device_array_view_t* y, double alpha, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && x && y, CUGRAPH_INVALID_INPUT, "NULL argument");
    block_sweep(h, *reinterpret_cast<block_impl*>(block), transposed == TRUE, use_weights == TRUE, V(x), V(y), alpha);
    check_last("block_sweep");
  });
}

cugraph_error_code_t cugraph_b200_katz_step(const cugraph_resource_handle_t* handle,
                                            const cugraph_type_erased_device_array_view_t* y,
                                            cugraph_type_erased_device_array_view_t* x, size_t n_local, double beta,
                                            double* partial_out_device, cugraph_error_t** error)
{
  auto const *yv = V(y), *xv = V(x);
  return owner_step(error, "katz_step", handle, {yv, xv}, n_local, partial_out_device, {}, [&](auto const& h, auto z, int32_t n, int grid) {
    using T = decltype(z);
    B200_LAUNCH(h, k_katz_step<T>, grid, kBlock, 0, (T const*)yv->data, (T*)xv->data, n, beta, partial_out_device);
  });
}

cugraph_error_code_t cugraph_b200_eigenvector_add_step(const cugraph_resource_handle_t* handle,
                                                       cugraph_type_erased_device_array_view_t* y,
                                                       const cugraph_type_erased_device_array_view_t* x, size_t n_local,
                                                       double* partial_out_device, cugraph_error_t** error)
{
  auto const *yv = V(y), *xv = V(x);
  return owner_step(error, "eigenvector_add_step", handle, {yv, xv}, n_local, partial_out_device, {},
                    [&](auto const& h, auto z, int32_t n, int grid) {
                      using T = decltype(z);
                      B200_LAUNCH(h, k_eig_add<T>, grid, kBlock, 0, (T*)yv->data, (T const*)xv->data, n, partial_out_device);
                    });
}

cugraph_error_code_t cugraph_b200_eigenvector_scale_step(const cugraph_resource_handle_t* handle,
                                                         cugraph_type_erased_device_array_view_t* y,
                                                         cugraph_type_erased_device_array_view_t* x, size_t n_local,
                                                         const double* sumsq_device, double* partial_out_device,
                                                         cugraph_error_t** error)
{
  auto const *yv = V(y), *xv = V(x);
  return owner_step(error, "eigenvector_scale_step", handle, {yv, xv}, n_local, partial_out_device, {sumsq_device},
                    [&](auto const& h, auto z, int32_t n, int grid) {
                      using T = decltype(z);
                      B200_LAUNCH(h, k_eig_scale<T>, grid, kBlock, 0, (T*)yv->data, (T*)xv->data, n, sumsq_device,
                                  partial_out_device);
                    });
}

cugraph_error_code_t cugraph_b200_hits_max_step(const cugraph_resource_handle_t* handle,
                                                const cugraph_type_erased_device_array_view_t* hubs,
                                                const cugraph_type_erased_device_array_view_t* authorities, size_t n_local,
                                                double* max_out_device, cugraph_error_t** error)
{
  auto const *hv = V(hubs), *av = V(authorities);
  return owner_step(error, "hits_max_step", handle, {hv, av}, n_local, max_out_device, {},
                    [&](auto const& h, auto z, int32_t n, int grid) {
                      using T = decltype(z);
                      B200_LAUNCH(h, k_hits_max<T>, grid, kBlock, 0, (T const*)hv->data, (T const*)av->data, n, max_out_device);
                    });
}

cugraph_error_code_t cugraph_b200_hits_scale_step(const cugraph_resource_handle_t* handle,
                                                  cugraph_type_erased_device_array_view_t* hubs,
                                                  cugraph_type_erased_device_array_view_t* authorities,
                                                  const cugraph_type_erased_device_array_view_t* prev_hubs, size_t n_local,
                                                  const double* max_device, double* partial_out_device, cugraph_error_t** error)
{
  auto const *hv = V(hubs), *av = V(authorities), *pv = V(prev_hubs);
  return owner_step(error, "hits_scale_step", handle, {hv, av, pv}, n_local, partial_out_device, {max_device},
                    [&](auto const& h, auto z, int32_t n, int grid) {
                      using T = decltype(z);
                      B200_LAUNCH(h, k_hits_scale<T>, grid, kBlock, 0, (T*)hv->data, (T*)av->data, (T const*)pv->data, n,
                                  max_device, partial_out_device);
                    });
}

cugraph_error_code_t cugraph_b200_vertex_sum(const cugraph_resource_handle_t* handle,
                                             const cugraph_type_erased_device_array_view_t* v, size_t n_local, bool_t squares,
                                             double* partial_out_device, cugraph_error_t** error)
{
  auto const* vv = V(v);
  const int mode = squares == TRUE ? 0 : 1;
  return owner_step(error, "vertex_sum", handle, {vv}, n_local, partial_out_device, {},
                    [&](auto const& h, auto z, int32_t n, int grid) {
                      using T = decltype(z);
                      B200_LAUNCH(h, k_norm<T>, grid, kBlock, 0, (T const*)vv->data, n, mode, partial_out_device);
                    });
}

cugraph_error_code_t cugraph_b200_vertex_scale(const cugraph_resource_handle_t* handle, cugraph_type_erased_device_array_view_t* v,
                                               size_t n_local, double inv, cugraph_error_t** error)
{
  auto const* vv = V(v);
  return owner_step(error, "vertex_scale", handle, {vv}, n_local, &inv, {}, [&](auto const& h, auto z, int32_t n, int grid) {
    using T = decltype(z);
    B200_LAUNCH(h, k_scale<T>, grid, kBlock, 0, (T*)vv->data, n, inv);
  });
}

cugraph_error_code_t cugraph_b200_pagerank_vertex_step(const cugraph_resource_handle_t* handle,
                                                       const cugraph_type_erased_device_array_view_t* y,
                                                       cugraph_type_erased_device_array_view_t* pr,
                                                       const cugraph_type_erased_device_array_view_t* out_w,
                                                       cugraph_type_erased_device_array_view_t* x, size_t n_local,
                                                       double alpha, double n_vertices_global, bool_t first,
                                                       const double* totals_prev_device, double* partial_out_device,
                                                       cugraph_error_t** error)
{
  return guarded(error, [&] {
    B200_EXPECTS(y && pr && out_w && x && partial_out_device, CUGRAPH_INVALID_INPUT, "NULL argument");
    pagerank_vertex_step(H(handle), V(y), V(pr), V(out_w), V(x), nullptr, n_local, alpha, n_vertices_global, 1.0, first,
                         totals_prev_device, partial_out_device);
    check_last("pagerank_vertex_step");
  });
}

cugraph_error_code_t cugraph_b200_pagerank_personalized_vertex_step(const cugraph_resource_handle_t* handle,
                                                                    const cugraph_type_erased_device_array_view_t* y,
                                                                    cugraph_type_erased_device_array_view_t* pr,
                                                                    const cugraph_type_erased_device_array_view_t* out_w,
                                                                    cugraph_type_erased_device_array_view_t* x,
                                                                    const cugraph_type_erased_device_array_view_t* pers,
                                                                    size_t n_local, double alpha, double pers_sum,
                                                                    bool_t first, const double* totals_prev_device,
                                                                    double* partial_out_device, cugraph_error_t** error)
{
  return guarded(error, [&] {
    B200_EXPECTS(y && pr && out_w && x && pers && partial_out_device && (first == TRUE || totals_prev_device),
                 CUGRAPH_INVALID_INPUT, "NULL argument");
    B200_EXPECTS(pers_sum > 0.0, CUGRAPH_INVALID_INPUT, "pers_sum must be positive");
    pagerank_vertex_step(H(handle), V(y), V(pr), V(out_w), V(x), V(pers), n_local, alpha, 1.0, pers_sum, first,
                         totals_prev_device, partial_out_device);
    check_last("pagerank_personalized_vertex_step");
  });
}

// cand[row slot] = global code of a frontier source adjacent to that (unvisited) row, or -1.  Asynchronous.
cugraph_error_code_t cugraph_b200_block_bfs_pull(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                 const cugraph_type_erased_device_array_view_t* frontier_cols,
                                                 const cugraph_type_erased_device_array_view_t* visited_rows, size_t maxpart,
                                                 int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* cand,
                                                 cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && frontier_cols && visited_rows && cand, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* fv = V(frontier_cols);
    auto const* vv = V(visited_rows);
    auto const* cv = V(cand);
    check_bfs_block_args(*b, fv, vv, cv, maxpart, grid_cols, grid_c);
    csx_t const& c = *b->csx;
    if (c.offs64)
      block_bfs_pull<int64_t>(h, c, (uint8_t const*)fv->data, (uint8_t const*)vv->data, (long long)maxpart, grid_cols, grid_c,
                              (long long*)cv->data, b->n_rows);
    else
      block_bfs_pull<int32_t>(h, c, (uint8_t const*)fv->data, (uint8_t const*)vv->data, (long long)maxpart, grid_cols, grid_c,
                              (long long*)cv->data, b->n_rows);
    check_last("block_bfs_pull");
  });
}

// cand[row slot] = largest global code of a frontier source of that (unvisited) row, or -1.  Asynchronous, apart from the
// read-back of the queue size (and the first call's push copy).
cugraph_error_code_t cugraph_b200_block_bfs_push(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                 const cugraph_type_erased_device_array_view_t* frontier_cols,
                                                 const cugraph_type_erased_device_array_view_t* visited_rows, size_t maxpart,
                                                 int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* cand,
                                                 cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && frontier_cols && visited_rows && cand, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* fv = V(frontier_cols);
    auto const* vv = V(visited_rows);
    auto const* cv = V(cand);
    check_bfs_block_args(*b, fv, vv, cv, maxpart, grid_cols, grid_c);
    auto* out = (long long*)cv->data;
    B200_LAUNCH(h, k_fill<long long>, grid_for(b->n_rows, 1, h.sm_count * 8), kBlock, 0, out, (int64_t)b->n_rows, -1ll);
    block_push_t& p     = push_copy(h, *b);
    auto const* front   = (uint8_t const*)fv->data;
    const block_bfs_push_op op{p.csx->row_vertex.as<int32_t>(), (uint8_t const*)vv->data, (long long)maxpart, grid_cols, grid_c,
                               out};
    if (p.csx->offs64) block_push_round<int64_t>(h, p, front, op);
    else block_push_round<int32_t>(h, p, front, op);
    check_last("block_bfs_push");
  });
}

// whether a direction-optimising BFS level runs bottom-up (bfs_bottom_up, common.cuh, with the handle's knobs)
bool_t cugraph_b200_bfs_bottom_up(const cugraph_resource_handle_t* handle, bool_t bottom_up_now, size_t n_f, size_t prev_n_f,
                                  size_t m_f, size_t m_u, size_t n_unvisited)
{
  if (!handle) return bottom_up_now;
  return bfs_bottom_up(H(handle), bottom_up_now == TRUE, (long long)n_f, (long long)prev_n_f, (unsigned long long)m_f,
                       (unsigned long long)m_u, (long long)n_unvisited)
           ? TRUE
           : FALSE;
}

// next_rows[row slot] = the batch bits of the frontier columns of that row which the row has not seen.  Asynchronous, apart
// from the read-back of the queue size (and the first call's push copy).
cugraph_error_code_t cugraph_b200_block_ms_bfs_push(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                    const cugraph_type_erased_device_array_view_t* cur_cols,
                                                    const cugraph_type_erased_device_array_view_t* seen_rows, int n_sources,
                                                    cugraph_type_erased_device_array_view_t* next_rows, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && cur_cols && seen_rows && next_rows, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* cv = V(cur_cols);
    auto const* sv = V(seen_rows);
    auto const* nv = V(next_rows);
    check_ms_bfs_block_args(*b, cv, sv, nv, n_sources);
    auto* next = (u64*)nv->data;
    CUDA_TRY(cudaMemsetAsync(next, 0, sizeof(u64) * (size_t)b->n_rows, h.stream));
    block_push_t& p = push_copy(h, *b);
    auto const* cur = (u64 const*)cv->data;
    const block_ms_push_op op{p.csx->row_vertex.as<int32_t>(), cur, (u64 const*)sv->data, batch_mask(n_sources), next};
    if (p.csx->offs64) block_push_round<int64_t>(h, p, cur, op);
    else block_push_round<int32_t>(h, p, cur, op);
    check_last("block_ms_bfs_push");
  });
}

// the same words by the block's own rows (pull direction).  Asynchronous.
cugraph_error_code_t cugraph_b200_block_ms_bfs_pull(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                    const cugraph_type_erased_device_array_view_t* cur_cols,
                                                    const cugraph_type_erased_device_array_view_t* seen_rows, int n_sources,
                                                    cugraph_type_erased_device_array_view_t* next_rows, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && cur_cols && seen_rows && next_rows, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* cv = V(cur_cols);
    auto const* sv = V(seen_rows);
    auto const* nv = V(next_rows);
    check_ms_bfs_block_args(*b, cv, sv, nv, n_sources);
    csx_t const& c = *b->csx;
    auto const* cur  = (u64 const*)cv->data;
    auto const* seen = (u64 const*)sv->data;
    if (c.offs64) block_ms_pull<int64_t>(h, c, cur, seen, batch_mask(n_sources), (u64*)nv->data, b->n_rows);
    else block_ms_pull<int32_t>(h, c, cur, seen, batch_mask(n_sources), (u64*)nv->data, b->n_rows);
    check_last("block_ms_bfs_pull");
  });
}

// pairs[k * seg + ...] = for every row slot with new bits and every such bit, the largest code of a column of that row with
// the bit in cur_cols, else -1.  Asynchronous.
cugraph_error_code_t cugraph_b200_block_ms_bfs_pred(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                    const cugraph_type_erased_device_array_view_t* cur_cols,
                                                    const cugraph_type_erased_device_array_view_t* new_rows, size_t maxpart,
                                                    int grid_cols, int grid_c, size_t seg,
                                                    cugraph_type_erased_device_array_view_t* pairs, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && cur_cols && new_rows && pairs, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* cv = V(cur_cols);
    auto const* nv = V(new_rows);
    auto const* pv = V(pairs);
    B200_EXPECTS(cv->type == INT64 && nv->type == INT64 && pv->type == INT64, CUGRAPH_INVALID_INPUT,
                 "cur_cols / new_rows / pairs must be INT64");
    B200_EXPECTS(maxpart > 0 && grid_cols > 0 && grid_c >= 0 && grid_c < grid_cols, CUGRAPH_INVALID_INPUT, "bad grid position");
    B200_EXPECTS((size_t)b->n_rows <= (size_t)grid_cols * maxpart, CUGRAPH_INVALID_INPUT,
                 "the block has more row slots than grid_cols * maxpart");
    B200_EXPECTS(cv->size >= (size_t)b->n_cols && nv->size >= (size_t)b->n_rows, CUGRAPH_INVALID_INPUT,
                 "word arrays shorter than the block's slots");
    B200_EXPECTS(pv->size >= (size_t)grid_cols * seg, CUGRAPH_INVALID_INPUT, "pairs must hold grid_cols * seg entries");
    csx_t const& c = *b->csx;
    auto const* cur = (u64 const*)cv->data;
    auto const* nw  = (u64 const*)nv->data;
    if (c.offs64)
      block_ms_pred<int64_t>(h, c, cur, nw, b->n_rows, (long long)maxpart, grid_cols, grid_c, (long long)seg, (long long*)pv->data);
    else
      block_ms_pred<int32_t>(h, c, cur, nw, b->n_rows, (long long)maxpart, grid_cols, grid_c, (long long)seg, (long long*)pv->data);
    check_last("block_ms_bfs_pred");
  });
}

// the owners' level update of a multi-source BFS batch (see k_ms_owner_step); counts[0..5) are overwritten.  Asynchronous.
cugraph_error_code_t cugraph_b200_ms_bfs_owner_step(const cugraph_resource_handle_t* handle,
                                                    const cugraph_type_erased_device_array_view_t* recv, int parts, size_t maxpart,
                                                    size_t n_local, int n_sources, int level,
                                                    cugraph_type_erased_device_array_view_t* seen,
                                                    cugraph_type_erased_device_array_view_t* cur,
                                                    cugraph_type_erased_device_array_view_t* distances,
                                                    const cugraph_type_erased_device_array_view_t* deg_out,
                                                    const cugraph_type_erased_device_array_view_t* deg_in,
                                                    cugraph_type_erased_device_array_view_t* counts, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(recv && seen && cur && distances && counts, CUGRAPH_INVALID_INPUT, "NULL argument");
    B200_EXPECTS((deg_out == nullptr) == (deg_in == nullptr), CUGRAPH_INVALID_INPUT, "give both degree arrays or neither");
    auto const* rv = V(recv);
    auto const* sv = V(seen);
    auto const* cv = V(cur);
    auto const* dv = V(distances);
    auto const* kv = V(counts);
    B200_EXPECTS(rv->type == INT64 && sv->type == INT64 && cv->type == INT64 && kv->type == INT64, CUGRAPH_INVALID_INPUT,
                 "recv / seen / cur / counts must be INT64");
    B200_EXPECTS(dv->type == INT32, CUGRAPH_INVALID_INPUT, "distances must be INT32");
    B200_EXPECTS(n_sources >= 1 && n_sources <= 64, CUGRAPH_INVALID_INPUT, "n_sources must be in [1, 64]");
    B200_EXPECTS(parts > 0 && maxpart > 0 && n_local <= maxpart && n_local < (1u << 31) && level > 0, CUGRAPH_INVALID_INPUT,
                 "bad parts / maxpart / n_local / level");
    B200_EXPECTS(rv->size >= (size_t)parts * maxpart, CUGRAPH_INVALID_INPUT, "recv must hold parts * maxpart words");
    B200_EXPECTS(sv->size >= n_local && cv->size >= n_local, CUGRAPH_INVALID_INPUT, "seen / cur shorter than n_local");
    B200_EXPECTS(dv->size >= (size_t)n_sources * n_local, CUGRAPH_INVALID_INPUT, "distances must hold n_sources * n_local");
    B200_EXPECTS(kv->size >= 5, CUGRAPH_INVALID_INPUT, "counts must hold 5 entries");
    long long const *dout = nullptr, *din = nullptr;
    if (deg_out) {
      auto const* ov = V(deg_out);
      auto const* iv = V(deg_in);
      B200_EXPECTS(ov->type == INT64 && iv->type == INT64 && ov->size >= n_local && iv->size >= n_local, CUGRAPH_INVALID_INPUT,
                   "degrees must be INT64 arrays of n_local entries");
      dout = (long long const*)ov->data;
      din  = (long long const*)iv->data;
    }
    auto* cnt = (unsigned long long*)kv->data;
    CUDA_TRY(cudaMemsetAsync(cnt, 0, 5 * sizeof(long long), h.stream));
    if (n_local == 0) return;
    B200_LAUNCH(h, k_ms_owner_step, grid_for((int64_t)n_local, 1, h.sm_count * 8), kBlock, 0, (u64 const*)rv->data, parts,
                (long long)maxpart, (int32_t)n_local, batch_mask(n_sources), level, (u64*)sv->data, (u64*)cv->data,
                (int32_t*)dv->data, dout, din, cnt);
    check_last("ms_bfs_owner_step");
  });
}

// pred[j * n_local + v] = the owner's pair of (v, bit j) for every bit j of new_words[v].  Asynchronous.
cugraph_error_code_t cugraph_b200_ms_bfs_owner_pred(const cugraph_resource_handle_t* handle,
                                                    const cugraph_type_erased_device_array_view_t* new_words,
                                                    const cugraph_type_erased_device_array_view_t* pairs, size_t n_local,
                                                    int n_sources, cugraph_type_erased_device_array_view_t* predecessors,
                                                    cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(new_words && pairs && predecessors, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* nv = V(new_words);
    auto const* av = V(pairs);
    auto const* pv = V(predecessors);
    B200_EXPECTS(nv->type == INT64 && av->type == INT64 && pv->type == INT64, CUGRAPH_INVALID_INPUT,
                 "new_words / pairs / predecessors must be INT64");
    B200_EXPECTS(n_sources >= 1 && n_sources <= 64, CUGRAPH_INVALID_INPUT, "n_sources must be in [1, 64]");
    B200_EXPECTS(n_local < (1u << 31) && nv->size >= n_local, CUGRAPH_INVALID_INPUT, "new_words shorter than n_local");
    B200_EXPECTS(pv->size >= (size_t)n_sources * n_local, CUGRAPH_INVALID_INPUT, "predecessors must hold n_sources * n_local");
    if (n_local == 0) return;
    auto const* nw = (u64 const*)nv->data;
    dbuf scan      = popc_scan(h, nw, (int64_t)n_local);
    B200_LAUNCH(h, k_ms_owner_pred, grid_for((int64_t)n_local, 1, h.sm_count * 8), kBlock, 0, nw, scan.as<long long>(),
                (int32_t)n_local, (long long const*)av->data, (long long)av->size, (long long*)pv->data);
    check_last("ms_bfs_owner_pred");
  });
}

// cand_rows[row slot] = min key over the proposals dist_cols[col] + w < cutoff of the active columns, else INT64_MAX
cugraph_error_code_t cugraph_b200_block_sssp_relax(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                   const cugraph_type_erased_device_array_view_t* dist_cols, double cutoff,
                                                   size_t maxpart, int grid_cols, int grid_c,
                                                   cugraph_type_erased_device_array_view_t* cand_rows, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && dist_cols && cand_rows, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* dv = V(dist_cols);
    auto const* cv = V(cand_rows);
    check_sssp_block_args(*b, dv, cv, maxpart, grid_cols, grid_c);
    if (b->wtype == FLOAT32) {  // the code takes the low 32 bits of the key
      const unsigned long long parts = (((unsigned long long)b->n_cols + maxpart - 1) / maxpart) * (unsigned long long)grid_cols;
      B200_EXPECTS(maxpart < (1ull << 32) && parts <= ((1ull << 32) - 1) / maxpart, CUGRAPH_INVALID_INPUT,
                   "FLOAT32 SSSP keys need R * grid_cols * maxpart < 2^32");
    }
    block_push_t& p = push_copy(h, *b);
    auto* cand      = (long long*)cv->data;
    by_float_type(b->wtype, [&](auto z) {
      using T       = decltype(z);
      auto const* d = (T const*)dv->data;
      block_push_min(h, *b, p, cand, d,
                     block_relax_op<T>{p.csx->row_vertex.as<int32_t>(), p.csx->weights.as<T>(), d, rounded_cutoff<T>(cutoff),
                                       (long long)maxpart, grid_cols, grid_c, cand});
    });
    check_last("block_sssp_relax");
  });
}

// code_rows[row slot] = smallest code of an active column with dist_cols[col] + w == win_rows[row], else INT64_MAX
cugraph_error_code_t cugraph_b200_block_sssp_pred(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                  const cugraph_type_erased_device_array_view_t* dist_cols,
                                                  const cugraph_type_erased_device_array_view_t* win_rows, size_t maxpart,
                                                  int grid_cols, int grid_c, cugraph_type_erased_device_array_view_t* code_rows,
                                                  cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && dist_cols && win_rows && code_rows, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* dv = V(dist_cols);
    auto const* wv = V(win_rows);
    auto const* cv = V(code_rows);
    check_sssp_block_args(*b, dv, cv, maxpart, grid_cols, grid_c);
    B200_EXPECTS(wv->type == b->wtype, CUGRAPH_INVALID_INPUT, "win_rows dtype must match the block's weights");
    B200_EXPECTS(wv->size >= (size_t)b->n_rows, CUGRAPH_INVALID_INPUT, "win_rows shorter than the block's row slots");
    block_push_t& p = push_copy(h, *b);
    auto* code      = (long long*)cv->data;
    by_float_type(b->wtype, [&](auto z) {
      using T       = decltype(z);
      auto const* d = (T const*)dv->data;
      block_push_min(h, *b, p, code, d,
                     block_pred_op<T>{p.csx->row_vertex.as<int32_t>(), p.csx->weights.as<T>(), d, (T const*)wv->data,
                                      (long long)maxpart, grid_cols, grid_c, code});
    });
    check_last("block_sssp_pred");
  });
}

// cand_rows[row slot] = smallest label_cols[col] over the row's sources, INT64_MAX when none is active
cugraph_error_code_t cugraph_b200_block_wcc_min(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                const cugraph_type_erased_device_array_view_t* label_cols,
                                                cugraph_type_erased_device_array_view_t* cand_rows, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && label_cols && cand_rows, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* lv = V(label_cols);
    auto const* cv = V(cand_rows);
    B200_EXPECTS(lv->type == INT64 && cv->type == INT64, CUGRAPH_INVALID_INPUT, "label_cols / cand_rows must be INT64");
    B200_EXPECTS(lv->size >= (size_t)b->n_cols && cv->size >= (size_t)b->n_rows, CUGRAPH_INVALID_INPUT,
                 "label / candidate arrays shorter than the block's slots");
    block_push_t& p   = push_copy(h, *b);
    auto const* label = (long long const*)lv->data;
    auto* cand        = (long long*)cv->data;
    block_push_min(h, *b, p, cand, label, block_wcc_op{p.csx->row_vertex.as<int32_t>(), label, cand});
    check_last("block_wcc_min");
  });
}

// out_dst[dst slot] = max of val_src (mode 0, from INT64_MIN) or the count (mode 1, from 0) over the dst slot's live edges from
// active sources with an equal key; forward (transposed = FALSE) from column to row slots, backward from row to column slots
cugraph_error_code_t cugraph_b200_block_scc_push(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                 bool_t transposed, int mode,
                                                 const cugraph_type_erased_device_array_view_t* key_src,
                                                 const cugraph_type_erased_device_array_view_t* val_src,
                                                 const cugraph_type_erased_device_array_view_t* key_dst, size_t maxpart,
                                                 int grid_rows, int grid_cols, int grid_r, int grid_c,
                                                 cugraph_type_erased_device_array_view_t* out_dst, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && key_src && val_src && key_dst && out_dst, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* ks = V(key_src);
    auto const* vs = V(val_src);
    auto const* kd = V(key_dst);
    auto const* ov = V(out_dst);
    const bool tr  = transposed == TRUE;
    B200_EXPECTS(ks->type == INT64 && vs->type == INT64 && kd->type == INT64 && ov->type == INT64, CUGRAPH_INVALID_INPUT,
                 "key_src / val_src / key_dst / out_dst must be INT64");
    const size_t n_src = (size_t)(tr ? b->n_rows : b->n_cols), n_dst = (size_t)(tr ? b->n_cols : b->n_rows);
    B200_EXPECTS(ks->size >= n_src && vs->size >= n_src && kd->size >= n_dst && ov->size >= n_dst, CUGRAPH_INVALID_INPUT,
                 "key / value / output arrays shorter than the block's source / destination slots");
    B200_EXPECTS(maxpart > 0 && maxpart < (1u << 31) && grid_rows > 0 && grid_cols > 0 && grid_r >= 0 && grid_r < grid_rows &&
                   grid_c >= 0 &&
                   grid_c < grid_cols,
                 CUGRAPH_INVALID_INPUT, "bad grid position");
    B200_EXPECTS(mode == kSccPushMax || mode == kSccPushCount, CUGRAPH_INVALID_INPUT, "mode must be 0 (max) or 1 (count)");
    auto* out = (long long*)ov->data;
    B200_LAUNCH(h, k_fill<long long>, grid_for((int64_t)n_dst, 1, h.sm_count * 8), kBlock, 0, out, (int64_t)n_dst,
                mode == kSccPushMax ? LLONG_MIN : 0ll);
    auto const* vals = (scc_value_t const*)vs->data;
    if (tr) {
      block_rows_queue_t& q = rows_queue(h, *b);
      csx_t const& c        = *b->csx;
      const block_scc_op op{c.row_vertex.as<int32_t>(), (long long const*)ks->data, (long long const*)vs->data,
                            (long long const*)kd->data, (int)maxpart, grid_cols, grid_r, grid_c, true, mode, out};
      if (c.offs64) block_rows_round<int64_t>(h, c, q, vals, op);
      else block_rows_round<int32_t>(h, c, q, vals, op);
    } else {
      block_push_t& p = push_copy(h, *b);
      const block_scc_op op{p.csx->row_vertex.as<int32_t>(), (long long const*)ks->data, (long long const*)vs->data,
                            (long long const*)kd->data, (int)maxpart, grid_cols, grid_r, grid_c, false, mode, out};
      if (p.csx->offs64) block_push_round<int64_t>(h, p, vals, op);
      else block_push_round<int32_t>(h, p, vals, op);
    }
    check_last("block_scc_push");
  });
}

// the edge rules of the BFS / SSSP certificate over the block (see block_check_op): flag_rows (zeroed first) and
// violations[0] (zeroed first); *edges_from_reached = the edges of the reached columns
cugraph_error_code_t cugraph_b200_block_check_paths(const cugraph_resource_handle_t* handle, cugraph_b200_block_t* block,
                                                    const cugraph_type_erased_device_array_view_t* dist_cols,
                                                    const cugraph_type_erased_device_array_view_t* dist_rows,
                                                    const cugraph_type_erased_device_array_view_t* pred_rows, double cutoff,
                                                    size_t maxpart, int grid_cols, int grid_c,
                                                    cugraph_type_erased_device_array_view_t* flag_rows,
                                                    cugraph_type_erased_device_array_view_t* violations,
                                                    uint64_t* edges_from_reached, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(block && dist_cols && dist_rows && pred_rows && flag_rows && violations && edges_from_reached,
                 CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* b        = reinterpret_cast<block_impl*>(block);
    auto const* dc = V(dist_cols);
    auto const* dr = V(dist_rows);
    auto const* pr = V(pred_rows);
    auto const* fv = V(flag_rows);
    auto const* vv = V(violations);
    const bool unit = dc->type == INT32;
    B200_EXPECTS(dr->type == dc->type, CUGRAPH_INVALID_INPUT, "dist_cols / dist_rows dtypes differ");
    B200_EXPECTS(unit || (b->weighted && dc->type == b->wtype), CUGRAPH_INVALID_INPUT,
                 "distances must be INT32 (unit steps) or the weight type of a weighted block");
    B200_EXPECTS(pr->type == INT64 && dtype_size(fv->type) == 1 && vv->type == INT64 && vv->size >= 1, CUGRAPH_INVALID_INPUT,
                 "pred_rows must be INT64, flag_rows byte flags, violations INT64");
    B200_EXPECTS(dc->size >= (size_t)b->n_cols && dr->size >= (size_t)b->n_rows && pr->size >= (size_t)b->n_rows &&
                   fv->size >= (size_t)b->n_rows,
                 CUGRAPH_INVALID_INPUT, "distance / predecessor / flag arrays shorter than the block's slots");
    B200_EXPECTS(maxpart > 0 && grid_cols > 0 && grid_c >= 0 && grid_c < grid_cols, CUGRAPH_INVALID_INPUT, "bad grid position");
    CUDA_TRY(cudaMemsetAsync(fv->data, 0, (size_t)b->n_rows, h.stream));
    CUDA_TRY(cudaMemsetAsync(vv->data, 0, sizeof(long long), h.stream));
    block_push_t& p = push_copy(h, *b);
    auto* flags     = (uint8_t*)fv->data;
    auto* viol      = (unsigned long long*)vv->data;
    auto run        = [&](auto op, auto const* cols) {
      const block_queue_counts_t hc =
        p.csx->offs64 ? block_push_round<int64_t>(h, p, cols, op) : block_push_round<int32_t>(h, p, cols, op);
      *edges_from_reached = (uint64_t)hc.edges;
    };
    if (unit) {
      auto const* d = (int32_t const*)dc->data;
      const long long lim = cutoff >= 9.2e18 ? LLONG_MAX : (long long)cutoff;
      run(block_check_op<int32_t>{p.csx->row_vertex.as<int32_t>(), nullptr, d, (int32_t const*)dr->data,
                                  (long long const*)pr->data, lim, (long long)maxpart, grid_cols, grid_c, flags, viol},
          d);
    } else {
      by_float_type(b->wtype, [&](auto z) {
        using T       = decltype(z);
        auto const* d = (T const*)dc->data;
        run(block_check_op<T>{p.csx->row_vertex.as<int32_t>(), p.csx->weights.as<T>(), d, (T const*)dr->data,
                              (long long const*)pr->data, rounded_cutoff<T>(cutoff), (long long)maxpart, grid_cols, grid_c,
                              flags, viol},
            d);
      });
    }
    check_last("block_check_paths");
  });
}

// answers[2i], answers[2i + 1] = external id and predecessor code of local id lids[i].  Asynchronous.
cugraph_error_code_t cugraph_b200_paths_answer(const cugraph_resource_handle_t* handle,
                                               const cugraph_type_erased_device_array_view_t* lids,
                                               const cugraph_type_erased_device_array_view_t* vertices,
                                               const cugraph_type_erased_device_array_view_t* pred_codes, size_t n_local,
                                               cugraph_type_erased_device_array_view_t* answers, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(lids && vertices && pred_codes && answers, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* lv = V(lids);
    auto const* vv = V(vertices);
    auto const* cv = V(pred_codes);
    auto const* av = V(answers);
    B200_EXPECTS(lv->type == INT32, CUGRAPH_INVALID_INPUT, "lids must be INT32");
    B200_EXPECTS(vv->type == INT32 || vv->type == INT64, CUGRAPH_INVALID_INPUT, "vertices must be INT32 / INT64");
    B200_EXPECTS(cv->type == INT64 && av->type == INT64, CUGRAPH_INVALID_INPUT, "pred_codes / answers must be INT64");
    B200_EXPECTS(n_local < (1u << 31) && vv->size >= n_local && cv->size >= n_local, CUGRAPH_INVALID_INPUT,
                 "vertices / pred_codes shorter than n_local");
    B200_EXPECTS(av->size >= 2 * lv->size, CUGRAPH_INVALID_INPUT, "answers must hold two entries per local id");
    const long long n = (long long)lv->size;
    if (n == 0) return;
    const int grid = grid_for(n, 1, h.sm_count * 8);
    if (vv->type == INT32)
      B200_LAUNCH(h, k_paths_answer<int32_t>, grid, kBlock, 0, (int32_t const*)lv->data, n, (int32_t const*)vv->data,
                  (long long const*)cv->data, (int32_t)n_local, (long long*)av->data);
    else
      B200_LAUNCH(h, k_paths_answer<int64_t>, grid, kBlock, 0, (int32_t const*)lv->data, n, (int64_t const*)vv->data,
                  (long long const*)cv->data, (int32_t)n_local, (long long*)av->data);
    check_last("paths_answer");
  });
}

// paths[row][pos] = the answered ids; the entries that go on, grouped by owner rank, into next_*, and counts[rank].
// Asynchronous.
cugraph_error_code_t cugraph_b200_paths_advance(const cugraph_resource_handle_t* handle,
                                                const cugraph_type_erased_device_array_view_t* answers,
                                                const cugraph_type_erased_device_array_view_t* rows,
                                                const cugraph_type_erased_device_array_view_t* positions,
                                                cugraph_type_erased_device_array_view_t* paths, size_t max_path_length,
                                                size_t maxpart, int world, cugraph_type_erased_device_array_view_t* next_lids,
                                                cugraph_type_erased_device_array_view_t* next_rows,
                                                cugraph_type_erased_device_array_view_t* next_positions,
                                                cugraph_type_erased_device_array_view_t* counts, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(answers && rows && positions && paths && next_lids && next_rows && next_positions && counts,
                 CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* av = V(answers);
    auto const* rv = V(rows);
    auto const* pv = V(positions);
    auto const* xv = V(paths);
    auto const* nl = V(next_lids);
    auto const* nr = V(next_rows);
    auto const* np = V(next_positions);
    auto const* cv = V(counts);
    const size_t n = rv->size;
    B200_EXPECTS(rv->type == INT32 && pv->type == INT32 && pv->size == n, CUGRAPH_INVALID_INPUT,
                 "rows / positions must be INT32 arrays of equal size");
    B200_EXPECTS(av->type == INT64 && av->size >= 2 * n, CUGRAPH_INVALID_INPUT, "answers must hold two INT64 entries per row");
    B200_EXPECTS(xv->type == INT32 || xv->type == INT64, CUGRAPH_INVALID_INPUT, "paths must be INT32 / INT64");
    B200_EXPECTS(max_path_length > 0 && xv->size % max_path_length == 0, CUGRAPH_INVALID_INPUT,
                 "paths must hold whole rows of max_path_length entries");
    B200_EXPECTS(nl->type == INT32 && nr->type == INT32 && np->type == INT32 && nl->size >= n && nr->size >= n && np->size >= n,
                 CUGRAPH_INVALID_INPUT, "next_lids / next_rows / next_positions must be INT32 arrays of at least n entries");
    B200_EXPECTS(world > 0 && cv->type == INT64 && cv->size >= (size_t)world, CUGRAPH_INVALID_INPUT,
                 "counts must be INT64 with one entry per rank");
    B200_EXPECTS(maxpart > 0 && maxpart < (1u << 31), CUGRAPH_INVALID_INPUT, "bad maxpart");
    auto* cnt   = (long long*)cv->data;
    dbuf cursor = make_dbuf<int>((size_t)world, h.stream);
    CUDA_TRY(cudaMemsetAsync(cnt, 0, sizeof(long long) * (size_t)world, h.stream));
    CUDA_TRY(cudaMemsetAsync(cursor.data(), 0, sizeof(int) * (size_t)world, h.stream));
    if (n == 0) return;
    const long long len = (long long)max_path_length, n_paths_rows = (long long)(xv->size / max_path_length);
    const int grid      = grid_for((int64_t)n, 1, h.sm_count * 8);
    auto const* ans     = (long long const*)av->data;
    auto const* r       = (int32_t const*)rv->data;
    auto const* p       = (int32_t const*)pv->data;
    B200_LAUNCH(h, k_paths_count, grid, kBlock, 0, ans, r, p, (long long)n, n_paths_rows, len, (long long)maxpart, world, cnt);
    if (xv->type == INT32)
      B200_LAUNCH(h, k_paths_advance<int32_t>, grid, kBlock, 0, ans, r, p, (long long)n, (int32_t*)xv->data, n_paths_rows, len,
                  (long long)maxpart, world, (long long const*)cnt, cursor.as<int>(), (int32_t*)nl->data, (int32_t*)nr->data,
                  (int32_t*)np->data);
    else
      B200_LAUNCH(h, k_paths_advance<int64_t>, grid, kBlock, 0, ans, r, p, (long long)n, (int64_t*)xv->data, n_paths_rows, len,
                  (long long)maxpart, world, (long long const*)cnt, cursor.as<int>(), (int32_t*)nl->data, (int32_t*)nr->data,
                  (int32_t*)np->data);
    check_last("paths_advance");
  });
}

// the reference's MG constructors take raft comms (not part of this build): see cugraph_b200/mg.py for the torch.distributed path
cugraph_error_code_t cugraph_graph_create_mg(cugraph_resource_handle_t const*, cugraph_graph_properties_t const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  bool_t, size_t, bool_t, bool_t, bool_t, bool_t, cugraph_graph_t**, cugraph_error_t** error)
{
  return guarded(error, [&] {
    throw capi_exception(CUGRAPH_NOT_IMPLEMENTED,
                         "cugraph_graph_create_mg needs raft comms; use cugraph_b200.mg.MGGraph (torch.distributed)");
  });
}
cugraph_error_code_t cugraph_graph_create_with_times_mg(cugraph_resource_handle_t const*, cugraph_graph_properties_t const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  cugraph_type_erased_device_array_view_t const* const*, cugraph_type_erased_device_array_view_t const* const*,
  bool_t, size_t, bool_t, bool_t, bool_t, bool_t, cugraph_graph_t**, cugraph_error_t** error)
{
  return guarded(error, [&] {
    throw capi_exception(CUGRAPH_NOT_IMPLEMENTED,
                         "cugraph_graph_create_with_times_mg needs raft comms; use cugraph_b200.mg.MGGraph (torch.distributed)");
  });
}

}  // extern "C"
