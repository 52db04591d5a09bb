// Strongly connected components (C API reference cpp/src/c_api/strongly_connected_components.cpp,
// cpp/include/cugraph_c/labeling_algorithms.h:76-95).  The reference runs a recursive forward-backward search over pivots
// (strongly_connected_components_impl.cuh:1989-2386); here: Multistep (Slota, Rajamanickam, Madduri, IPDPS 2014), every
// phase a frontier loop on the load-balanced advance (advance.cuh) over the out-edges (push_view) or the in-edges (in_view):
//  1. trim: a live vertex without a live in-edge or without a live out-edge is an SCC of its own.  Live in- and
//     out-degree counters (self-loops not counted, multi-edges counted per edge); the peeled vertices' out-edges lower their
//     targets' in-degrees, their in-edges their sources' out-degrees, and a counter that reaches 0 queues its vertex for the
//     next round (once: a compare-and-swap on its subproblem word).  Rounds = the longest peel chain.
//  2. forward-backward from one pivot (the live vertex with the largest live in-degree x out-degree, ties to the smallest
//     id): FW ∩ BW is one SCC (the giant one of a power-law graph); FW\BW, BW\FW and the rest become three subproblems.
//     Rounds = the forward plus the backward reach depth.
//  3. colouring until no live vertex is left: the largest id is propagated forward along edges inside a subproblem until
//     nothing changes; every vertex r whose colour is r is a root, and the backward reach from all roots at once, among
//     vertices of the root's colour, is exactly SCC(r).  Those SCCs are removed, every other vertex's colour becomes its
//     subproblem, and the round repeats; each round resolves at least one SCC.  Rounds per outer round = colour
//     propagation depth + backward reach depth.
// Every round of every phase costs one read-back of the queue counters (as BFS levels do).
// The label of a vertex is the external id of the member of its SCC with the smallest internal id (an atomicMin per SCC,
// then a gather: WCC's rule, components.cu), so labels depend neither on the schedule nor on the phase that found the SCC.
#include "advance.cuh"

#include <chrono>
#include <climits>

namespace b200 {
namespace {

// what a frontier round leaves for the host
struct scc_counters_t {
  int n;                      // entries appended to the next queue
  int pad;
  unsigned long long m_out;   // out-degree sum of the appended entries (their advance over push_view)
  unsigned long long m_in;    // in-degree sum of the appended entries (their advance over in_view)
  unsigned long long resolved;  // vertices resolved by a vertex pass
};

// per-vertex state shared by the phases
struct scc_state_t {
  int32_t* sub;          // subproblem of a live vertex (>= 0); -1 once its SCC is known
  int32_t* comp;         // a member of the vertex's SCC, set when it is resolved
  int32_t const* dout;   // row lengths of push_view (out-edges stored, self-loops included)
  int32_t const* din;    // row lengths of in_view
  int32_t* q_next;       // the queue being filled
  scc_counters_t* cnt;
  __device__ __forceinline__ void push(int v) const
  {
    const int pos = warp_append(&cnt->n);
    q_next[pos]   = v;
    warp_add_u64(&cnt->m_out, (unsigned)dout[v]);
    warp_add_u64(&cnt->m_in, (unsigned)din[v]);
  }
  __device__ __forceinline__ void resolve(int v, int member) const
  {
    sub[v]  = -1;
    comp[v] = member;
    warp_add_u64(&cnt->resolved, 1u);
  }
};

// row length and the number of entries that are not self-loops, a warp per row
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_row_degrees(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t nv, int32_t* __restrict__ full,
              int32_t* __restrict__ live)
{
  const int lane = threadIdx.x & 31;
  for (long long v = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; v < nv; v += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long b = (long long)off[v], e = (long long)off[v + 1];
    unsigned c        = 0;
    for (long long k = b + lane; k < e; k += 32) c += idx[k] != (int32_t)v;
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) {
      full[v] = (int32_t)(e - b);
      live[v] = (int32_t)c;
    }
  }
}

// ---- 1. trim
__global__ void k_trim_seed(int32_t nv, int32_t const* __restrict__ in_live, int32_t const* __restrict__ out_live, scc_state_t s)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    if (in_live[v] == 0 || out_live[v] == 0) {
      s.resolve(v, v);
      s.push(v);
    } else {
      s.sub[v] = 0;
    }
  }
}

// an edge of a peeled vertex v: over push_view nbr loses an in-edge, over in_view an out-edge
struct peel_op {
  int32_t* live_deg;  // the counter of nbr that loses the edge
  scc_state_t s;
  __device__ __forceinline__ void edge(int v, long long, int nbr) const
  {
    if (nbr == v || s.sub[nbr] < 0) return;
    if (atomicAdd(live_deg + nbr, -1) != 1) return;
    if (atomicCAS(s.sub + nbr, 0, -1) != 0) return;  // both counters may reach 0: the first one queues the vertex
    s.comp[nbr] = nbr;
    warp_add_u64(&s.cnt->resolved, 1u);
    s.push(nbr);
  }
};

// ---- 2. forward-backward from one pivot
__global__ void k_pivot_score(int32_t nv, int32_t const* __restrict__ sub, int32_t const* __restrict__ in_live,
                              int32_t const* __restrict__ out_live, unsigned long long* best)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x)
    if (sub[v] >= 0) atomicMax(best, (unsigned long long)in_live[v] * (unsigned long long)out_live[v]);
}
__global__ void k_pivot_pick(int32_t nv, int32_t const* __restrict__ sub, int32_t const* __restrict__ in_live,
                             int32_t const* __restrict__ out_live, unsigned long long const* __restrict__ best, int* pivot)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x)
    if (sub[v] >= 0 && (unsigned long long)in_live[v] * (unsigned long long)out_live[v] == *best) atomicMin(pivot, v);
}

// queue one vertex and stamp it
__global__ void k_seed_one(int v, int32_t* mark, int epoch, scc_state_t s)
{
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    mark[v] = epoch;
    s.push(v);
  }
}

// reach among live vertices of v's subproblem (and, with `key`, of v's key); a vertex joins once per epoch
struct reach_op {
  int32_t const* key;
  int32_t* mark;
  int epoch;
  scc_state_t s;
  __device__ __forceinline__ void edge(int v, long long, int nbr) const
  {
    if (nbr == v) return;
    const int sn = s.sub[nbr];
    if (sn < 0 || sn != s.sub[v]) return;
    if (key && key[nbr] != key[v]) return;
    if (mark[nbr] == epoch || atomicExch(mark + nbr, epoch) == epoch) return;
    s.push(nbr);
  }
  void next_round(int&) {}
};

// FW ∩ BW is the pivot's SCC; FW only, BW only and the rest become subproblems 1, 2 and 3
__global__ void k_fwbw_split(int32_t nv, int32_t const* __restrict__ fw, int fw_epoch, int32_t const* __restrict__ bw, int bw_epoch,
                             int pivot, scc_state_t s)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    if (s.sub[v] < 0) continue;
    const bool f = fw[v] == fw_epoch, b = bw[v] == bw_epoch;
    if (f && b) s.resolve(v, pivot);
    else s.sub[v] = f ? 1 : (b ? 2 : 3);
  }
}

// ---- 3. colouring
__global__ void k_colour_seed(int32_t nv, int32_t* __restrict__ colour, int32_t* __restrict__ stamp, int epoch, scc_state_t s)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    if (s.sub[v] < 0) continue;
    colour[v] = v;
    stamp[v]  = epoch;
    s.push(v);
  }
}

// the largest colour flows forward inside a subproblem; a vertex whose colour rose is queued once per round.  A stale
// (smaller) colour read for v only delays the flow: v's rise queued v again.
struct colour_op {
  int32_t* colour;
  int32_t* stamp;
  int epoch;  // the round being filled
  scc_state_t s;
  __device__ __forceinline__ void edge(int v, long long, int nbr) const
  {
    if (nbr == v) return;
    const int sn = s.sub[nbr];
    if (sn < 0 || sn != s.sub[v]) return;
    const int c = ((volatile int32_t const*)colour)[v];
    if (((volatile int32_t const*)colour)[nbr] >= c || atomicMax(colour + nbr, c) >= c) return;
    if (atomicExch(stamp + nbr, epoch) != epoch) s.push(nbr);
  }
  void next_round(int& e) { epoch = ++e; }
};

__global__ void k_colour_roots(int32_t nv, int32_t const* __restrict__ colour, int32_t* __restrict__ mark, int epoch, scc_state_t s)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    if (s.sub[v] < 0 || colour[v] != v) continue;
    mark[v] = epoch;
    s.push(v);
  }
}

// the roots' backward reach is resolved; every other live vertex keeps its colour as its subproblem
__global__ void k_colour_split(int32_t nv, int32_t const* __restrict__ colour, int32_t const* __restrict__ mark, int epoch, scc_state_t s)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
    if (s.sub[v] < 0) continue;
    if (mark[v] == epoch) s.resolve(v, colour[v]);
    else s.sub[v] = colour[v];
  }
}

// ---- labels: the smallest internal id of every SCC, gathered to its members
__global__ void k_scc_min(int32_t nv, int32_t const* __restrict__ comp, int32_t* __restrict__ min_member)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) atomicMin(min_member + comp[v], v);
}
__global__ void k_scc_gather(int32_t nv, int32_t const* __restrict__ comp, int32_t const* __restrict__ min_member, int32_t* __restrict__ label)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) label[v] = min_member[comp[v]];
}

class scc_run {
 public:
  scc_run(handle_impl const& h, csx_t const& out, csx_t const& in, int32_t nv)
    : h_(h), out_(out), in_(in), nv_(nv), vgrid_(grid_for(nv, 1, h.sm_count * 8))
  {
    for (dbuf* b : {&dout_, &din_, &out_live_, &in_live_, &sub_, &comp_, &colour_, &mark_a_, &mark_b_, &qa_, &qb_})
      *b = make_dbuf<int32_t>(nv, h.stream);
    cnt_ = make_dbuf<scc_counters_t>(1, h.stream);
    CUDA_TRY(cudaMemsetAsync(mark_a_.data(), 0, sizeof(int32_t) * nv, h.stream));
    CUDA_TRY(cudaMemsetAsync(mark_b_.data(), 0, sizeof(int32_t) * nv, h.stream));
    adv_.init(h, nv, std::max(out.nnz, in.nnz));
  }

  // labels[v] = the smallest internal id of v's SCC
  void run(int32_t* labels)
  {
    trim();
    if (resolved_ < nv_) forward_backward();
    colouring();
    B200_LAUNCH(h_, (k_fill<int32_t>), vgrid_, kBlock, 0, mark_a_.as<int32_t>(), (int64_t)nv_, INT_MAX);
    B200_LAUNCH(h_, k_scc_min, vgrid_, kBlock, 0, nv_, comp_.as<int32_t>(), mark_a_.as<int32_t>());
    B200_LAUNCH(h_, k_scc_gather, vgrid_, kBlock, 0, nv_, comp_.as<int32_t>(), mark_a_.as<int32_t>(), labels);
  }

 private:
  handle_impl const& h_;
  csx_t const &out_, &in_;
  int32_t nv_;
  int vgrid_;
  dbuf dout_, din_, out_live_, in_live_, sub_, comp_, colour_, mark_a_, mark_b_, qa_, qb_, cnt_;
  advance_scratch_t adv_;
  int32_t *cur_{nullptr}, *nxt_{nullptr};
  int epoch_{0};             // stamps of marks: every reach and colour round takes a new one, so marks are never reset
  long long resolved_{0};    // vertices whose SCC is known
  std::chrono::steady_clock::time_point t0_{std::chrono::steady_clock::now()};

  scc_state_t state(int32_t* q_next) const
  {
    return scc_state_t{sub_.as<int32_t>(), comp_.as<int32_t>(), dout_.as<int32_t>(), din_.as<int32_t>(), q_next,
                       cnt_.as<scc_counters_t>()};
  }
  void reset_counters() { CUDA_TRY(cudaMemsetAsync(cnt_.data(), 0, sizeof(scc_counters_t), h_.stream)); }
  scc_counters_t counters() const
  {
    auto* hc = reinterpret_cast<scc_counters_t*>(h_.pinned);
    CUDA_TRY(cudaMemcpyAsync(hc, cnt_.data(), sizeof(scc_counters_t), cudaMemcpyDeviceToHost, h_.stream));
    sync(h_);
    return *hc;
  }
  template <typename Op>
  void advance_over(csx_t const& c, int32_t const* q, int n, unsigned long long m, Op const& op)
  {
    if (c.offs64) advance<int64_t>(h_, adv_, c.offsets.as<int64_t>(), c.indices.as<int32_t>(), q, n, m, op);
    else advance<int32_t>(h_, adv_, c.offsets.as<int32_t>(), c.indices.as<int32_t>(), q, n, m, op);
  }
  // CUGRAPH_B200_SCC_TRACE: rounds, resolved vertices and time (since the previous line, device work included) of a phase
  void trace(const char* phase, const char* detail, long long resolved)
  {
    if (!h_.tune.scc_trace) return;
    sync(h_);
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "scc %-10s %s resolved=%lld time_ms=%.3f\n", phase, detail, resolved,
                 std::chrono::duration<double, std::milli>(t1 - t0_).count());
    t0_ = t1;
  }

  // advance the queue in cur_ (n entries, m edges in c) with op round after round until it is empty; returns the rounds
  template <typename Op>
  int frontier(csx_t const& c, bool in_edges, scc_counters_t k, Op op)
  {
    int rounds = 0;
    while (k.n > 0) {
      reset_counters();
      op.next_round(epoch_);
      op.s = state(nxt_);
      advance_over(c, cur_, k.n, in_edges ? k.m_in : k.m_out, op);
      k = counters();
      std::swap(cur_, nxt_);
      ++rounds;
    }
    return rounds;
  }

  void trim()
  {
    if (out_.offs64) B200_LAUNCH(h_, (k_row_degrees<int64_t>), grid_for((int64_t)nv_ * 32, 1, h_.sm_count * 16), kBlock, 0,
                                 out_.offsets.as<int64_t>(), out_.indices.as<int32_t>(), nv_, dout_.as<int32_t>(), out_live_.as<int32_t>());
    else B200_LAUNCH(h_, (k_row_degrees<int32_t>), grid_for((int64_t)nv_ * 32, 1, h_.sm_count * 16), kBlock, 0,
                     out_.offsets.as<int32_t>(), out_.indices.as<int32_t>(), nv_, dout_.as<int32_t>(), out_live_.as<int32_t>());
    if (in_.offs64) B200_LAUNCH(h_, (k_row_degrees<int64_t>), grid_for((int64_t)nv_ * 32, 1, h_.sm_count * 16), kBlock, 0,
                                in_.offsets.as<int64_t>(), in_.indices.as<int32_t>(), nv_, din_.as<int32_t>(), in_live_.as<int32_t>());
    else B200_LAUNCH(h_, (k_row_degrees<int32_t>), grid_for((int64_t)nv_ * 32, 1, h_.sm_count * 16), kBlock, 0,
                     in_.offsets.as<int32_t>(), in_.indices.as<int32_t>(), nv_, din_.as<int32_t>(), in_live_.as<int32_t>());
    cur_ = qa_.as<int32_t>();
    nxt_ = qb_.as<int32_t>();
    reset_counters();
    B200_LAUNCH(h_, k_trim_seed, vgrid_, kBlock, 0, nv_, in_live_.as<int32_t>(), out_live_.as<int32_t>(), state(cur_));
    scc_counters_t k = counters();
    long long resolved = (long long)k.resolved;
    int rounds         = 0;
    while (k.n > 0) {  // the peeled vertices of a round are advanced over both orientations into one next queue
      reset_counters();
      advance_over(out_, cur_, k.n, k.m_out, peel_op{in_live_.as<int32_t>(), state(nxt_)});
      advance_over(in_, cur_, k.n, k.m_in, peel_op{out_live_.as<int32_t>(), state(nxt_)});
      k = counters();
      resolved += (long long)k.resolved;
      std::swap(cur_, nxt_);
      ++rounds;
    }
    resolved_ += resolved;
    char d[64];
    std::snprintf(d, sizeof d, "rounds=%d", rounds);
    trace("trim", d, resolved);
  }

  void forward_backward()
  {
    dbuf best = make_dbuf<unsigned long long>(1, h_.stream), piv = make_dbuf<int>(1, h_.stream);
    CUDA_TRY(cudaMemsetAsync(best.data(), 0, sizeof(unsigned long long), h_.stream));
    B200_LAUNCH(h_, (k_fill<int>), 1, kBlock, 0, piv.as<int>(), (int64_t)1, INT_MAX);
    B200_LAUNCH(h_, k_pivot_score, vgrid_, kBlock, 0, nv_, sub_.as<int32_t>(), in_live_.as<int32_t>(), out_live_.as<int32_t>(),
                best.as<unsigned long long>());
    B200_LAUNCH(h_, k_pivot_pick, vgrid_, kBlock, 0, nv_, sub_.as<int32_t>(), in_live_.as<int32_t>(), out_live_.as<int32_t>(),
                best.as<unsigned long long>(), piv.as<int>());
    const int pivot = read_back(h_, piv.as<int>());
    int rounds[2];
    int epochs[2];
    for (int dir = 0; dir < 2; ++dir) {  // 0: forward over the out-edges (marks in mark_a), 1: backward over the in-edges (mark_b)
      int32_t* mark = (dir == 0 ? mark_a_ : mark_b_).as<int32_t>();
      epochs[dir]   = ++epoch_;
      reset_counters();
      B200_LAUNCH(h_, k_seed_one, 1, 32, 0, pivot, mark, epochs[dir], state(cur_));
      rounds[dir] = frontier(dir == 0 ? out_ : in_, dir == 1, counters(), reach_op{nullptr, mark, epochs[dir], state(nxt_)});
    }
    reset_counters();
    B200_LAUNCH(h_, k_fwbw_split, vgrid_, kBlock, 0, nv_, mark_a_.as<int32_t>(), epochs[0], mark_b_.as<int32_t>(), epochs[1], pivot,
                state(cur_));
    const long long resolved = (long long)counters().resolved;
    resolved_ += resolved;
    char d[96];
    std::snprintf(d, sizeof d, "pivot=%d fw_rounds=%d bw_rounds=%d", pivot, rounds[0], rounds[1]);
    trace("fw-bw", d, resolved);
  }

  void colouring()
  {
    int outer = 0;
    long long colour_rounds = 0, reach_rounds = 0, resolved = 0;
    int32_t* colour = colour_.as<int32_t>();
    while (resolved_ < nv_) {
      reset_counters();
      int e = ++epoch_;
      B200_LAUNCH(h_, k_colour_seed, vgrid_, kBlock, 0, nv_, colour, mark_a_.as<int32_t>(), e, state(cur_));
      colour_rounds += frontier(out_, false, counters(), colour_op{colour, mark_a_.as<int32_t>(), e, state(nxt_)});
      reset_counters();
      e = ++epoch_;
      B200_LAUNCH(h_, k_colour_roots, vgrid_, kBlock, 0, nv_, colour, mark_b_.as<int32_t>(), e, state(cur_));
      reach_rounds += frontier(in_, true, counters(), reach_op{colour, mark_b_.as<int32_t>(), e, state(nxt_)});
      reset_counters();
      B200_LAUNCH(h_, k_colour_split, vgrid_, kBlock, 0, nv_, colour, mark_b_.as<int32_t>(), e, state(cur_));
      const long long r = (long long)counters().resolved;
      B200_EXPECTS(r > 0, CUGRAPH_UNKNOWN_ERROR, "strongly_connected_components: a colouring round resolved no vertex");
      resolved += r;
      resolved_ += r;
      ++outer;
    }
    char d[96];
    std::snprintf(d, sizeof d, "outer_rounds=%d colour_rounds=%lld reach_rounds=%lld", outer, colour_rounds, reach_rounds);
    trace("colouring", d, resolved);
  }
};

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_strongly_connected_components(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                           bool_t do_expensive_check, cugraph_labeling_result_t** result,
                                                           cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    // strongly_connected_components_impl.cuh:2013-2015
    B200_EXPECTS(!g->is_symmetric, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: call weakly_connected_components instead for symmetric graphs.");
    const int32_t nv = g->n_vertices;
    dbuf label       = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    if (nv > 0) {
      csx_t const& out = push_view(h, *g);
      csx_t const& in  = in_view(h, *g);
      scc_run(h, out, in, nv).run(label.as<int32_t>());
    }
    // labels: external ids, reported in the result's vertex order (as WCC)
    dbuf label_ext(std::max<size_t>(nv, 1) * dtype_size(g->vertex_type), h.stream);
    int_to_ext(h, *g, label.as<int32_t>(), (size_t)nv, label_ext.data());
    auto res      = std::make_unique<labeling_result_impl>();
    res->vertices = new device_array_impl{reported_vertices(h, *g), (size_t)nv, g->vertex_type};
    res->labels   = new device_array_impl{to_reported_order(h, *g, label_ext.data(), dtype_size(g->vertex_type)), (size_t)nv, g->vertex_type};
    check_last("strongly_connected_components");
    sync(h);
    *result = reinterpret_cast<cugraph_labeling_result_t*>(res.release());
  });
}

}  // extern "C"
