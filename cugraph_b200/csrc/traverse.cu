// Frontier engine + BFS + SSSP on one GPU, and their C-ABI entry points.
// Replaces: transform_reduce_if_v_frontier_outgoing_e_by_dst / extract_transform_if_v_frontier_e
// (cpp/include/cugraph/prims/transform_reduce_if_v_frontier_outgoing_e_by_dst.cuh:604-1128,
//  detail/extract_transform_if_v_frontier_e.cuh:127-518), the BFS driver
// (cpp/src/traversal/bfs_impl.cuh:133-869), the SSSP driver (sssp_impl.cuh:169-566) and
// cpp/src/c_api/{bfs,sssp}.cpp.
//
// Design differences from the reference (same results, see traversal_algorithms.h):
//  * the advance writes straight into per-vertex slots guarded by a visited bitmap (BFS) or an
//    atomicMin on the distance word (SSSP); there is no emit-buffer + per-level radix sort/unique
//    (transform_reduce_if_v_frontier_outgoing_e_by_dst.cuh:225-600).
//  * load balance: the merge-path advance (advance.cuh, DESIGN §3.4) cuts the summed edge range of a queue into tiles of
//    equal size, whatever the mix of degrees; a CTA finds the queue entries of its tile and strides over its edges.
//  * bottom-up BFS steps process 32 consecutive vertices per warp: one visited-word load, early
//    exit on the first parent in the frontier bitmap (neighbours are sorted by internal id, i.e.
//    hubs first), the next-frontier word is assembled with a ballot — no atomics.
#include "advance.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <cfloat>
#include <chrono>
#include <climits>
#include <cstdlib>
#include <cmath>
#include <limits>
#include <vector>

namespace b200 {
namespace {

struct frontier_counters_t {
  int n_small;              // entries appended to the next queue
  int n_conv;               // bitmap -> queue conversion cursor
  unsigned long long m_f;   // sum of degrees of the vertices appended (direction-optimising heuristic)
  unsigned long long packed;  // SSSP with 32-bit offsets: (sum of degrees << 32) | entries appended — ONE atomic per append
};

// every edge of the graph, edge-balanced (the same k_tile_owners / k_advance as advance(), advance.cuh): the row offsets are the scan of the identity queue
template <typename Op>
void advance_all_edges(handle_impl const& h, int32_t const* off, int32_t const* idx, int32_t n_vertices, long long nnz, Op op)
{
  if (nnz <= 0) return;
  const int n_tiles = (int)((nnz + kTileEdges - 1) / kTileEdges);
  dbuf tile_k       = make_dbuf<int2>((size_t)n_tiles, h.stream);
  B200_LAUNCH(h, k_tile_owners, (n_tiles + kBlock - 1) / kBlock, kBlock, 0, off, n_vertices, n_tiles, tile_k.as<int2>());
  int grid = (int)std::min<long long>((long long)n_tiles, (long long)h.sm_count * 8);
  B200_LAUNCH(h, (k_advance<int32_t, Op, true>), grid, kBlock, 0, off, idx, (int32_t const*)nullptr, n_vertices, off,
              tile_k.as<int2>(), n_tiles, op);
}

// ------------------------------------------------------------------------------------------
// BFS
// ------------------------------------------------------------------------------------------
// append v to the queue and its degree to the parallel degree array (the next advance scans the degrees as they are: no
// degree pass over the queue); returns the degree.  One queue whatever the degree: the merge-path advance balances any mix.
template <typename O>
__device__ __forceinline__ unsigned enqueue_with_degree(O const* off, int v, int32_t* q, int32_t* q_deg,
                                                        frontier_counters_t* cnt)
{
  const unsigned d = (unsigned)((long long)off[v + 1] - (long long)off[v]);
  const int pos    = warp_append(&cnt->n_small);
  q[pos]           = v;
  q_deg[pos]       = (int32_t)d;
  return d;
}

// SSSP flavour: count and degree sum advance with one warp-aggregated 64-bit atomic (every append of a round hits the same
// address; two atomics per append were two serialised streams at the L2).  With 64-bit offsets the degree sum of a round may
// pass 2^32: the two separate counters are kept there.
template <typename O>
__device__ __forceinline__ void enqueue_counted(O const* off, int v, int32_t* q, int32_t* q_deg, frontier_counters_t* cnt)
{
  if (sizeof(O) == 8) {
    const unsigned d = enqueue_with_degree(off, v, q, q_deg, cnt);
    warp_add_u64(&cnt->m_f, d);
    return;
  }
  const unsigned d    = (unsigned)((long long)off[v + 1] - (long long)off[v]);
  const unsigned mask = __activemask();
  const int leader = __ffs(mask) - 1, lane = threadIdx.x & 31;
  const unsigned sum = __reduce_add_sync(mask, d);
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(&cnt->packed, ((unsigned long long)sum << 32) | (unsigned)__popc(mask));
  base          = __shfl_sync(mask, base, leader);
  const int pos = (int)(unsigned)(base & 0xffffffffull) + __popc(mask & ((1u << lane) - 1u));
  q[pos]        = v;
  q_deg[pos]    = (int32_t)d;
}
// what the host reads back after a round (pinned copy of the counters)
template <typename O>
inline void read_counters(frontier_counters_t const* hc, int& n, unsigned long long& edges)
{
  if (sizeof(O) == 8) {
    n     = hc->n_small;
    edges = hc->m_f;
  } else {
    n     = (int)(unsigned)(hc->packed & 0xffffffffull);
    edges = hc->packed >> 32;
  }
}

template <typename O>
struct bfs_topdown_op {
  O const* off;
  uint32_t* visited;
  int32_t* dist;
  int32_t* pred;  // may be null
  int32_t* next_q;
  int32_t* next_q_deg;  // degrees of the entries of next_q
  frontier_counters_t* cnt;
  int level;
  __device__ __forceinline__ void edge(int src, long long, int nbr) const
  {
    const uint32_t bit = 1u << (nbr & 31);
    if (visited[nbr >> 5] & bit) return;
    const uint32_t old = atomicOr(visited + (nbr >> 5), bit);
    if (old & bit) return;
    dist[nbr] = level + 1;
    if (pred) pred[nbr] = src;
    const unsigned d = enqueue_with_degree(off, nbr, next_q, next_q_deg, cnt);
    warp_add_u64(&cnt->m_f, d);
  }
};

// 32 consecutive vertices per warp; parents looked up in the frontier bitmap
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_bfs_bottomup(O const* __restrict__ off, int32_t const* __restrict__ idx, uint32_t* __restrict__ visited,
               uint32_t const* __restrict__ frontier_bm, uint32_t* __restrict__ next_bm, int32_t* __restrict__ dist,
               int32_t* __restrict__ pred, int level, int n_vertices, frontier_counters_t* cnt)
{
  const int lane     = threadIdx.x & 31;
  const int n_words  = (n_vertices + 31) >> 5;
  unsigned my_count  = 0;
  unsigned my_deg    = 0;
  for (int w = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5); w < n_words;
       w += (int)(((long long)gridDim.x * blockDim.x) >> 5)) {
    const uint32_t vis = visited[w];
    const int v        = (w << 5) + lane;
    bool found         = false;
    if (v < n_vertices && !((vis >> lane) & 1u)) {
      const long long beg = (long long)off[v], end = (long long)off[v + 1];
      for (long long e = beg; e < end; ++e) {
        const int u = idx[e];
        if ((frontier_bm[u >> 5] >> (u & 31)) & 1u) {
          dist[v] = level + 1;
          if (pred) pred[v] = u;
          found = true;
          my_count += 1;
          my_deg += (unsigned)(end - beg);
          break;
        }
      }
    }
    const uint32_t word = __ballot_sync(0xffffffffu, found);
    if (lane == 0) {
      next_bm[w] = word;
      if (word) visited[w] = vis | word;  // word w belongs to this warp alone: no separate OR pass over the bitmaps
    }
  }
  my_count = __reduce_add_sync(0xffffffffu, my_count);
  my_deg   = __reduce_add_sync(0xffffffffu, my_deg);
  if (lane == 0 && my_count) {
    atomicAdd(&cnt->n_small, (int)my_count);
    atomicAdd(&cnt->m_f, (unsigned long long)my_deg);
  }
}

__global__ void k_queue_to_bitmap(int32_t const* __restrict__ q, int n, uint32_t* __restrict__ bm)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) atomicOr(bm + (q[i] >> 5), 1u << (q[i] & 31));
}

__global__ void k_bitmap_to_queue(uint32_t const* __restrict__ bm, int n_words, int32_t* __restrict__ q, int* counter)
{
  // the whole CTA takes each step, so that every warp stays converged for its shuffles
  for (int64_t w0 = blockIdx.x * (int64_t)blockDim.x; w0 < n_words; w0 += (int64_t)gridDim.x * blockDim.x) {
    const int w   = (int)(w0 + threadIdx.x);
    uint32_t word = (w < n_words) ? bm[w] : 0u;
    int c         = __popc(word);
    // warp-level exclusive scan of counts, one atomic per warp
    int lane = threadIdx.x & 31;
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    int total = __shfl_sync(0xffffffffu, incl, 31);
    int base  = 0;
    if (lane == 31 && total) base = atomicAdd(counter, total);
    base = __shfl_sync(0xffffffffu, base, 31) + incl - c;
    while (word) {
      int b     = __ffs(word) - 1;
      q[base++] = (w << 5) + b;
      word &= word - 1;
    }
  }
}

template <typename O>
__global__ void k_bfs_seed(int32_t const* __restrict__ src, int n, uint32_t* visited, int32_t* dist, int32_t* q,
                           frontier_counters_t* cnt, O const* __restrict__ off)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int v        = src[i];
    uint32_t bit = 1u << (v & 31);
    uint32_t old = atomicOr(visited + (v >> 5), bit);
    if (old & bit) continue;  // duplicate source
    dist[v]     = 0;
    int pos     = atomicAdd(&cnt->n_small, 1);
    q[pos]      = v;
    unsigned d  = (unsigned)((long long)off[v + 1] - (long long)off[v]);
    atomicAdd(&cnt->m_f, (unsigned long long)d);
  }
}

__global__ void k_widen_dist(int32_t const* in, int32_t n, int64_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[i] == INT_MAX ? LLONG_MAX : (int64_t)in[i];
}

template <typename O>
void run_bfs(handle_impl const& h, csx_t const& c, int32_t nv, int32_t const* sources, int n_sources,
             bool direction_optimizing, int depth_limit, int32_t* dist, int32_t* pred)
{
  O const* off       = c.offsets.as<O>();
  int32_t const* idx = c.indices.as<int32_t>();
  const int n_words  = (nv + 31) / 32;
  dbuf visited = make_dbuf<uint32_t>(n_words, h.stream), fbm = make_dbuf<uint32_t>(n_words, h.stream),
       nbm = make_dbuf<uint32_t>(n_words, h.stream);
  dbuf qa = make_dbuf<int32_t>(nv, h.stream), qb = make_dbuf<int32_t>(nv, h.stream);
  dbuf la = make_dbuf<int32_t>((size_t)nv + 1, h.stream), lb = make_dbuf<int32_t>((size_t)nv + 1, h.stream);  // queue degrees
  dbuf cnt = make_dbuf<frontier_counters_t>(1, h.stream);
  frontier_counters_t* dc = cnt.as<frontier_counters_t>();
  CUDA_TRY(cudaMemsetAsync(visited.data(), 0, sizeof(uint32_t) * n_words, h.stream));
  CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
  B200_LAUNCH(h, (k_fill<int32_t>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, dist, (int64_t)nv, INT_MAX);
  if (pred) B200_LAUNCH(h, (k_fill<int32_t>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, pred, (int64_t)nv, -1);
  B200_LAUNCH(h, (k_bfs_seed<O>), grid_for(n_sources), kBlock, 0, sources, n_sources, visited.as<uint32_t>(), dist,
              qa.as<int32_t>(), dc, off);
  frontier_counters_t* hc = reinterpret_cast<frontier_counters_t*>(h.pinned);
  CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(frontier_counters_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  // the current frontier is either a queue (cur, with the entries' degrees in cur_l once a top-down level wrote it) or
  // a bitmap (fbm)
  int n_f                  = hc->n_small;
  unsigned long long m_f   = hc->m_f;
  unsigned long long m_vis = m_f;  // edges incident to visited vertices
  long long n_vis          = n_f;
  const unsigned long long m_total = (unsigned long long)c.nnz;
  int32_t *cur = qa.as<int32_t>(), *nxt = qb.as<int32_t>();
  int32_t *cur_l = la.as<int32_t>(), *nxt_l = lb.as<int32_t>();
  bool bottom_up = false, frontier_is_bitmap = false;
  bool deg_ready = false;  // cur_l holds the degrees of the entries of cur (written by the top-down level that built it)
  int level = 0, prev_n_f = 0;
  // Beamer's switch points (bfs_bottom_up, common.cuh): only the schedule depends on them, never the result
  const bool trace = h.tune.bfs_trace;
  advance_scratch_t adv;
  adv.init(h, nv, (int64_t)c.nnz);
  while (n_f > 0 && level < depth_limit) {
    if (direction_optimizing)
      bottom_up = bfs_bottom_up(h, bottom_up, n_f, prev_n_f, m_f, m_total - std::min(m_vis, m_total), nv - n_vis);
    CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
    if (!bottom_up) {
      if (frontier_is_bitmap) {
        B200_LAUNCH(h, k_bitmap_to_queue, grid_for(n_words), kBlock, 0, fbm.as<uint32_t>(), n_words, cur, &dc->n_conv);
        frontier_is_bitmap = false;
        deg_ready          = false;
      }
      bfs_topdown_op<O> op{off, visited.as<uint32_t>(), dist, pred, nxt, nxt_l, dc, level};
      advance<O>(h, adv, off, idx, cur, n_f, m_f, op, deg_ready ? cur_l : (int32_t const*)nullptr);
      std::swap(cur, nxt);
      std::swap(cur_l, nxt_l);
      deg_ready = true;
    } else {
      if (!frontier_is_bitmap) {
        CUDA_TRY(cudaMemsetAsync(fbm.data(), 0, sizeof(uint32_t) * n_words, h.stream));
        if (n_f > 0) B200_LAUNCH(h, k_queue_to_bitmap, grid_for(n_f), kBlock, 0, cur, n_f, fbm.as<uint32_t>());
        frontier_is_bitmap = true;
      }
      int grid = grid_for((int64_t)n_words * 32, 1, h.sm_count * 16);
      B200_LAUNCH(h, (k_bfs_bottomup<O>), grid, kBlock, 0, off, idx, visited.as<uint32_t>(), fbm.as<uint32_t>(),
                  nbm.as<uint32_t>(), dist, pred, level, nv, dc);
      std::swap(fbm, nbm);
    }
    CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(frontier_counters_t), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    if (trace)
      std::fprintf(stderr, "bfs level %d %s n_f=%d m_f=%llu m_vis=%llu n_vis=%lld -> next n_f=%d m_f=%llu\n", level,
                   bottom_up ? "bottom-up" : "top-down", n_f, m_f, m_vis, n_vis, hc->n_small, hc->m_f);
    prev_n_f = n_f;
    n_f      = hc->n_small;  // both directions count the next frontier in n_small
    m_f      = hc->m_f;
    m_vis += m_f;
    n_vis += n_f;
    ++level;
  }
  check_last("bfs");
}

// ------------------------------------------------------------------------------------------
// Multi-source BFS: one BFS per source, a batch of up to 64 sources per pass over the graph (bit-parallel BFS: Then et al.,
// "The More the Merrier", VLDB 2015).  Bit j of a vertex's 64-bit words stands for source j of the batch:
//   seen : the sources that have reached the vertex;   cur : those that reached it at this level;   next : at the next one.
// A top-down level advances the vertices with a non-zero cur word (a queue, as in run_bfs) and ORs cur[u] into next[v] for
// every edge u -> v; a bottom-up level ORs the cur words of v's in-edges into the bits v still wants.  One edge read
// advances every BFS of the batch.  dist / pred hold one int32 row of V entries per source of the batch, row j at j * V.
// ------------------------------------------------------------------------------------------
struct ms_counters_t {
  frontier_counters_t f;        // next frontier: vertices with a non-zero word (n_small, n_conv) and their out-degree sum (m_f)
  unsigned long long n_full;    // vertices whose seen word became the whole batch ...
  unsigned long long m_full;    // ... and their out-degree sum (Beamer's rule counts them as visited)
};

// write distance d (and predecessor u) of vertex v into the rows of the bits set in `bits`
__device__ __forceinline__ void ms_write_rows(unsigned long long bits, int v, long long nv, int32_t d, int32_t* dist, int32_t* pred,
                                              int u)
{
  if (!dist) return;  // betweenness: the levels are kept as queues instead (ms_level_sink)
  while (bits) {
    const long long j = __ffsll((long long)bits) - 1;
    dist[j * nv + v] = d;
    if (pred) pred[j * nv + v] = u;
    bits &= bits - 1;
  }
}

// the four level counters of a thread, summed over the warp and added with one atomic each (every lane must call it)
__device__ __forceinline__ void ms_commit(ms_counters_t* cnt, unsigned long long n, unsigned long long m, unsigned long long n_full,
                                          unsigned long long m_full)
{
  n = warp_sum_u64(n), m = warp_sum_u64(m), n_full = warp_sum_u64(n_full), m_full = warp_sum_u64(m_full);
  if ((threadIdx.x & 31) == 0) {
    if (n) atomicAdd(&cnt->f.n_small, (int)n);
    if (m) atomicAdd(&cnt->f.m_f, m);
    if (n_full) atomicAdd(&cnt->n_full, n_full);
    if (m_full) atomicAdd(&cnt->m_full, m_full);
  }
}

template <typename O>
__device__ __forceinline__ unsigned long long out_degree(O const* off, int v)
{
  return (unsigned long long)((long long)off[v + 1] - (long long)off[v]);
}

// bit j for source j of the batch; every distinct source vertex is queued once, with its degree
template <typename O>
__global__ void k_ms_seed(int32_t const* __restrict__ src, int n, O const* __restrict__ off, unsigned long long* seen,
                          unsigned long long* cur, int32_t* dist, long long nv, unsigned long long mask, int32_t* q, int32_t* q_deg,
                          ms_counters_t* cnt)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int v                   = src[i];
    const unsigned long long bit  = 1ull << i;
    const unsigned long long old  = atomicOr(seen + v, bit);
    atomicOr(cur + v, bit);
    if (dist) dist[i * nv + v] = 0;
    if (old == 0) {
      const unsigned d = enqueue_with_degree(off, v, q, q_deg, &cnt->f);
      atomicAdd(&cnt->f.m_f, (unsigned long long)d);
    }
    if ((old | bit) == mask) {
      atomicAdd(&cnt->n_full, 1ull);
      atomicAdd(&cnt->m_full, out_degree(off, v));
    }
  }
}

// top-down edge u -> v: the sources that reached u at this level and have not reached v.  seen is read-only during the
// level (k_ms_fold folds next into it afterwards); the thread whose atomicOr set a bit first writes that source's row.
template <typename O>
struct ms_topdown_op {
  O const* off;
  unsigned long long const* cur;
  unsigned long long const* seen;
  unsigned long long* next;
  int32_t* dist;
  int32_t* pred;  // may be null
  long long nv;
  int32_t* next_q;
  int32_t* next_q_deg;
  frontier_counters_t* cnt;
  int level;
  __device__ __forceinline__ void edge(int src, long long, int nbr) const
  {
    const unsigned long long bits = cur[src] & ~seen[nbr];
    if (!(bits & ~next[nbr])) return;  // next only gains bits during the level: a stale read costs an atomic, never a bit
    const unsigned long long old = atomicOr(next + nbr, bits);
    ms_write_rows(bits & ~old, nbr, nv, level + 1, dist, pred, src);
    if (old == 0) {
      const unsigned d = enqueue_with_degree(off, nbr, next_q, next_q_deg, cnt);
      warp_add_u64(&cnt->m_f, d);
    }
  }
};

// after a top-down level: seen |= next for the vertices of the new queue (*n_new entries, written by the level), and the
// cur words of the old queue are cleared, so that cur serves as the next level's all-zero `next`
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_ms_fold(int32_t const* __restrict__ old_q, int n_old, int32_t const* __restrict__ new_q, int const* __restrict__ n_new,
          unsigned long long* __restrict__ cur, unsigned long long const* __restrict__ next, unsigned long long* __restrict__ seen,
          unsigned long long mask, O const* __restrict__ off, ms_counters_t* cnt)
{
  const long long n = (long long)n_old + *n_new;
  unsigned long long n_full = 0, m_full = 0;
  for (long long i0 = blockIdx.x * (long long)blockDim.x; i0 < n; i0 += (long long)gridDim.x * blockDim.x) {
    const long long i = i0 + threadIdx.x;
    if (i < n_old) {
      cur[old_q[i]] = 0ull;
    } else if (i < n) {
      const int v                    = new_q[i - n_old];
      const unsigned long long s     = seen[v] | next[v];
      seen[v]                        = s;
      if (s == mask) {  // next[v] holds bits seen[v] lacked: the word became whole now
        n_full += 1;
        m_full += out_degree(off, v);
      }
    }
  }
  ms_commit(cnt, 0, 0, n_full, m_full);
}

// Bottom-up level over the physical rows of the in-edge view: v ORs cur[u] & want over its in-edges u, want = the batch
// bits v has not seen, and stops once every wanted bit is found.  The predecessor of a bit is the in-neighbour that first
// supplied it.  The kernel owns v's words: it writes next[v], seen[v] and v's entries of the rows itself.  Rows are sorted
// by descending in-degree: the first n_hub (degree >= 32) are read by a warp each, 32 in-edges per step with a prefix OR
// over the lanes to find which lane supplied a bit first; the rest by a thread each.
template <typename OI, typename O>
__global__ void __launch_bounds__(kBlock)
k_ms_bottomup(OI const* __restrict__ in_off, int32_t const* __restrict__ in_idx, int32_t const* __restrict__ row_vertex,
              int n_rows, int n_hub, O const* __restrict__ off, unsigned long long const* __restrict__ cur,
              unsigned long long* __restrict__ next, unsigned long long* __restrict__ seen, int32_t* __restrict__ dist,
              int32_t* __restrict__ pred, long long nv, unsigned long long mask, int level, ms_counters_t* cnt)
{
  const int lane         = threadIdx.x & 31;
  const long long tid    = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned long long c_n = 0, c_m = 0, c_full = 0, c_mfull = 0;
  for (long long r = tid >> 5; r < n_hub; r += stride >> 5) {
    const int v                     = row_vertex ? row_vertex[r] : (int)r;
    const unsigned long long s      = seen[v];
    const unsigned long long want   = ~s & mask;
    if (!want) continue;  // warp-uniform
    unsigned long long found = 0;
    const long long end      = (long long)in_off[r + 1];
    for (long long e0 = (long long)in_off[r]; e0 < end; e0 += 32) {
      const long long e             = e0 + lane;
      const int u                   = e < end ? in_idx[e] : 0;
      const unsigned long long mine = e < end ? cur[u] & want & ~found : 0ull;
      unsigned long long incl       = mine;  // inclusive prefix OR over the lanes
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl |= t;
      }
      const unsigned long long before = __shfl_up_sync(0xffffffffu, incl, 1);
      ms_write_rows(lane ? mine & ~before : mine, v, nv, level + 1, dist, pred, u);
      found |= __shfl_sync(0xffffffffu, incl, 31);
      if (found == want) break;
    }
    if (lane == 0 && found) {
      next[v] = found;
      seen[v] = s | found;
      c_n += 1;
      c_m += out_degree(off, v);
      if ((s | found) == mask) {
        c_full += 1;
        c_mfull += out_degree(off, v);
      }
    }
  }
  for (long long r = n_hub + tid; r < n_rows; r += stride) {
    const int v                   = row_vertex ? row_vertex[r] : (int)r;
    const unsigned long long s    = seen[v];
    const unsigned long long want = ~s & mask;
    if (!want) continue;
    unsigned long long found = 0;
    const long long end      = (long long)in_off[r + 1];
    for (long long e = (long long)in_off[r]; e < end; ++e) {
      const int u                   = in_idx[e];
      const unsigned long long bits = cur[u] & want & ~found;
      if (!bits) continue;
      ms_write_rows(bits, v, nv, level + 1, dist, pred, u);
      found |= bits;
      if (found == want) break;
    }
    if (found) {
      next[v] = found;
      seen[v] = s | found;
      c_n += 1;
      c_m += out_degree(off, v);
      if ((s | found) == mask) {
        c_full += 1;
        c_mfull += out_degree(off, v);
      }
    }
  }
  ms_commit(cnt, c_n, c_m, c_full, c_mfull);
}

// One batch of nb <= 64 sources (internal ids).  dist and pred (each may be null) hold nb rows of nv entries, filled here.
// Direction per level: Beamer's rule (bfs_bottom_up), with a vertex counted as visited once every source of the batch has
// reached it.  Only the schedule depends on it, never the result.  sink (may be null) is handed every level's frontier.
template <typename O>
void run_multi_source_bfs_batch(handle_impl const& h, graph_impl& g, csx_t const& c, int32_t nv, int32_t const* sources, int nb,
                                int depth_limit, int32_t* dist, int32_t* pred, int batch, ms_level_sink* sink)
{
  using u64          = unsigned long long;
  O const* off       = c.offsets.as<O>();
  int32_t const* idx = c.indices.as<int32_t>();
  const u64 mask     = nb == 64 ? ~0ull : (1ull << nb) - 1ull;
  const long long cells = (long long)nb * nv;
  dbuf seen = make_dbuf<u64>(nv, h.stream), wa = make_dbuf<u64>(nv, h.stream), wb = make_dbuf<u64>(nv, h.stream);
  for (dbuf* w : {&seen, &wa, &wb}) CUDA_TRY(cudaMemsetAsync(w->data(), 0, sizeof(u64) * nv, h.stream));
  dbuf qa = make_dbuf<int32_t>(nv, h.stream), qb = make_dbuf<int32_t>(nv, h.stream);
  dbuf la = make_dbuf<int32_t>((size_t)nv + 1, h.stream), lb = make_dbuf<int32_t>((size_t)nv + 1, h.stream);  // queue degrees
  dbuf cnt = make_dbuf<ms_counters_t>(1, h.stream);
  ms_counters_t* dc = cnt.as<ms_counters_t>();
  CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(ms_counters_t), h.stream));
  if (dist) B200_LAUNCH(h, (k_fill<int32_t>), grid_for(cells, 1, h.sm_count * 32), kBlock, 0, dist, (int64_t)cells, INT_MAX);
  if (pred) B200_LAUNCH(h, (k_fill<int32_t>), grid_for(cells, 1, h.sm_count * 32), kBlock, 0, pred, (int64_t)cells, -1);
  u64 *cur = wa.as<u64>(), *nxt = wb.as<u64>();
  int32_t *cur_q = qa.as<int32_t>(), *nxt_q = qb.as<int32_t>();
  int32_t *cur_l = la.as<int32_t>(), *nxt_l = lb.as<int32_t>();
  B200_LAUNCH(h, (k_ms_seed<O>), 1, 64, 0, sources, nb, off, seen.as<u64>(), cur, dist, (long long)nv, mask, cur_q, cur_l, dc);
  auto* hc = reinterpret_cast<ms_counters_t*>(h.pinned);
  CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(ms_counters_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  int n_f = hc->f.n_small, prev_n_f = 0;
  u64 m_f = hc->f.m_f, m_full = hc->m_full;
  long long n_full = (long long)hc->n_full;
  const u64 m_total = (u64)c.nnz;
  // the frontier is the cur words, and also a queue (cur_q; degrees in cur_l once a top-down level or the seed wrote them)
  // except after a bottom-up level
  bool bottom_up = false, have_queue = true, deg_ready = true;
  csx_t const* in = nullptr;  // the in-edge view, fetched at the first bottom-up level (a non-symmetric CSR graph builds it then)
  advance_scratch_t adv;
  adv.init(h, nv, (int64_t)c.nnz);
  const bool trace = h.tune.bfs_trace;
  if (sink && n_f > 0) sink->level(0, cur, cur_q, n_f);
  for (int level = 0; n_f > 0 && level < depth_limit; ++level) {
    const auto t0 = std::chrono::steady_clock::now();
    bottom_up     = bfs_bottom_up(h, bottom_up, n_f, prev_n_f, m_f, m_total - std::min(m_full, m_total), nv - n_full);
    CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(ms_counters_t), h.stream));
    if (!bottom_up) {
      if (!have_queue) {
        B200_LAUNCH(h, k_ms_words_to_queue, grid_for(nv, 1, h.sm_count * 16), kBlock, 0, cur, nv, cur_q, &dc->f.n_conv);
        have_queue = true;
        deg_ready  = false;
      }
      ms_topdown_op<O> op{off, cur, seen.as<u64>(), nxt, dist, pred, (long long)nv, nxt_q, nxt_l, &dc->f, level};
      advance<O>(h, adv, off, idx, cur_q, n_f, m_f, op, deg_ready ? cur_l : (int32_t const*)nullptr);
      B200_LAUNCH(h, (k_ms_fold<O>), grid_for((int64_t)n_f + nv, 1, h.sm_count * 8), kBlock, 0, cur_q, n_f, nxt_q,
                  &dc->f.n_small, cur, nxt, seen.as<u64>(), mask, off, dc);
      std::swap(cur_q, nxt_q);
      std::swap(cur_l, nxt_l);
      deg_ready = true;
    } else {
      if (!in) in = &pull_view(h, g);  // rows = destinations: the primary itself on a symmetric or transposed graph
      const int n_hub = in->seg[0];    // rows of in-degree >= 32
      const int grid  = grid_for(std::max<int64_t>((int64_t)n_hub * 32, (int64_t)nv - n_hub), 1, h.sm_count * 16);
      if (in->offs64)
        B200_LAUNCH(h, (k_ms_bottomup<int64_t, O>), grid, kBlock, 0, in->offsets.as<int64_t>(), in->indices.as<int32_t>(),
                    in->row_vertex.as<int32_t>(), in->n_rows, n_hub, off, cur, nxt, seen.as<u64>(), dist, pred, (long long)nv,
                    mask, level, dc);
      else
        B200_LAUNCH(h, (k_ms_bottomup<int32_t, O>), grid, kBlock, 0, in->offsets.as<int32_t>(), in->indices.as<int32_t>(),
                    in->row_vertex.as<int32_t>(), in->n_rows, n_hub, off, cur, nxt, seen.as<u64>(), dist, pred, (long long)nv,
                    mask, level, dc);
      CUDA_TRY(cudaMemsetAsync(cur, 0, sizeof(u64) * nv, h.stream));
      have_queue = false;
    }
    std::swap(cur, nxt);
    CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(ms_counters_t), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    if (trace)
      std::fprintf(stderr, "ms-bfs batch %d level %d %s n_f=%d m_f=%llu full=%lld -> next n_f=%d m_f=%llu, %.3f ms\n", batch, level,
                   bottom_up ? "bottom-up" : "top-down", n_f, m_f, n_full, hc->f.n_small, hc->f.m_f,
                   std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    prev_n_f = n_f;
    n_f      = hc->f.n_small;
    m_f      = hc->f.m_f;
    n_full += (long long)hc->n_full;
    m_full += hc->m_full;
    if (sink && n_f > 0) sink->level(level + 1, cur, have_queue ? cur_q : nullptr, n_f);
  }
  check_last("multi_source_bfs");
}

}  // namespace

void multi_source_bfs_batch(handle_impl const& h, graph_impl& g, int32_t const* sources, int nb, int depth_limit, int32_t* dist,
                            int32_t* pred, int batch, ms_level_sink* sink)
{
  csx_t const& c = push_view(h, g);
  if (c.offs64)
    run_multi_source_bfs_batch<int64_t>(h, g, c, g.n_vertices, sources, nb, depth_limit, dist, pred, batch, sink);
  else
    run_multi_source_bfs_batch<int32_t>(h, g, c, g.n_vertices, sources, nb, depth_limit, dist, pred, batch, sink);
}

namespace {

// ------------------------------------------------------------------------------------------
// SSSP: near/far piles with threshold stepping (sssp_impl.cuh:246-265, 373-566)
// ------------------------------------------------------------------------------------------
// There is no far PILE: the vertices a window [lo, hi) has to relax are exactly those whose tentative distance lies in
// it (a vertex enters a near queue only when its distance drops below the current bound, so anything at or beyond the
// bound has never been relaxed at its current distance).  The next window's queue is therefore selected by ONE dense,
// coalesced pass over the distance array (35 MB at RMAT-24, ~10 us) instead of splitting a queue of up to 7.6 M far
// vertices with three random accesses each at every window change (that split once took more than half of a traversal).
// Where the tentative distances live.  dist_plain: one word per vertex, lowered with an atomic min (non-negative floats
// order as integers); predecessors, if wanted, come from a pass over the distance fixpoint afterwards.  dist_packed (float
// with predecessors): (distance bits << 32 | predecessor) in one 64-bit word lowered with ONE atomic min, i.e. the
// predecessor is recorded by the relaxation that set the distance, as in the reference (sssp_impl.cuh:43-73,
// reduce_op::minimum over (distance, predecessor) tuples): always a tree and no predecessor pass.  The word only changes on a
// STRICT improvement of the distance, so a vertex's parent attained its distance before the vertex did: no cycles through
// zero-weight or absorbed edges.
template <typename T>
struct dist_plain {
  T* d;
  __device__ __forceinline__ T get(int v) const { return d[v]; }
  __device__ __forceinline__ T get_fresh(int v) const { return *reinterpret_cast<volatile T const*>(d + v); }  // not through a stale L1 line
  __device__ __forceinline__ bool improve(int v, T nd, int) const { return nd < atomic_min_nonneg(d + v, nd); }
  __device__ __forceinline__ void set_source(int v) const { d[v] = (T)0; }
};
struct dist_packed {
  unsigned long long* p;
  static __host__ __device__ __forceinline__ unsigned long long pack(unsigned dist_bits, int pred)
  {
    return ((unsigned long long)dist_bits << 32) | (unsigned)pred;
  }
  __device__ __forceinline__ float get(int v) const { return __uint_as_float((unsigned)(p[v] >> 32)); }
  __device__ __forceinline__ float get_fresh(int v) const
  {
    return __uint_as_float((unsigned)(*reinterpret_cast<volatile unsigned long long const*>(p + v) >> 32));
  }
  // STRICT improvement only (compare-and-swap loop): with a plain 64-bit atomicMin a relaxation at an EQUAL distance and a
  // smaller source id would replace the predecessor; the pre-check that should prevent it reads through L1, which is not
  // coherent with the other SMs' atomics, and on hardware that produced predecessor cycles inside zero-weight cycles.
  // With strict improvements every vertex's parent attained its value before the vertex did: always a tree.
  __device__ __forceinline__ bool improve(int v, float nd, int src) const
  {
    const unsigned long long want = pack(__float_as_uint(nd), src);
    unsigned long long cur        = *reinterpret_cast<volatile unsigned long long*>(p + v);
    while (nd < __uint_as_float((unsigned)(cur >> 32))) {
      const unsigned long long prev = atomicCAS(p + v, cur, want);
      if (prev == cur) return true;
      cur = prev;
    }
    return false;
  }
  __device__ __forceinline__ void set_source(int v) const { p[v] = pack(0u, -1); }
};

__global__ void k_unpack_dist(unsigned long long const* __restrict__ p, int n, float* __restrict__ dist, int32_t* __restrict__ pred)
{
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long x = p[v];
    dist[v]                    = __uint_as_float((unsigned)(x >> 32));
    pred[v]                    = (int32_t)(unsigned)(x & 0xffffffffu);
  }
}

template <typename O, typename T, typename DA>
struct sssp_relax_op {
  O const* off;
  T const* w;
  DA dist;
  int32_t* stamp;  // round in which the vertex was last put on a near queue
  int32_t* next_near;
  int32_t* next_near_deg;  // degrees of the entries of next_near
  frontier_counters_t* cnt;
  T threshold;
  T cutoff;
  int round;
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const T nd = dist.get(src) + w[e];
    if (!(nd < dist.get(nbr)) || !(nd < cutoff)) return;
    if (!dist.improve(nbr, nd, src)) return;
    if (nd < threshold) {
      if (atomicExch(stamp + nbr, round) != round) enqueue_counted(off, nbr, next_near, next_near_deg, cnt);
    }
  }
};

// ---- rounds with a SMALL near queue run inside ONE CTA, round after round, without the host: on RMAT-24 two thirds of the
// ~208 rounds of a traversal relax fewer than 16 K edges, and each cost ~45 us of launches (scan, tile owners, advance) plus a
// read-back.  The CTA scans the degrees of the queue (<= kSmallVerts entries) in shared memory, strides over the edges
// (owner by binary search in the scan), relaxes them exactly like sssp_relax_op and appends to the other queue through a
// shared-memory counter; it stops when the window's queue is empty, outgrows the limits or max_rounds is reached, and leaves
// the state for the host.  Distances are read with volatile loads: within one kernel the L1 may hold the value from before
// another thread's atomic improved it — relaxing from a stale (larger) distance would lose the improvement for good.
constexpr int kSmallVerts   = 2048;
constexpr int kSmallEdges   = 16384;
constexpr int kSmallThreads = 1024;
struct sssp_small_state_t {
  int n;                     // entries of the queue that is current on exit
  int round;                 // last round number used
  int rounds_done;
  int cur;                   // 0: the current queue is the one passed as `qa`, 1: `qb`
  unsigned long long edges;  // degree sum of the current queue
  unsigned long long relaxed;  // edges relaxed by this call (trace)
};

template <typename O, typename T, typename DA>
__global__ void __launch_bounds__(kSmallThreads)
k_sssp_small_rounds(O const* __restrict__ off, int32_t const* __restrict__ idx, T const* __restrict__ w, DA dist, int32_t* stamp,
                    int32_t* qa, int32_t* la, int32_t* qb, int32_t* lb, int n0, int round0, T threshold, T cutoff, int max_rounds,
                    sssp_small_state_t* __restrict__ out)
{
  __shared__ int s_scan[kSmallVerts + 1];
  __shared__ int s_warp[kSmallThreads / 32];
  __shared__ unsigned long long s_next;  // (degree sum << 32) | entries of the next queue
  constexpr int kPer = kSmallVerts / kSmallThreads;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int32_t *q = qa, *l = la, *nq = qb, *nl = lb;
  int n = n0, round = round0, done = 0, cur = 0;
  unsigned long long edges = 0, relaxed = 0;
  while (true) {
    // exclusive scan of the queue's degrees
    int d[kPer], mine = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = threadIdx.x * kPer + j;
      d[j]        = i < n ? l[i] : 0;
      mine += d[j];
    }
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[wid] = incl;
    if (threadIdx.x == 0) s_next = 0ull;
    __syncthreads();
    int before = 0, total = 0;
    for (int k = 0; k < kSmallThreads / 32; ++k) {
      const int c = s_warp[k];
      if (k < wid) before += c;
      total += c;
    }
    int run = before + incl - mine;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = threadIdx.x * kPer + j;
      if (i <= n) s_scan[i] = run;
      run += d[j];
    }
    if (threadIdx.x == 0) s_scan[n] = total;  // n <= kSmallVerts: the slot exists
    __syncthreads();
    ++round;
    relaxed += (unsigned long long)total;
    for (int e = threadIdx.x; e < total; e += kSmallThreads) {
      int lo = 0, hi = n;  // last k with s_scan[k] <= e
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_scan[mid] <= e) lo = mid; else hi = mid;
      }
      const int v         = q[lo];
      const long long pos = (long long)off[v] + (e - s_scan[lo]);
      const int nbr       = idx[pos];
      const T nd          = dist.get_fresh(v) + w[pos];
      if (!(nd < dist.get_fresh(nbr)) || !(nd < cutoff)) continue;
      if (!dist.improve(nbr, nd, v)) continue;
      if (nd < threshold && atomicExch(stamp + nbr, round) != round) {
        const unsigned dg = (unsigned)((long long)off[nbr + 1] - (long long)off[nbr]);
        const int p       = (int)(unsigned)(atomicAdd(&s_next, ((unsigned long long)dg << 32) | 1ull) & 0xffffffffull);
        nq[p]             = nbr;
        nl[p]             = (int32_t)dg;
      }
    }
    __syncthreads();
    const unsigned long long nx = s_next;
    n     = (int)(unsigned)(nx & 0xffffffffull);
    edges = nx >> 32;
    ++done;
    cur ^= 1;
    int32_t* t = q; q = nq; nq = t;
    t = l; l = nl; nl = t;
    __syncthreads();  // everybody has read s_next before thread 0 clears it
    if (n == 0 || n > kSmallVerts || edges > (unsigned long long)kSmallEdges || done >= max_rounds) break;
  }
  if (threadIdx.x == 0) {
    out->n           = n;
    out->round       = round;
    out->rounds_done = done;
    out->cur         = cur;
    out->edges       = edges;
    out->relaxed     = relaxed;
  }
}

// mid-window split: keep the queue entries below the new bound (the others are found again by the window selection)
template <typename O, typename T, typename DA>
__global__ void k_split_near(O const* __restrict__ off, int32_t const* __restrict__ q_in, int n, DA dist,
                             T hi, int32_t* stamp, int round, int32_t* near_out, int32_t* near_deg_out,
                             frontier_counters_t* cnt)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = q_in[i];
    if (dist.get(v) < hi) {
      stamp[v] = round;
      enqueue_counted(off, v, near_out, near_deg_out, cnt);
    }
  }
}

// dense pass 1: smallest tentative distance at or beyond `hi` (reached vertices only)
template <typename T, typename DA>
__global__ void k_min_beyond(DA dist, int n, T hi, T unreached, T* out_min)
{
  T m = (T)INFINITY;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T d = dist.get(i);
    if (d >= hi && d < unreached && d < m) m = d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    T t = __shfl_xor_sync(0xffffffffu, m, o);
    m   = t < m ? t : m;
  }
  if ((threadIdx.x & 31) == 0 && m < (T)INFINITY) atomic_min_nonneg(out_min, m);
}

// the window state lives on the device: the next window's bounds are computed from the result of pass 1 by a one-thread
// kernel, pass 2 reads them — one host synchronisation per window change instead of two
template <typename T>
struct sssp_window_t {
  T lo, hi;
  int any;  // 0: nothing is pending beyond the old bound (the traversal is complete)
};
template <typename T>
__global__ void k_next_window(T const* __restrict__ pending_min, T delta, sssp_window_t<T>* __restrict__ win)
{
  const T hmin = *pending_min, hi = win->hi;
  const T inf  = (T)INFINITY;
  if (!(hmin < inf)) {
    win->any = 0;
    return;
  }
  const T steps = floor((hmin - hi) / delta);
  T nhi         = hi + (steps > (T)0 ? steps : (T)0) * delta + delta;
  if (!(nhi > hmin)) nhi = nextafter(hmin, inf);  // rounding must not produce a window without its smallest entry
  win->lo  = hi;
  win->hi  = nhi;
  win->any = 1;
}

// dense pass 2: the vertices of the window [lo, hi) form the next near queue.  Block-level compaction: a CTA looks at 2048
// consecutive vertices per step and reserves queue space with ONE atomic (the per-warp appends of the first version were
// up to 275 K atomics on one address per window: 139 us per pass, 9.5 ms of a 31 ms traversal on RMAT-24).
constexpr int kSelectPer = 8;  // vertices per thread and step
template <typename O, typename T, typename DA>
__global__ void __launch_bounds__(kBlock)
k_select_window(O const* __restrict__ off, DA dist, int n, sssp_window_t<T> const* __restrict__ win, int32_t* stamp,
                int round, int32_t* near_out, int32_t* near_deg_out, frontier_counters_t* cnt)
{
  if (!win->any) return;
  __shared__ int s_warp[kBlock / 32];
  __shared__ long long s_base;
  const T lo = win->lo, hi = win->hi;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (long long base = (long long)blockIdx.x * (kBlock * kSelectPer); base < n; base += (long long)gridDim.x * (kBlock * kSelectPer)) {
    unsigned sel = 0;
    int mine     = 0;
#pragma unroll
    for (int k = 0; k < kSelectPer; ++k) {
      const long long v = base + k * kBlock + threadIdx.x;
      if (v < n) {
        const T d = dist.get((int)v);
        if (d >= lo && d < hi) {
          sel |= 1u << k;
          ++mine;
        }
      }
    }
    int incl = mine;  // inclusive scan over the CTA
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kBlock / 32; ++w) {
      const int c = s_warp[w];
      if (w < wid) before += c;
      total += c;
    }
    if (total > 0) {  // CTA-uniform
      unsigned long long dsum = 0;
      // degrees first: the reservation carries their sum
      int32_t dg[kSelectPer];
#pragma unroll
      for (int k = 0; k < kSelectPer; ++k) {
        dg[k] = 0;
        if (sel & (1u << k)) {
          const long long v = base + k * kBlock + threadIdx.x;
          dg[k]             = (int32_t)((long long)off[v + 1] - (long long)off[v]);
          dsum += (unsigned)dg[k];
        }
      }
      unsigned long long wsum = dsum;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
      __shared__ unsigned long long s_deg[kBlock / 32];
      if (lane == 0) s_deg[wid] = wsum;
      __syncthreads();
      if (threadIdx.x == 0) {
        unsigned long long ds = 0;
        for (int w = 0; w < kBlock / 32; ++w) ds += s_deg[w];
        if (sizeof(O) == 8) {
          s_base = atomicAdd(&cnt->n_small, total);
          atomicAdd(&cnt->m_f, ds);
        } else {
          s_base = (long long)(atomicAdd(&cnt->packed, (ds << 32) | (unsigned)total) & 0xffffffffull);
        }
      }
      __syncthreads();
      int pos = (int)s_base + before + incl - mine;
#pragma unroll
      for (int k = 0; k < kSelectPer; ++k) {
        if (sel & (1u << k)) {
          const int v       = (int)(base + k * kBlock + threadIdx.x);
          stamp[v]          = round;
          near_out[pos]     = v;
          near_deg_out[pos] = dg[k];
          ++pos;
        }
      }
    }
    __syncthreads();  // s_warp / s_base are reused by the next step
  }
}

// Predecessors from the distance fixpoint (double weights, and float without the packed word).  A tree parent u of v has
// dist[v] == fl(dist[u] + w(u,v)); with dist[u] < dist[v] any such u is valid and the parent pointers cannot form a cycle
// (distances strictly decrease along them).  Tight edges between vertices at the SAME distance (zero-weight edges, or a
// weight absorbed by rounding) are tight in both directions on a symmetric graph: pass 1 therefore only accepts strictly
// closer parents.  Vertices left without a parent (their distance arrived over a same-distance edge) are attached in extra
// passes, each to a tight same-distance neighbour that ALREADY has a parent (or is the source), with a compare-and-swap
// from "none": a parent pointer is written once, so a vertex only ever points at a vertex attached before it, and a cycle —
// which could only consist of same-distance edges — would need one that points at a later one.  (An id-ordered acceptance
// inside a plateau in pass 1 looked like a shortcut and is wrong: x takes the smaller-id v in pass 1, the orphan v then finds
// the "attached" x.)  The reference records the predecessor at the relaxation that set the distance, sssp_impl.cuh:43-73.
// An unreached vertex holds max(), which a sum that rounds to exactly max() would match: it never takes a parent.
template <typename O, typename T>
__global__ void k_sssp_pred(O const* __restrict__ off, int32_t const* __restrict__ idx, T const* __restrict__ w,
                            T const* __restrict__ dist, int32_t n_vertices, int32_t source, T unreached,
                            int32_t* __restrict__ pred)
{
  const int lane = threadIdx.x & 31;
  for (long long u = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; u < n_vertices;
       u += ((long long)gridDim.x * blockDim.x) >> 5) {
    const T du = dist[u];
    if (du == unreached) continue;
    for (long long e = (long long)off[u] + lane; e < (long long)off[u + 1]; e += 32) {
      const int v = idx[e];
      const T dv  = dist[v];
      if (v != source && v != (int)u && du < dv && dv != unreached && du + w[e] == dv) pred[v] = (int32_t)u;
    }
  }
}

template <typename T>
struct sssp_pred_op {
  T const* w;
  T const* dist;
  int32_t* pred;
  int32_t source;
  T unreached;
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const T du = dist[src], dv = dist[nbr];
    if (du != unreached && dv != unreached && nbr != source && nbr != src && du < dv && du + w[e] == dv) pred[nbr] = src;
  }
};

// one pass of the equal-distance attachment, edge-balanced (advance_all_edges)
template <typename T>
struct sssp_tie_op {
  T const* w;
  T const* dist;
  int32_t* pred;
  int32_t source;
  T unreached;
  int* changed;
  __device__ __forceinline__ void edge(int src, long long e, int nbr) const
  {
    const T du = dist[src];
    if (du == unreached || nbr == source || nbr == src || dist[nbr] != du || du + w[e] != du) return;
    if (src != source && ((volatile int32_t*)pred)[src] < 0) return;  // src itself is not attached yet
    if (((volatile int32_t*)pred)[nbr] >= 0) return;
    if (atomicCAS(pred + nbr, -1, (int32_t)src) == -1) *changed = 1;
  }
};

// reached vertices other than the source that still have no parent
template <typename T>
__global__ void k_sssp_count_orphans(T const* __restrict__ dist, int32_t const* __restrict__ pred, int32_t n, int32_t source,
                                     T unreached, int* __restrict__ out)
{
  int c = 0;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    c += (v != source && dist[v] != unreached && pred[v] < 0) ? 1 : 0;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// one pass of the equal-distance attachment: v (no parent yet) takes a tight neighbour u at the same distance that
// already has a parent or is the source
template <typename O, typename T>
__global__ void k_sssp_pred_ties(O const* __restrict__ off, int32_t const* __restrict__ idx, T const* __restrict__ w,
                                 T const* __restrict__ dist, int32_t n_vertices, int32_t source, T unreached,
                                 int32_t* __restrict__ pred, int* __restrict__ changed)
{
  const int lane = threadIdx.x & 31;
  for (long long u = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; u < n_vertices;
       u += ((long long)gridDim.x * blockDim.x) >> 5) {
    const T du = dist[u];
    if (du == unreached) continue;
    if ((int)u != source && ((volatile int32_t*)pred)[u] < 0) continue;  // u itself is not attached yet
    for (long long e = (long long)off[u] + lane; e < (long long)off[u + 1]; e += 32) {
      const int v = idx[e];
      if (v == source || v == (int)u || dist[v] != du || du + w[e] != du) continue;
      if (atomicCAS(pred + v, -1, (int32_t)u) == -1) *changed = 1;
    }
  }
}

template <typename T>
__global__ void k_sum_weights(T const* __restrict__ w, long long n, double* out)
{
  double s = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) s += (double)w[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}

template <typename O, typename DA>
__global__ void k_sssp_seed(DA dist, int32_t* stamp, int32_t* q, int32_t* q_deg, O const* off, int32_t source)
{
  dist.set_source(source);
  stamp[source] = 1;
  q[0]          = source;
  q_deg[0]      = (int32_t)((long long)off[source + 1] - (long long)off[source]);
}

// the window loop; the distances are initialised (unreached everywhere) by the caller
template <typename O, typename T, typename DA>
void sssp_windows(handle_impl const& h, csx_t const& c, int32_t nv, int32_t source, double cutoff_d, DA dist)
{
  O const* off       = c.offsets.as<O>();
  int32_t const* idx = c.indices.as<int32_t>();
  T const* w         = c.weights.as<T>();
  const T unreached  = std::numeric_limits<T>::max();
  const T cutoff     = cutoff_d >= (double)unreached ? unreached : (T)cutoff_d;
  // delta = warp_size * average weight / average degree  (sssp_impl.cuh:233-247)
  dbuf wsum = make_dbuf<double>(2, h.stream);
  CUDA_TRY(cudaMemsetAsync(wsum.data(), 0, 2 * sizeof(double), h.stream));
  B200_LAUNCH(h, (k_sum_weights<T>), h.sm_count * 8, kBlock, 0, w, (long long)c.nnz, wsum.as<double>());
  const double avg_w   = read_back(h, wsum.as<double>()) / (double)c.nnz;
  const double avg_deg = (double)c.nnz / (double)nv;
  const double delta_scale = h.tune.sssp_delta_scale;  // tuning knob (results do not depend on it)
  T delta = (T)(32.0 * avg_w / std::max(avg_deg, 1e-30) * delta_scale);
  if (!(delta > (T)0)) delta = (T)1;
  // Window width control (results do not depend on it; CUGRAPH_B200_SSSP_ADAPTIVE=0 keeps the fixed reference width).
  // Inside one window the near pile is relaxed Bellman-Ford style, so a vertex re-relaxes all its edges every time its
  // tentative distance improves.  With the reference's width a power-law graph puts nearly every vertex into the first
  // window (RMAT-24, uniform weights: 90 % of the edge endpoints lie within 0.05 of the source, the width is 0.27) and
  // the traversal relaxes 6 x E edges in 30 rounds.  The controller starts 64 times narrower and steers the width by
  // the number of rounds the last window took: <= 2 rounds: twice as wide (sparse stretches cost one cheap window per
  // doubling), >= 6 rounds: half as wide.
  const bool adaptive = h.tune.sssp_adaptive;
  const T delta_floor = delta / (T)4096;
  if (adaptive) delta = delta / (T)h.tune.sssp_start_div;

  dbuf stamp = make_dbuf<int32_t>(nv, h.stream);
  CUDA_TRY(cudaMemsetAsync(stamp.data(), 0, sizeof(int32_t) * nv, h.stream));
  // every queue holds a vertex at most once per round (stamps), so V entries suffice
  dbuf qa = make_dbuf<int32_t>(nv, h.stream), qb = make_dbuf<int32_t>(nv, h.stream);
  dbuf la = make_dbuf<int32_t>((size_t)nv + 1, h.stream), lb = make_dbuf<int32_t>((size_t)nv + 1, h.stream);  // queue degrees
  dbuf cnt = make_dbuf<frontier_counters_t>(1, h.stream);
  frontier_counters_t* dc = cnt.as<frontier_counters_t>();
  CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
  dbuf dmin = make_dbuf<T>(1, h.stream);
  B200_LAUNCH(h, (k_sssp_seed<O, DA>), 1, 1, 0, dist, stamp.as<int32_t>(), qa.as<int32_t>(), la.as<int32_t>(), off, source);
  frontier_counters_t* hc = reinterpret_cast<frontier_counters_t*>(h.pinned);
  T* hmin_pinned          = reinterpret_cast<T*>(reinterpret_cast<char*>(h.pinned) + 256);
  auto* hwin              = reinterpret_cast<sssp_window_t<T>*>(reinterpret_cast<char*>(h.pinned) + 320);
  dbuf dwin               = make_dbuf<sssp_window_t<T>>(1, h.stream);
  auto* hsmall            = reinterpret_cast<sssp_small_state_t*>(reinterpret_cast<char*>(h.pinned) + 384);
  dbuf dsmall             = make_dbuf<sssp_small_state_t>(1, h.stream);
  const bool small_rounds = h.tune.sssp_small_rounds;
  int tr_small            = 0;
  int32_t *near = qa.as<int32_t>(), *next_near = qb.as<int32_t>();
  int32_t *near_deg = la.as<int32_t>(), *next_near_deg = lb.as<int32_t>();  // degrees of the queue entries
  int n_near = 1, round = 1, window = 1;
  // the seed kernel wrote the source's degree next to it: read it back (the first advance needs the edge count)
  unsigned long long near_edges = (unsigned long long)(unsigned)read_back(h, near_deg);
  advance_scratch_t adv;
  adv.init(h, nv, (int64_t)c.nnz);
  T lo = (T)0, hi = delta;
  const bool trace    = h.tune.sssp_trace;
  unsigned long long tr_edges = 0;
  int tr_rounds = 0, tr_splits = 0;
  const int split_rounds = h.tune.sssp_split_rounds;
  // a split costs about one round (a kernel + a read-back): only worth it when the pending round is real work
  const unsigned long long split_min_edges = h.tune.sssp_split_min_edges;
  while (true) {
    int window_rounds = 0;
    while (n_near > 0) {
      if (small_rounds && sizeof(O) == 4 && n_near <= kSmallVerts && near_edges <= (unsigned long long)kSmallEdges) {
        // the tail of the window: rounds on the device until the queue is empty or grows past one CTA's reach
        B200_LAUNCH(h, (k_sssp_small_rounds<O, T, DA>), 1, kSmallThreads, 0, off, idx, w, dist, stamp.as<int32_t>(), near, near_deg,
                    next_near, next_near_deg, n_near, round, hi, cutoff, 256, dsmall.as<sssp_small_state_t>());
        CUDA_TRY(cudaMemcpyAsync(hsmall, dsmall.data(), sizeof(sssp_small_state_t), cudaMemcpyDeviceToHost, h.stream));
        sync(h);
        n_near     = hsmall->n;
        near_edges = hsmall->edges;
        round      = hsmall->round;
        window_rounds += hsmall->rounds_done;
        tr_rounds += hsmall->rounds_done;
        tr_edges += hsmall->relaxed;
        ++tr_small;
        if (hsmall->cur) {
          std::swap(near, next_near);
          std::swap(near_deg, next_near_deg);
        }
        continue;
      }
      ++round;
      ++tr_rounds;
      ++window_rounds;
      tr_edges += near_edges;
      CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
      sssp_relax_op<O, T, DA> op{off, w, dist, stamp.as<int32_t>(), next_near, next_near_deg, dc, hi, cutoff, round};
      advance<O>(h, adv, off, idx, near, n_near, near_edges, op, near_deg);
      CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(frontier_counters_t), cudaMemcpyDeviceToHost, h.stream));
      sync(h);
      read_counters<O>(hc, n_near, near_edges);
      std::swap(near, next_near);
      std::swap(near_deg, next_near_deg);
      // A window that is still busy after `split_rounds` rounds is too wide for this stretch of the graph (the hub core
      // of a power-law graph sits in a very narrow distance band): cut it in half now instead of after the damage.  The
      // pending near entries at or beyond the new bound are dropped from the queue (the window selection finds them again
      // when their turn comes), the rest form the next round's queue.
      if (adaptive && window_rounds >= split_rounds && n_near > 0 && near_edges >= split_min_edges &&
          near_edges * 128ull >= (unsigned long long)c.nnz) {
        const T nhi = lo + (hi - lo) * (T)0.5;
        if (nhi > lo && nhi < hi) {
          ++round;
          CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
          B200_LAUNCH(h, (k_split_near<O, T, DA>), grid_for(n_near), kBlock, 0, off, near, n_near, dist, nhi, stamp.as<int32_t>(),
                      round, next_near, next_near_deg, dc);
          CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(frontier_counters_t), cudaMemcpyDeviceToHost, h.stream));
          sync(h);
          read_counters<O>(hc, n_near, near_edges);
          std::swap(near, next_near);
          std::swap(near_deg, next_near_deg);
          hi = nhi;
          if (delta > delta_floor) delta = delta / (T)2;
          window_rounds = 0;
          ++tr_splits;
        }
      }
    }
    if (trace)
      std::fprintf(stderr, "sssp window %d hi=%g width %g: %d rounds, rounds so far %d (single-CTA calls %d), edges relaxed so far %llu, splits so far %d\n",
                   window, (double)hi, (double)delta, window_rounds, tr_rounds, tr_small, tr_edges, tr_splits);
    if (adaptive) {
      if (window_rounds <= 2) { if (delta < std::numeric_limits<T>::max() / (T)4) delta = delta * (T)2; }
      else if (window_rounds >= 6 && delta > delta_floor) delta = delta / (T)2;
    }
    // advance the window to the smallest pending distance (dense pass 1), then select its vertices (dense pass 2); the
    // bounds are computed on the device in between, the host reads them back together with the new queue's size
    const T inf = (T)INFINITY;
    hwin->lo = lo; hwin->hi = hi; hwin->any = 1;
    *hmin_pinned = inf;
    CUDA_TRY(cudaMemcpyAsync(dwin.data(), hwin, sizeof(sssp_window_t<T>), cudaMemcpyHostToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(dmin.data(), hmin_pinned, sizeof(T), cudaMemcpyHostToDevice, h.stream));
    B200_LAUNCH(h, (k_min_beyond<T, DA>), grid_for(nv, 1, h.sm_count * 64), kBlock, 0, dist, nv, hi, unreached, dmin.as<T>());
    B200_LAUNCH(h, (k_next_window<T>), 1, 1, 0, dmin.as<T>(), delta, dwin.as<sssp_window_t<T>>());
    ++round;
    ++window;
    CUDA_TRY(cudaMemsetAsync(cnt.data(), 0, sizeof(frontier_counters_t), h.stream));
    B200_LAUNCH(h, (k_select_window<O, T, DA>), grid_for(nv, kSelectPer, h.sm_count * 8), kBlock, 0, off, dist, nv, dwin.as<sssp_window_t<T>>(),
                stamp.as<int32_t>(), round, near, near_deg, dc);
    CUDA_TRY(cudaMemcpyAsync(hc, cnt.data(), sizeof(frontier_counters_t), cudaMemcpyDeviceToHost, h.stream));
    CUDA_TRY(cudaMemcpyAsync(hwin, dwin.data(), sizeof(sssp_window_t<T>), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    if (!hwin->any) break;  // nothing pending: done
    lo = hwin->lo;
    hi = hwin->hi;
    read_counters<O>(hc, n_near, near_edges);
  }
  check_last("sssp");
}

template <typename O, typename T>
void run_sssp(handle_impl const& h, csx_t const& c, int32_t nv, int32_t source, double cutoff_d, T* dist, int32_t* pred)
{
  O const* off       = c.offsets.as<O>();
  int32_t const* idx = c.indices.as<int32_t>();
  T const* w         = c.weights.as<T>();
  const T unreached  = std::numeric_limits<T>::max();
  if (pred) B200_LAUNCH(h, (k_fill<int32_t>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, pred, (int64_t)nv, -1);
  if (c.nnz == 0) {
    B200_LAUNCH(h, (k_fill<T>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, dist, (int64_t)nv, unreached);
    B200_LAUNCH(h, (k_fill<T>), 1, 1, 0, dist + source, (int64_t)1, (T)0);
    return;
  }
  if (pred && std::is_same<T, float>::value) {  // float with predecessors: (distance, predecessor) in one word
    dbuf packed = make_dbuf<unsigned long long>(nv, h.stream);
    B200_LAUNCH(h, (k_fill<unsigned long long>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, packed.as<unsigned long long>(),
                (int64_t)nv, dist_packed::pack(0x7f7fffffu, -1));
    sssp_windows<O, float, dist_packed>(h, c, nv, source, cutoff_d, dist_packed{packed.as<unsigned long long>()});
    B200_LAUNCH(h, k_unpack_dist, grid_for(nv), kBlock, 0, packed.as<unsigned long long>(), nv, reinterpret_cast<float*>(dist), pred);
    check_last("sssp");
    return;
  }
  B200_LAUNCH(h, (k_fill<T>), grid_for(nv, 1, h.sm_count * 32), kBlock, 0, dist, (int64_t)nv, unreached);
  sssp_windows<O, T, dist_plain<T>>(h, c, nv, source, cutoff_d, dist_plain<T>{dist});
  if (pred) {
    if (sizeof(O) == 4) {
      sssp_pred_op<T> pop{w, dist, pred, source, unreached};
      advance_all_edges(h, (int32_t const*)off, idx, nv, (long long)c.nnz, pop);
    } else {
      B200_LAUNCH(h, (k_sssp_pred<O, T>), h.sm_count * 16, kBlock, 0, off, idx, w, dist, nv, source, unreached, pred);
    }
    // vertices whose tight edges all come from their own distance level (zero-weight / absorbed edges): rare
    dbuf flags = make_dbuf<int>(2, h.stream);
    int* hflags = reinterpret_cast<int*>(reinterpret_cast<char*>(h.pinned) + 512);
    CUDA_TRY(cudaMemsetAsync(flags.data(), 0, 2 * sizeof(int), h.stream));
    B200_LAUNCH(h, (k_sssp_count_orphans<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, dist, pred, nv, source, unreached,
                flags.as<int>());
    CUDA_TRY(cudaMemcpyAsync(hflags, flags.data(), 2 * sizeof(int), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    for (int pass = 0; hflags[0] > 0 && pass < nv; ++pass) {
      CUDA_TRY(cudaMemsetAsync(flags.as<int>() + 1, 0, sizeof(int), h.stream));
      if (sizeof(O) == 4) {
        sssp_tie_op<T> top{w, dist, pred, source, unreached, flags.as<int>() + 1};
        advance_all_edges(h, (int32_t const*)off, idx, nv, (long long)c.nnz, top);
      } else {
        B200_LAUNCH(h, (k_sssp_pred_ties<O, T>), h.sm_count * 16, kBlock, 0, off, idx, w, dist, nv, source, unreached, pred,
                    flags.as<int>() + 1);
      }
      CUDA_TRY(cudaMemcpyAsync(hflags, flags.data(), 2 * sizeof(int), cudaMemcpyDeviceToHost, h.stream));
      sync(h);
      if (hflags[1] == 0) break;
    }
  }
  check_last("sssp");
}

device_array_impl* make_array(dbuf&& b, size_t n, cugraph_data_type_id_t t) { return new device_array_impl{std::move(b), n, t}; }

// internal predecessors (int32, internal ids) -> reported order, external ids, graph's vertex dtype, into ext_out (V elements)
void predecessors_to_ext(handle_impl const& h, graph_impl const& g, int32_t const* pred_int, void* ext_out)
{
  dbuf ordered = to_reported_order(h, g, pred_int, sizeof(int32_t));
  int_to_ext(h, g, ordered.as<int32_t>(), (size_t)g.n_vertices, ext_out);
}

device_array_impl* finish_predecessors(handle_impl const& h, graph_impl const& g, int32_t const* pred_int)
{
  dbuf ext((size_t)g.n_vertices * dtype_size(g.vertex_type), h.stream);
  predecessors_to_ext(h, g, pred_int, ext.data());
  return make_array(std::move(ext), (size_t)g.n_vertices, g.vertex_type);
}

}  // namespace
}  // namespace b200

using namespace b200;

namespace b200 {
namespace {

// ---- extract_paths (reference cpp/src/traversal/extract_bfs_paths_impl.cuh:129-238, cpp/src/c_api/extract_paths.cpp): walk the
// predecessor chain of every destination back to its source.  Row i of the result holds the path source ... destination_i in
// columns 0 .. distance(destination_i), the rest is the invalid vertex (-1); the row length is 1 + the largest distance of
// a destination that has a predecessor.  One thread per destination (paths are as short as the BFS is deep); the
// reference does one gather round per path position over all destinations.
template <typename D>
__global__ void k_scatter_to_internal(int32_t const* __restrict__ int_of_pos, D const* __restrict__ dist_pos,
                                      int32_t const* __restrict__ pred_int_pos, int32_t n, long long* __restrict__ dist_int,
                                      int32_t* __restrict__ pred_int)
{
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int v = int_of_pos[p];
    if (v < 0) continue;
    dist_int[v] = (long long)dist_pos[p];
    pred_int[v] = pred_int_pos[p];
  }
}

__global__ void k_paths_max_len(int32_t const* __restrict__ dest, int32_t n_dest, long long const* __restrict__ dist,
                                int32_t const* __restrict__ pred, int32_t nv, long long unreachable, long long* __restrict__ out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_dest; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = dest[i];
    if (v < 0 || v >= nv || pred[v] < 0 || dist[v] >= unreachable) continue;
    atomicMax(reinterpret_cast<unsigned long long*>(out), (unsigned long long)dist[v]);
  }
}

__global__ void k_paths_walk(int32_t const* __restrict__ dest, int32_t n_dest, long long const* __restrict__ dist,
                             int32_t const* __restrict__ pred, int32_t nv, long long unreachable, long long len,
                             int32_t* __restrict__ paths)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_dest; i += (int64_t)gridDim.x * blockDim.x) {
    int v = dest[i];
    if (v < 0 || v >= nv) continue;
    long long d = dist[v];
    if (d >= unreachable || d >= len) continue;  // not reached: the row stays invalid
    for (; d >= 0 && v >= 0; --d) {
      paths[i * len + d] = v;
      v = pred[v];
    }
  }
}

}  // namespace
}  // namespace b200

extern "C" {

cugraph_type_erased_device_array_view_t* cugraph_paths_result_get_vertices(cugraph_paths_result_t* r)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<paths_result_impl*>(r)->vertices->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_paths_result_get_distances(cugraph_paths_result_t* r)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<paths_result_impl*>(r)->distances->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_paths_result_get_predecessors(cugraph_paths_result_t* r)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<paths_result_impl*>(r)->predecessors->new_view());
}
void cugraph_paths_result_free(cugraph_paths_result_t* r)
{
  if (!r) return;
  auto* p = reinterpret_cast<paths_result_impl*>(r);
  delete p->vertices;
  delete p->distances;
  delete p->predecessors;
  delete p;
}

cugraph_error_code_t cugraph_bfs(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                 cugraph_type_erased_device_array_view_t* sources, bool_t direction_optimizing,
                                 size_t depth_limit, bool_t compute_predecessors, bool_t do_expensive_check,
                                 cugraph_paths_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(sources != nullptr, CUGRAPH_INVALID_INPUT, "sources is NULL");
    auto const* s = V(sources);
    B200_EXPECTS(s->type == g->vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and sources must match");
    B200_EXPECTS(g->is_symmetric || direction_optimizing == FALSE, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: input graph should be symmetric for direction optimizing BFS.");
    const int32_t nv = g->n_vertices;
    dbuf src_int     = make_dbuf<int32_t>(std::max<size_t>(s->size, 1), h.stream);
    ext_to_int(h, *g, s->data, s->size, src_int.as<int32_t>());
    if (s->size > 0) {
      std::vector<int32_t> hs(s->size);
      CUDA_TRY(cudaMemcpyAsync(hs.data(), src_int.data(), sizeof(int32_t) * s->size, cudaMemcpyDeviceToHost, h.stream));
      sync(h);
      for (auto v : hs) B200_EXPECTS(v >= 0, CUGRAPH_INVALID_INPUT, "Found invalid vertex in the input sources");
    }
    dbuf dist = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    dbuf pred;
    if (compute_predecessors) pred = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    const int dl = (int)std::min<size_t>(depth_limit, (size_t)INT_MAX);
    if (nv > 0) {
      csx_t const& c = push_view(h, *g);
      if (c.offs64)
        run_bfs<int64_t>(h, c, nv, src_int.as<int32_t>(), (int)s->size, direction_optimizing == TRUE, dl,
                         dist.as<int32_t>(), pred.as<int32_t>());
      else
        run_bfs<int32_t>(h, c, nv, src_int.as<int32_t>(), (int)s->size, direction_optimizing == TRUE, dl,
                         dist.as<int32_t>(), pred.as<int32_t>());
    }
    auto res      = std::make_unique<paths_result_impl>();
    res->vertices = make_array(reported_vertices(h, *g), (size_t)nv, g->vertex_type);
    dbuf dord     = to_reported_order(h, *g, dist.data(), sizeof(int32_t));
    if (g->vertex_type == INT64) {
      dbuf wide = make_dbuf<int64_t>(std::max(nv, 1), h.stream);
      B200_LAUNCH(h, k_widen_dist, grid_for(nv), kBlock, 0, dord.as<int32_t>(), nv, wide.as<int64_t>());
      res->distances = make_array(std::move(wide), (size_t)nv, INT64);
    } else {
      res->distances = make_array(std::move(dord), (size_t)nv, INT32);
    }
    if (compute_predecessors) res->predecessors = finish_predecessors(h, *g, pred.as<int32_t>());
    else res->predecessors = make_array(dbuf(0, h.stream), 0, g->vertex_type);
    sync(h);
    *result = reinterpret_cast<cugraph_paths_result_t*>(res.release());
  });
}

cugraph_error_code_t cugraph_b200_multi_source_bfs(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                   const cugraph_type_erased_device_array_view_t* sources, size_t depth_limit,
                                                   bool_t compute_predecessors, cugraph_paths_result_t** result,
                                                   cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(sources != nullptr, CUGRAPH_INVALID_INPUT, "sources is NULL");
    auto const* s = V(sources);
    B200_EXPECTS(s->type == g->vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and sources must match");
    const int32_t nv = g->n_vertices;
    const size_t n   = s->size;
    dbuf src_int     = make_dbuf<int32_t>(std::max<size_t>(n, 1), h.stream);
    ext_to_int(h, *g, s->data, n, src_int.as<int32_t>());
    if (n > 0) {
      std::vector<int32_t> hs(n);
      CUDA_TRY(cudaMemcpyAsync(hs.data(), src_int.data(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, h.stream));
      sync(h);
      for (auto v : hs) B200_EXPECTS(v >= 0, CUGRAPH_INVALID_INPUT, "Found invalid vertex in the input sources");
    }
    // source-major results: row k (source k) starts at entry k * nv, 64-bit offsets (n * nv passes 2^31 early)
    const size_t es    = dtype_size(g->vertex_type);
    const size_t cells = n * (size_t)nv;
    dbuf dist_out(cells * es, h.stream), pred_out(compute_predecessors ? cells * es : 0, h.stream);
    const int dl = (int)std::min<size_t>(depth_limit, (size_t)INT_MAX);
    if (cells > 0) {
      const int nb_max = (int)std::min<size_t>(n, 64);
      // one batch's internal rows; each row goes to reported order and external ids straight into the result
      dbuf dist_b = make_dbuf<int32_t>((size_t)nb_max * nv, h.stream), pred_b;
      if (compute_predecessors) pred_b = make_dbuf<int32_t>((size_t)nb_max * nv, h.stream);
      dbuf wide_tmp;
      if (g->vertex_type == INT64) wide_tmp = make_dbuf<int32_t>(nv, h.stream);
      for (size_t b0 = 0; b0 < n; b0 += 64) {
        const int nb = (int)std::min<size_t>(n - b0, 64);
        multi_source_bfs_batch(h, *g, src_int.as<int32_t>() + b0, nb, dl, dist_b.as<int32_t>(), pred_b.as<int32_t>(),
                               (int)(b0 / 64), nullptr);
        for (int j = 0; j < nb; ++j) {
          int32_t const* row = dist_b.as<int32_t>() + (size_t)j * nv;
          char* out          = dist_out.as<char>() + (b0 + j) * (size_t)nv * es;
          if (g->vertex_type == INT64) {
            to_reported_order_into(h, *g, row, sizeof(int32_t), wide_tmp.data());
            B200_LAUNCH(h, k_widen_dist, grid_for(nv), kBlock, 0, wide_tmp.as<int32_t>(), nv, (int64_t*)out);
          } else {
            to_reported_order_into(h, *g, row, sizeof(int32_t), out);
          }
          if (compute_predecessors)
            predecessors_to_ext(h, *g, pred_b.as<int32_t>() + (size_t)j * nv, pred_out.as<char>() + (b0 + j) * (size_t)nv * es);
        }
      }
      check_last("multi_source_bfs");
    }
    auto res          = std::make_unique<paths_result_impl>();
    res->vertices     = make_array(reported_vertices(h, *g), (size_t)nv, g->vertex_type);
    res->distances    = make_array(std::move(dist_out), cells, g->vertex_type);
    res->predecessors = make_array(std::move(pred_out), compute_predecessors ? cells : 0, g->vertex_type);
    sync(h);
    *result = reinterpret_cast<cugraph_paths_result_t*>(res.release());
  });
}

cugraph_error_code_t cugraph_sssp(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, size_t source,
                                  double cutoff, bool_t compute_predecessors, bool_t do_expensive_check,
                                  cugraph_paths_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(g->weighted, CUGRAPH_INVALID_INPUT, "SSSP requires a weighted graph");
    const int32_t nv = g->n_vertices;
    // external source id -> internal
    dbuf src_ext(8, h.stream), src_int = make_dbuf<int32_t>(1, h.stream);
    int64_t s64 = (int64_t)source;
    int32_t s32 = (int32_t)source;
    if (g->vertex_type == INT64) CUDA_TRY(cudaMemcpyAsync(src_ext.data(), &s64, 8, cudaMemcpyHostToDevice, h.stream));
    else CUDA_TRY(cudaMemcpyAsync(src_ext.data(), &s32, 4, cudaMemcpyHostToDevice, h.stream));
    ext_to_int(h, *g, src_ext.data(), 1, src_int.as<int32_t>());
    const int32_t src = read_back(h, src_int.as<int32_t>());
    B200_EXPECTS(src >= 0 && (g->vertex_type == INT64 || source <= (size_t)INT_MAX), CUGRAPH_INVALID_INPUT,
                 "Invalid input argument: source vertex is invalid.");
    csx_t const& c = push_view(h, *g);
    auto res       = std::make_unique<paths_result_impl>();
    res->vertices  = make_array(reported_vertices(h, *g), (size_t)nv, g->vertex_type);
    dbuf pred;
    if (compute_predecessors) pred = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    if (g->weight_type == FLOAT32) {
      dbuf dist = make_dbuf<float>(std::max(nv, 1), h.stream);
      if (c.offs64) run_sssp<int64_t, float>(h, c, nv, src, cutoff, dist.as<float>(), pred.as<int32_t>());
      else run_sssp<int32_t, float>(h, c, nv, src, cutoff, dist.as<float>(), pred.as<int32_t>());
      res->distances = make_array(to_reported_order(h, *g, dist.data(), sizeof(float)), (size_t)nv, FLOAT32);
    } else {
      dbuf dist = make_dbuf<double>(std::max(nv, 1), h.stream);
      if (c.offs64) run_sssp<int64_t, double>(h, c, nv, src, cutoff, dist.as<double>(), pred.as<int32_t>());
      else run_sssp<int32_t, double>(h, c, nv, src, cutoff, dist.as<double>(), pred.as<int32_t>());
      res->distances = make_array(to_reported_order(h, *g, dist.data(), sizeof(double)), (size_t)nv, FLOAT64);
    }
    if (compute_predecessors) res->predecessors = finish_predecessors(h, *g, pred.as<int32_t>());
    else res->predecessors = make_array(dbuf(0, h.stream), 0, g->vertex_type);
    sync(h);
    *result = reinterpret_cast<cugraph_paths_result_t*>(res.release());
  });
}


struct extract_paths_result_impl {
  size_t max_path_length{0};
  device_array_impl* paths{nullptr};
};

cugraph_error_code_t cugraph_extract_paths(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                           const cugraph_type_erased_device_array_view_t* sources,
                                           const cugraph_paths_result_t* paths_result,
                                           const cugraph_type_erased_device_array_view_t* destinations,
                                           cugraph_extract_paths_result_t** result, cugraph_error_t** error)
{
  (void)sources;  // the reference takes them and does not read them either (c_api/extract_paths.cpp:60-130)
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(paths_result != nullptr && destinations != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* pr = reinterpret_cast<paths_result_impl const*>(paths_result);
    auto const* dv = V(destinations);
    B200_EXPECTS(dv->type == g->vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and destinations must match");
    B200_EXPECTS(pr->distances && pr->vertices, CUGRAPH_INVALID_INPUT, "Invalid input argument: distances cannot be null");
    B200_EXPECTS(pr->predecessors && pr->predecessors->size == pr->vertices->size, CUGRAPH_INVALID_INPUT,
                 "Invalid input argument: predecessors cannot be null");
    B200_EXPECTS(pr->distances->type == INT32 || pr->distances->type == INT64, CUGRAPH_INVALID_INPUT,
                 "extract_paths expects the integer distances of a BFS result");
    const int32_t nv = g->n_vertices;
    B200_EXPECTS((size_t)nv == pr->vertices->size, CUGRAPH_INVALID_INPUT, "the paths result does not belong to this graph");
    const size_t nd = dv->size;
    // result positions -> internal ids; distances / predecessors re-indexed by internal id
    dbuf int_of_pos = make_dbuf<int32_t>(std::max(nv, 1), h.stream), pred_pos = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    ext_to_int(h, *g, pr->vertices->buf.data(), (size_t)nv, int_of_pos.as<int32_t>());
    ext_to_int(h, *g, pr->predecessors->buf.data(), (size_t)nv, pred_pos.as<int32_t>());
    dbuf dist_int = make_dbuf<long long>(std::max(nv, 1), h.stream), pred_int = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    const long long unreachable = pr->distances->type == INT64 ? (long long)INT64_MAX : (long long)INT32_MAX;
    if (nv > 0) {
      if (pr->distances->type == INT64)
        B200_LAUNCH(h, (k_scatter_to_internal<int64_t>), grid_for(nv), kBlock, 0, int_of_pos.as<int32_t>(),
                    pr->distances->buf.as<int64_t>(), pred_pos.as<int32_t>(), nv, dist_int.as<long long>(), pred_int.as<int32_t>());
      else
        B200_LAUNCH(h, (k_scatter_to_internal<int32_t>), grid_for(nv), kBlock, 0, int_of_pos.as<int32_t>(),
                    pr->distances->buf.as<int32_t>(), pred_pos.as<int32_t>(), nv, dist_int.as<long long>(), pred_int.as<int32_t>());
    }
    dbuf dest_int = make_dbuf<int32_t>(std::max<size_t>(nd, 1), h.stream);
    ext_to_int(h, *g, dv->data, nd, dest_int.as<int32_t>());
    dbuf d_max = make_dbuf<long long>(1, h.stream);
    CUDA_TRY(cudaMemsetAsync(d_max.data(), 0, sizeof(long long), h.stream));
    if (nd > 0)
      B200_LAUNCH(h, k_paths_max_len, grid_for((int64_t)nd), kBlock, 0, dest_int.as<int32_t>(), (int32_t)nd, dist_int.as<long long>(),
                  pred_int.as<int32_t>(), nv, unreachable, d_max.as<long long>());
    const long long len = read_back(h, d_max.as<long long>()) + 1;
    const size_t total  = nd * (size_t)len;
    dbuf paths_int      = make_dbuf<int32_t>(std::max<size_t>(total, 1), h.stream);
    if (total > 0) {
      CUDA_TRY(cudaMemsetAsync(paths_int.data(), 0xff, sizeof(int32_t) * total, h.stream));  // -1 = invalid vertex
      B200_LAUNCH(h, k_paths_walk, grid_for((int64_t)nd), kBlock, 0, dest_int.as<int32_t>(), (int32_t)nd, dist_int.as<long long>(),
                  pred_int.as<int32_t>(), nv, unreachable, len, paths_int.as<int32_t>());
    }
    dbuf paths_ext(std::max<size_t>(total, 1) * dtype_size(g->vertex_type), h.stream);
    int_to_ext(h, *g, paths_int.as<int32_t>(), total, paths_ext.data());
    check_last("extract_paths");
    auto res             = std::make_unique<extract_paths_result_impl>();
    res->max_path_length = (size_t)len;
    res->paths           = make_array(std::move(paths_ext), total, g->vertex_type);
    sync(h);
    *result = reinterpret_cast<cugraph_extract_paths_result_t*>(res.release());
  });
}

size_t cugraph_extract_paths_result_get_max_path_length(cugraph_extract_paths_result_t* result)
{
  return result ? reinterpret_cast<extract_paths_result_impl*>(result)->max_path_length : 0;
}

cugraph_type_erased_device_array_view_t* cugraph_extract_paths_result_get_paths(cugraph_extract_paths_result_t* result)
{
  if (!result) return nullptr;
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<extract_paths_result_impl*>(result)->paths->new_view());
}

void cugraph_extract_paths_result_free(cugraph_extract_paths_result_t* result)
{
  if (!result) return;
  auto* r = reinterpret_cast<extract_paths_result_impl*>(result);
  delete r->paths;
  delete r;
}

}  // extern "C"
