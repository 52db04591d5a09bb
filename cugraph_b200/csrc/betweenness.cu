// Vertex and edge betweenness centrality (reference cpp/src/centrality/betweenness_centrality_impl.cuh, C API
// cpp/src/c_api/betweenness_centrality.cpp): Brandes' algorithm over batches of up to 64 sources, on the levels of the
// multi-source BFS (traverse.cu, multi_source_bfs_batch).  Paths are counted by hops; edge weights are never read.
//
// Forward.  The BFS hands every level d to bc_levels (an ms_level_sink), which keeps the level as a queue of (vertex, word)
// entries: the vertices that gained bits at d and those bits, i.e. the (source, vertex) pairs at distance d.  No distance
// array exists.  Right after level d is kept, the sigma pull gives each of its pairs its path count:
//   sigma_s(v) = sum of sigma_s(u) over the in-edges u -> v whose u holds bit s at level d - 1,
// read from a V-sized word array into which level d - 1 was scattered.  Every in-edge is read (every predecessor counts).
// Backward.  Levels from the deepest to 0; level d + 1 is scattered into the word array first, then for every pair (s, u)
// at level d, over u's out-edges u -> v whose v holds bit s at level d + 1:
//   c = sigma_s(u) / sigma_s(v) * (1 + delta_s(v)),   delta_s(u) = sum of c,   ebc[u -> v] += sum of c over the sources,
// and bc[u] += sum of delta_s(u) over the sources (level 0 is the sources themselves and adds nothing, as in Brandes).
// One warp owns one queue entry: lanes over the sources (source j on lane j and lane j - 32), each in-/out-edge read once
// per warp and its word broadcast.  The warp sums its lanes with a fixed shuffle tree and is the only writer of bc[u] and of
// the ebc entries of u's out-edges at that level, so results are bit-identical from run to run without atomics.
//
// sigma and delta are fp64 [V][ld] (ld = the batch width): the reference keeps sigma in edge_t, which overflows int32 once
// a vertex has more than 2^31 shortest paths from one source; fp64 keeps a relative error near 2^-53 per addition instead.
#include "advance.cuh"
#include "graph.cuh"
#include "staging.cuh"

#include <cugraph_c/algorithms.h>
#include <cugraph_c/random.h>
#include <cugraph_c/sampling_algorithms.h>

#include <climits>
#include <cmath>
#include <memory>
#include <vector>

namespace b200 {
namespace {

using u64 = unsigned long long;

// lw[i] = words[q[i]]
__global__ void k_bc_gather(int32_t const* __restrict__ q, int n, u64 const* __restrict__ words, u64* __restrict__ lw)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) lw[i] = words[q[i]];
}

// words[q[i]] = lw[i], or 0 with lw == nullptr
__global__ void k_bc_scatter(int32_t const* __restrict__ q, int n, u64 const* __restrict__ lw, u64* __restrict__ words)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    words[q[i]] = lw ? lw[i] : 0ull;
}

// level 0: sigma_j(source j) = 1
__global__ void k_bc_sigma_seed(int32_t const* __restrict__ q, int n, u64 const* __restrict__ lw, double* __restrict__ sigma, int ld)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    for (u64 b = lw[i]; b; b &= b - 1) sigma[(int64_t)q[i] * ld + (__ffsll((long long)b) - 1)] = 1.0;
  }
}

// sigma of the pairs of level d (entries q, lw) from level d - 1 (prev: V words); in-edges from a vertex-indexed in-edge view
template <typename OI>
__global__ void __launch_bounds__(kBlock)
k_bc_sigma_pull(OI const* __restrict__ in_off, int32_t const* __restrict__ in_idx, int32_t const* __restrict__ q,
                u64 const* __restrict__ lw, int n, u64 const* __restrict__ prev, double* __restrict__ sigma, int ld)
{
  const int lane     = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nw   = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nw) {
    const int v   = q[i];
    const u64 w   = lw[i];
    const bool b0 = (w >> lane) & 1ull, b1 = lane + 32 < ld && ((w >> (lane + 32)) & 1ull);
    double a0 = 0.0, a1 = 0.0;
    const int64_t end = (int64_t)in_off[v + 1];
    for (int64_t e0 = (int64_t)in_off[v]; e0 < end; e0 += 32) {
      const int64_t e = e0 + lane;
      const int u     = e < end ? in_idx[e] : 0;
      const u64 pw    = e < end ? prev[u] & w : 0ull;
      for (unsigned live = __ballot_sync(0xffffffffu, pw != 0ull); live; live &= live - 1) {
        const int k   = __ffs((int)live) - 1;
        const int uk  = __shfl_sync(0xffffffffu, u, k);
        const u64 pk  = __shfl_sync(0xffffffffu, pw, k);
        if ((pk >> lane) & 1ull) a0 += sigma[(int64_t)uk * ld + lane];
        if (lane + 32 < ld && ((pk >> (lane + 32)) & 1ull)) a1 += sigma[(int64_t)uk * ld + lane + 32];
      }
    }
    if (b0) sigma[(int64_t)v * ld + lane] = a0;
    if (b1) sigma[(int64_t)v * ld + lane + 32] = a1;
  }
}

// delta of the pairs of level d (entries q, lw) from level d + 1 (next: V words), bc and ebc (nullable) accumulated.
// level 0 (sources = true) adds nothing to bc but, with endpoints, the source's reached - 1 = delta_s(s) (an integer).
// With endpoints every other pair adds 1.
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_bc_backward(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ q, u64 const* __restrict__ lw,
              int n, u64 const* __restrict__ next, double const* __restrict__ sigma, double* __restrict__ delta, int ld,
              double* __restrict__ bc, double* __restrict__ ebc, int sources, int endpoints)
{
  const int lane     = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nw   = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nw) {
    const int u     = q[i];
    const u64 w     = lw[i];
    const bool b0   = (w >> lane) & 1ull, b1 = lane + 32 < ld && ((w >> (lane + 32)) & 1ull);
    const double s0 = b0 ? sigma[(int64_t)u * ld + lane] : 0.0;
    const double s1 = b1 ? sigma[(int64_t)u * ld + lane + 32] : 0.0;
    double a0 = 0.0, a1 = 0.0;
    const int64_t end = (int64_t)off[u + 1];
    for (int64_t e0 = (int64_t)off[u]; e0 < end; e0 += 32) {
      const int64_t e = e0 + lane;
      const int v     = e < end ? idx[e] : 0;
      const u64 nx    = e < end ? next[v] & w : 0ull;
      for (unsigned live = __ballot_sync(0xffffffffu, nx != 0ull); live; live &= live - 1) {
        const int k  = __ffs((int)live) - 1;
        const int vk = __shfl_sync(0xffffffffu, v, k);
        const u64 nk = __shfl_sync(0xffffffffu, nx, k);
        double c     = 0.0;
        if ((nk >> lane) & 1ull) {
          const int64_t p = (int64_t)vk * ld + lane;
          const double t  = s0 / sigma[p] * (1.0 + delta[p]);
          a0 += t;
          c += t;
        }
        if (lane + 32 < ld && ((nk >> (lane + 32)) & 1ull)) {
          const int64_t p = (int64_t)vk * ld + lane + 32;
          const double t  = s1 / sigma[p] * (1.0 + delta[p]);
          a1 += t;
          c += t;
        }
        if (ebc) {
          c = warp_sum(c);
          if (lane == 0) ebc[e0 + k] += c;
        }
      }
    }
    if (b0) delta[(int64_t)u * ld + lane] = a0;
    if (b1) delta[(int64_t)u * ld + lane + 32] = a1;
    double mine;
    if (sources) mine = endpoints ? rint(a0) + rint(a1) : 0.0;
    else mine = a0 + a1 + (endpoints ? (double)b0 + (double)b1 : 0.0);
    mine = warp_sum(mine);
    if (lane == 0) bc[u] += mine;
  }
}

template <typename T>
__global__ void k_bc_finish(double const* __restrict__ bc, int nv, uint8_t const* __restrict__ is_source, int scaled, T s_non,
                            T s_src, T* __restrict__ out)
{
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < nv; v += (int64_t)gridDim.x * blockDim.x) {
    const T x = (T)bc[v];
    out[v]    = scaled ? x / (is_source[v] ? s_src : s_non) : x;
  }
}

template <typename T>
__global__ void k_ebc_finish(double const* __restrict__ ebc, int64_t m, int scaled, T sf, T* __restrict__ out)
{
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    const T x = (T)ebc[e];
    out[e]    = scaled ? x / sf : x;
  }
}

__global__ void k_mark_sources(int32_t const* __restrict__ s, int64_t n, uint8_t* __restrict__ is_source)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) is_source[s[i]] = 1;
}

// keys of the vertices by rank: mix64(seed ^ (counter + rank)), a bijection of the rank, so no two keys tie
__global__ void k_random_keys(u64* __restrict__ keys, int32_t* __restrict__ ranks, int nv, u64 seed, u64 counter)
{
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nv; r += (int64_t)gridDim.x * blockDim.x) {
    u64 z = seed ^ (counter + (u64)r);
    z += 0x9e3779b97f4a7c15ull;
    z        = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z        = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    keys[r]  = z ^ (z >> 31);
    ranks[r] = (int32_t)r;
  }
}

__global__ void k_rank_to_int(int32_t* __restrict__ a, int64_t n, int32_t const* __restrict__ int_of_rank)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = int_of_rank[a[i]];
}

// ---- forward levels: the per-level queues of one batch and the sigma pull (see the top of the file)
struct bc_levels final : ms_level_sink {
  handle_impl const& h;
  csx_t const& in;   // vertex-indexed in-edges
  int32_t nv;
  double* sigma;
  int ld;
  dbuf q, w;                   // queue entries of every level of the batch, level after level
  size_t cap{0};
  std::vector<size_t> first{0};  // level d: entries [first[d], first[d + 1])
  dbuf words;                  // V words: the last level kept (forward), level d + 1 (backward); zero elsewhere
  dbuf counter = make_dbuf<int>(1, h.stream);
  bool timed;
  cudaEvent_t e0{}, e1{};
  double pull_ms{0.0};

  bc_levels(handle_impl const& hh, csx_t const& c, int32_t n, double* s, int l)
      : h(hh), in(c), nv(n), sigma(s), ld(l), words(make_dbuf<u64>(std::max(n, 1), hh.stream)), timed(hh.tune.bc_trace)
  {
    CUDA_TRY(cudaMemsetAsync(words.data(), 0, sizeof(u64) * std::max(nv, 1), h.stream));
    if (timed) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
    }
  }
  ~bc_levels()
  {
    if (timed) {
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
    }
  }
  int levels() const { return (int)first.size() - 1; }
  int32_t* lq(int d) const { return q.as<int32_t>() + first[d]; }
  u64* lw(int d) const { return w.as<u64>() + first[d]; }
  int count(int d) const { return (int)(first[d + 1] - first[d]); }
  void reset() { first.assign(1, 0); }
  // level d's words into `words`, or zeros there
  void scatter(int d, bool set) const
  {
    B200_LAUNCH(h, k_bc_scatter, grid_for(count(d), 1, h.sm_count * 8), kBlock, 0, lq(d), count(d), set ? lw(d) : nullptr,
                words.as<u64>());
  }
  void level(int d, u64 const* bfs_words, int32_t const* queue, int n) override
  {
    const size_t used = first.back();
    if (used + n > cap) {  // grow the queue storage (the BFS reads every level's size back, so it is known here)
      const size_t nc = std::max(used + n, 2 * cap);
      dbuf nq = make_dbuf<int32_t>(nc, h.stream), nw = make_dbuf<u64>(nc, h.stream);
      if (used) {
        CUDA_TRY(cudaMemcpyAsync(nq.data(), q.data(), sizeof(int32_t) * used, cudaMemcpyDeviceToDevice, h.stream));
        CUDA_TRY(cudaMemcpyAsync(nw.data(), w.data(), sizeof(u64) * used, cudaMemcpyDeviceToDevice, h.stream));
      }
      q = std::move(nq), w = std::move(nw), cap = nc;
    }
    int32_t* dq = q.as<int32_t>() + used;
    u64* dw     = w.as<u64>() + used;
    if (queue) {
      CUDA_TRY(cudaMemcpyAsync(dq, queue, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, h.stream));
    } else {
      CUDA_TRY(cudaMemsetAsync(counter.data(), 0, sizeof(int), h.stream));
      B200_LAUNCH(h, k_ms_words_to_queue, grid_for(nv, 1, h.sm_count * 16), kBlock, 0, bfs_words, nv, dq, counter.as<int>());
    }
    B200_LAUNCH(h, k_bc_gather, grid_for(n, 1, h.sm_count * 8), kBlock, 0, dq, n, bfs_words, dw);
    first.push_back(used + n);
    if (timed) cudaEventRecord(e0, h.stream);
    if (d == 0) {
      B200_LAUNCH(h, k_bc_sigma_seed, grid_for(n, 1, h.sm_count * 8), kBlock, 0, dq, n, dw, sigma, ld);
    } else {
      const int grid = grid_for((int64_t)n * 32, 1, h.sm_count * 16);
      if (in.offs64)
        B200_LAUNCH(h, (k_bc_sigma_pull<int64_t>), grid, kBlock, 0, in.offsets.as<int64_t>(), in.indices.as<int32_t>(), dq, dw, n,
                    words.as<u64>(), sigma, ld);
      else
        B200_LAUNCH(h, (k_bc_sigma_pull<int32_t>), grid, kBlock, 0, in.offsets.as<int32_t>(), in.indices.as<int32_t>(), dq, dw, n,
                    words.as<u64>(), sigma, ld);
      scatter(d - 1, false);
    }
    if (timed) {
      cudaEventRecord(e1, h.stream);
      cudaEventSynchronize(e1);
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      pull_ms += ms;
    }
    scatter(d, true);
  }
};

// Sources per batch: sigma and delta take 16 * nb bytes per vertex; nb is the largest width <= 64 (and <= the number of
// sources) whose sigma + delta fit half of the free device memory, at least 1.  The level queues grow as the levels come.
int batch_width(int32_t nv, size_t n_sources)
{
  size_t free_b = 0, total_b = 0;
  CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
  const size_t fit = free_b / 2 / (16 * (size_t)std::max(nv, 1));
  return (int)std::max<size_t>(1, std::min<size_t>({64, n_sources, fit}));
}

// Brandes over every batch: bc (V, internal order) and, if non-null, ebc (push view edge order) accumulated in fp64
void brandes(handle_impl const& h, graph_impl& g, int32_t const* sources, size_t n, bool endpoints, double* bc, double* ebc)
{
  const int32_t nv = g.n_vertices;
  if (n == 0 || nv == 0) return;
  csx_t const& out = push_view(h, g);
  csx_t const& in  = in_view(h, g);
  const int ld     = batch_width(nv, n);
  dbuf sigma = make_dbuf<double>((size_t)ld * nv, h.stream), delta = make_dbuf<double>((size_t)ld * nv, h.stream);
  bc_levels lv(h, in, nv, sigma.as<double>(), ld);
  const bool trace = h.tune.bc_trace;
  cudaEvent_t t0{}, t1{}, t2{};
  if (trace) {
    cudaEventCreate(&t0);
    cudaEventCreate(&t1);
    cudaEventCreate(&t2);
  }
  for (size_t b0 = 0; b0 < n; b0 += (size_t)ld) {
    const int nb = (int)std::min<size_t>(n - b0, (size_t)ld);
    lv.reset();
    lv.pull_ms = 0.0;
    if (trace) cudaEventRecord(t0, h.stream);
    multi_source_bfs_batch(h, g, sources + b0, nb, INT_MAX, nullptr, nullptr, (int)(b0 / ld), &lv);
    if (trace) cudaEventRecord(t1, h.stream);
    const int D = lv.levels() - 1;  // deepest level; the words array holds it
    lv.scatter(D, false);
    for (int d = D; d >= 0; --d) {
      if (d + 2 <= D) lv.scatter(d + 2, false);
      if (d + 1 <= D) lv.scatter(d + 1, true);
      const int cnt  = lv.count(d);
      const int grid = grid_for((int64_t)cnt * 32, 1, h.sm_count * 16);
      if (out.offs64)
        B200_LAUNCH(h, (k_bc_backward<int64_t>), grid, kBlock, 0, out.offsets.as<int64_t>(), out.indices.as<int32_t>(), lv.lq(d),
                    lv.lw(d), cnt, lv.words.as<u64>(), sigma.as<double>(), delta.as<double>(), ld, bc, ebc, d == 0, endpoints);
      else
        B200_LAUNCH(h, (k_bc_backward<int32_t>), grid, kBlock, 0, out.offsets.as<int32_t>(), out.indices.as<int32_t>(), lv.lq(d),
                    lv.lw(d), cnt, lv.words.as<u64>(), sigma.as<double>(), delta.as<double>(), ld, bc, ebc, d == 0, endpoints);
    }
    if (D >= 1) lv.scatter(1, false);  // the words array is all zero again for the next batch
    if (trace) {
      cudaEventRecord(t2, h.stream);
      cudaEventSynchronize(t2);
      float fwd = 0.f, bwd = 0.f;
      cudaEventElapsedTime(&fwd, t0, t1);
      cudaEventElapsedTime(&bwd, t1, t2);
      std::fprintf(stderr, "betweenness batch %d sources %d levels %d entries %zu: bfs %.3f ms sigma %.3f ms backward %.3f ms\n",
                   (int)(b0 / ld), nb, D + 1, lv.first.back(), fwd - lv.pull_ms, lv.pull_ms, bwd);
    }
  }
  if (trace) {
    cudaEventDestroy(t0);
    cudaEventDestroy(t1);
    cudaEventDestroy(t2);
  }
  check_last("betweenness");
}

// the sources: every vertex (vertex_list == NULL) or the list's vertices as internal ids
dbuf sources_of(handle_impl const& h, graph_impl const& g, device_array_view_impl const* vl, size_t& n)
{
  const int32_t nv = g.n_vertices;
  if (!vl) {
    n        = (size_t)nv;
    dbuf all = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    B200_LAUNCH(h, k_iota<int32_t>, grid_for(nv), kBlock, 0, all.as<int32_t>(), (int64_t)nv);
    return all;
  }
  B200_EXPECTS(vl->type == g.vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and vertex_list must match");
  n        = vl->size;
  dbuf out = make_dbuf<int32_t>(std::max<size_t>(n, 1), h.stream);
  ext_to_int(h, g, vl->data, n, out.as<int32_t>());
  if (n > 0) {
    std::vector<int32_t> hs(n);
    CUDA_TRY(cudaMemcpyAsync(hs.data(), out.data(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    for (auto v : hs) B200_EXPECTS(v >= 0, CUGRAPH_INVALID_INPUT, "Invalid input argument: sources have invalid vertex IDs.");
  }
  return out;
}

// betweenness_centrality_impl.cuh:1432-1490, in the weight type
template <typename T>
void vertex_betweenness(handle_impl const& h, graph_impl& g, device_array_view_impl const* vl, bool normalized, bool endpoints,
                        centrality_result_impl& res)
{
  const int32_t nv = g.n_vertices;
  size_t n         = 0;
  dbuf src         = sources_of(h, g, vl, n);
  dbuf bc          = make_dbuf<double>(std::max(nv, 1), h.stream);
  CUDA_TRY(cudaMemsetAsync(bc.data(), 0, sizeof(double) * std::max(nv, 1), h.stream));
  brandes(h, g, src.as<int32_t>(), n, endpoints, bc.as<double>(), nullptr);
  dbuf is_source = make_dbuf<uint8_t>(std::max(nv, 1), h.stream);
  CUDA_TRY(cudaMemsetAsync(is_source.data(), 0, std::max(nv, 1), h.stream));
  if (n) B200_LAUNCH(h, k_mark_sources, grid_for((int64_t)n), kBlock, 0, src.as<int32_t>(), (int64_t)n, is_source.as<uint8_t>());
  T num_vertices = (T)nv;
  if (!endpoints) num_vertices = num_vertices - 1;
  const T ns = (T)n;
  T s_non, s_src;
  if ((T)(int64_t)n == num_vertices || endpoints) {
    if (normalized) s_non = (T)(ns * (num_vertices - 1));
    else if (g.is_symmetric) s_non = (T)(ns * 2) / num_vertices;
    else s_non = ns / num_vertices;
    s_src = s_non;
  } else if (normalized) {
    s_non = ns * (num_vertices - 1);
    s_src = (T)(n - 1) * (num_vertices - 1);
  } else {
    s_non = ns / num_vertices;
    s_src = (T)(n - 1) / num_vertices;
    if (g.is_symmetric) {
      s_non *= 2;
      s_src *= 2;
    }
  }
  dbuf vals = make_dbuf<T>(std::max(nv, 1), h.stream);
  B200_LAUNCH(h, (k_bc_finish<T>), grid_for(nv), kBlock, 0, bc.as<double>(), nv, is_source.as<uint8_t>(), 1, s_non, s_src, vals.as<T>());
  res.vertices  = new device_array_impl{reported_vertices(h, g), (size_t)nv, g.vertex_type};
  res.values    = new device_array_impl{to_reported_order(h, g, vals.data(), sizeof(T)), (size_t)nv, g.weight_type};
  res.converged = true;
  check_last("betweenness_centrality");
  sync(h);
}

struct edge_centrality_result_impl {
  device_array_impl* src{nullptr};
  device_array_impl* dst{nullptr};
  device_array_impl* values{nullptr};
};

// betweenness_centrality_impl.cuh:1581-1606, in the weight type; one row per edge of the push view, in its order
template <typename T>
void edge_betweenness(handle_impl const& h, graph_impl& g, device_array_view_impl const* vl, bool normalized,
                      edge_centrality_result_impl& res)
{
  const int32_t nv = g.n_vertices;
  size_t n         = 0;
  dbuf src         = sources_of(h, g, vl, n);
  csx_t const& out = push_view(h, g);
  const int64_t m  = out.nnz;
  dbuf ebc         = make_dbuf<double>(std::max<int64_t>(m, 1), h.stream);
  dbuf bc          = make_dbuf<double>(std::max(nv, 1), h.stream);
  CUDA_TRY(cudaMemsetAsync(ebc.data(), 0, sizeof(double) * std::max<int64_t>(m, 1), h.stream));
  CUDA_TRY(cudaMemsetAsync(bc.data(), 0, sizeof(double) * std::max(nv, 1), h.stream));
  brandes(h, g, src.as<int32_t>(), n, false, bc.as<double>(), ebc.as<double>());
  bool scaled = false;
  T sf        = (T)1;
  if (normalized) {
    const T nn = (T)nv;
    sf         = nn * (nn - 1);
    scaled     = true;
  } else if (g.is_symmetric) {
    sf     = (T)2;
    scaled = true;
  }
  if (scaled && nv > 1 && (int64_t)n < (int64_t)nv) sf *= (T)n / (T)nv;
  scaled = scaled && nv > 1;
  dbuf vals = make_dbuf<T>(std::max<int64_t>(m, 1), h.stream);
  B200_LAUNCH(h, (k_ebc_finish<T>), grid_for(m), kBlock, 0, ebc.as<double>(), m, scaled, sf, vals.as<T>());
  const size_t es = dtype_size(g.vertex_type);
  dbuf maj        = m ? expand_majors(h, out) : dbuf();
  dbuf s_ext((size_t)m * es, h.stream), d_ext((size_t)m * es, h.stream);
  int_to_ext(h, g, maj.as<int32_t>(), (size_t)m, s_ext.data());
  int_to_ext(h, g, out.indices.as<int32_t>(), (size_t)m, d_ext.data());
  res.src    = new device_array_impl{std::move(s_ext), (size_t)m, g.vertex_type};
  res.dst    = new device_array_impl{std::move(d_ext), (size_t)m, g.vertex_type};
  res.values = new device_array_impl{std::move(vals), (size_t)m, g.weight_type};
  check_last("edge_betweenness_centrality");
  sync(h);
}

struct rng_state_impl {
  uint64_t seed;
  uint64_t counter;  // stream position of the next draw
};

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_betweenness_centrality(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                    const cugraph_type_erased_device_array_view_t* vertex_list, bool_t normalized,
                                                    bool_t include_endpoints, bool_t do_expensive_check,
                                                    cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;  // invalid sources are always rejected
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result  = nullptr;
    auto res = std::make_unique<centrality_result_impl>();
    if (g->weight_type == FLOAT64)
      vertex_betweenness<double>(h, *g, V(vertex_list), normalized == TRUE, include_endpoints == TRUE, *res);
    else
      vertex_betweenness<float>(h, *g, V(vertex_list), normalized == TRUE, include_endpoints == TRUE, *res);
    *result = reinterpret_cast<cugraph_centrality_result_t*>(res.release());
  });
}

cugraph_error_code_t cugraph_edge_betweenness_centrality(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                         const cugraph_type_erased_device_array_view_t* vertex_list,
                                                         bool_t normalized, bool_t do_expensive_check,
                                                         cugraph_edge_centrality_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result  = nullptr;
    auto res = std::make_unique<edge_centrality_result_impl>();
    if (g->weight_type == FLOAT64) edge_betweenness<double>(h, *g, V(vertex_list), normalized == TRUE, *res);
    else edge_betweenness<float>(h, *g, V(vertex_list), normalized == TRUE, *res);
    *result = reinterpret_cast<cugraph_edge_centrality_result_t*>(res.release());
  });
}

static edge_centrality_result_impl* ER(cugraph_edge_centrality_result_t* r) { return reinterpret_cast<edge_centrality_result_impl*>(r); }

cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_src_vertices(cugraph_edge_centrality_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(ER(result)->src->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_dst_vertices(cugraph_edge_centrality_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(ER(result)->dst->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_edge_ids(cugraph_edge_centrality_result_t* result)
{
  (void)result;  // no edge ids are stored
  return nullptr;
}
cugraph_type_erased_device_array_view_t* cugraph_edge_centrality_result_get_values(cugraph_edge_centrality_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(ER(result)->values->new_view());
}
void cugraph_edge_centrality_result_free(cugraph_edge_centrality_result_t* result)
{
  if (!result) return;
  auto* r = ER(result);
  delete r->src;
  delete r->dst;
  delete r->values;
  delete r;
}

cugraph_error_code_t cugraph_rng_state_create(const cugraph_resource_handle_t* handle, uint64_t seed, cugraph_rng_state_t** state,
                                              cugraph_error_t** error)
{
  return guarded(error, [&] {
    (void)H(handle);
    B200_EXPECTS(state != nullptr, CUGRAPH_INVALID_INPUT, "state out-pointer is NULL");
    *state = reinterpret_cast<cugraph_rng_state_t*>(new rng_state_impl{seed, 0});
  });
}

void cugraph_rng_state_free(cugraph_rng_state_t* p) { delete reinterpret_cast<rng_state_impl*>(p); }

cugraph_error_code_t cugraph_select_random_vertices(const cugraph_resource_handle_t* handle, const cugraph_graph_t* graph,
                                                    cugraph_rng_state_t* rng_state, size_t num_vertices,
                                                    cugraph_type_erased_device_array_t** vertices, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto const* g = G(const_cast<cugraph_graph_t*>(graph));
    B200_EXPECTS(rng_state != nullptr, CUGRAPH_INVALID_INPUT, "rng_state is NULL");
    B200_EXPECTS(vertices != nullptr, CUGRAPH_INVALID_INPUT, "vertices out-pointer is NULL");
    *vertices        = nullptr;
    const int32_t nv = g->n_vertices;
    B200_EXPECTS(num_vertices <= (size_t)nv, CUGRAPH_INVALID_INPUT,
                 "Invalid input arguments: select_count should not exceed the number of vertices when sampling without replacement.");
    auto* st = reinterpret_cast<rng_state_impl*>(rng_state);
    dbuf keys = make_dbuf<u64>(std::max(nv, 1), h.stream), ranks = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    dbuf keys_s = make_dbuf<u64>(std::max(nv, 1), h.stream), ranks_s = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    B200_LAUNCH(h, k_random_keys, grid_for(nv), kBlock, 0, keys.as<u64>(), ranks.as<int32_t>(), nv, (u64)st->seed, (u64)st->counter);
    st->counter += (uint64_t)nv;
    if (nv > 0) sort_pairs<u64, int32_t>(h, keys.as<u64>(), keys_s.as<u64>(), ranks.as<int32_t>(), ranks_s.as<int32_t>(), nv, 0, 64);
    B200_LAUNCH(h, k_rank_to_int, grid_for((int64_t)num_vertices), kBlock, 0, ranks_s.as<int32_t>(), (int64_t)num_vertices,
                g->int_of_rank.as<int32_t>());
    dbuf out(num_vertices * dtype_size(g->vertex_type), h.stream);
    int_to_ext(h, *g, ranks_s.as<int32_t>(), num_vertices, out.data());
    check_last("select_random_vertices");
    sync(h);
    *vertices = wrap_array(std::move(out), num_vertices, g->vertex_type);
  });
}

}  // extern "C"
