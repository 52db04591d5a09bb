// The load-balanced frontier advance (merge-path partition of a queue's edges into equal tiles) and the small device
// helpers around it.  Shared by the single-GPU traversals (traverse.cu: BFS top-down levels, SSSP rounds), strongly
// connected components (scc.cu: trim, reach and colouring rounds) and the multi-GPU
// block relaxation (mg.cu: cugraph_b200_block_sssp_relax / _pred), which advance over a queue of physical rows of a block's
// push copy.  Everything lives in an anonymous namespace: every translation unit gets its own instantiations.
#pragma once
#include "graph.cuh"

#include <cub/cub.cuh>

#include <algorithm>

namespace b200 {
namespace {

// ------------------------------------------------------------------------------------------
// warp-aggregated append: the active lanes of a diverged warp claim consecutive queue slots
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int warp_append(int* counter)
{
  unsigned mask = __activemask();
  int leader    = __ffs(mask) - 1;
  int lane      = threadIdx.x & 31;
  int base      = 0;
  if (lane == leader) base = atomicAdd(counter, __popc(mask));
  base = __shfl_sync(mask, base, leader);
  return base + __popc(mask & ((1u << lane) - 1u));
}

// the active lanes of a diverged warp add their values to *target with one atomic
__device__ __forceinline__ void warp_add_u64(unsigned long long* target, unsigned v)
{
  unsigned mask = __activemask();
  unsigned sum  = __reduce_add_sync(mask, v);
  if ((threadIdx.x & 31) == __ffs(mask) - 1) atomicAdd(target, (unsigned long long)sum);
}

// the sum of v over a whole warp, in every lane (every lane must call it)
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------
// generic load-balanced advance over a queue of frontier vertices (merge-path style):
//   1. degrees of the queue entries -> exclusive scan (CUB, library code for the tiny per-level scan)
//   2. the summed edge range is cut into tiles of kTileEdges; a CTA finds the vertices of its tile by
//      binary search, stages their scan / offsets in shared memory and strides over the tile's edges.
// Every CTA gets the same number of edges whatever the degree mix (a 400k-edge hub is spread over
// ~200 CTAs, 2000 degree-1 vertices share one).
// Op: __device__ void edge(int src, long long e, int nbr)
// ------------------------------------------------------------------------------------------
constexpr int kTileEdges = 2048;
constexpr int kTileVerts = 2048;

template <typename O>
__global__ void k_queue_degrees(O const* __restrict__ off, int32_t const* __restrict__ q, int n, int32_t* __restrict__ deg)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) deg[i] = (int32_t)((long long)off[q[i] + 1] - (long long)off[q[i]]);
  if (i == n) deg[i] = 0;
}

__device__ __forceinline__ int upper_bound_minus1(int32_t const* a, int n, int key)
{
  int lo = 0, hi = n;  // first index with a[idx] > key
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] <= key) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

// first and last queue entry of every tile: two binary searches per tile, all tiles in parallel (the merge-path
// partition).  Done inside k_advance by thread 0 of every CTA they were 2 x log2(n) dependent global loads that the
// other 255 threads waited for, tile after tile.
__global__ void k_tile_owners(int32_t const* __restrict__ scan, int n_frontier, int n_tiles, int2* __restrict__ tile_k)
{
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tiles) return;
  const long long total = scan[n_frontier];  // < 2^31 (advance() splits larger queues); the tile bounds are computed in 64 bits
  const long long e0    = (long long)t * kTileEdges;
  const long long e1    = (e0 + kTileEdges < total) ? e0 + kTileEdges : total;
  if (e0 >= total) {
    tile_k[t] = make_int2(0, -1);
    return;
  }
  tile_k[t] = make_int2(upper_bound_minus1(scan, n_frontier, (int)e0), upper_bound_minus1(scan, n_frontier, (int)(e1 - 1)));
}

// IDENT: the queue is the identity (vertex k is queue entry k) and `scan` are the row offsets themselves
template <typename O, typename Op, bool IDENT>
__global__ void __launch_bounds__(kBlock)
k_advance(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ frontier,
          int n_frontier, int32_t const* __restrict__ scan /* n_frontier + 1 */, int2 const* __restrict__ tile_k, int n_tiles,
          Op op)
{
  __shared__ int s_scan[kTileVerts + 1];
  __shared__ int s_owner[kTileEdges];
  __shared__ int s_warp[kBlock / 32];
  constexpr int kPer = kTileEdges / kBlock;  // consecutive slots per thread in the owner fill
  const int total    = scan[n_frontier];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int tile = blockIdx.x; tile < n_tiles && (long long)tile * kTileEdges < total; tile += gridDim.x) {
    const int e0  = tile * kTileEdges;  // < total < 2^31 by the loop condition
    const int e1  = ((long long)e0 + kTileEdges < (long long)total) ? e0 + kTileEdges : total;
    const int2 kk = tile_k[tile];
    const int k0 = kk.x, k1 = kk.y;
    const int nv = k1 - k0 + 1;
    const bool staged = nv <= kTileVerts;
    for (int i = threadIdx.x; i < kTileEdges; i += kBlock) s_owner[i] = -1;
    if (staged)
      for (int i = threadIdx.x; i <= nv; i += kBlock) s_scan[i] = scan[k0 + i];
    __syncthreads();
    // mark the first slot of every queue entry of the tile (empty entries share a slot with their
    // successor: the largest index wins), then fill forward with a block-wide max-scan
    for (int k = k0 + threadIdx.x; k <= k1; k += kBlock) {
      const int start = staged ? s_scan[k - k0] : scan[k];
      const int p     = (start > e0 ? start : e0) - e0;
      if (p < e1 - e0) atomicMax(s_owner + p, k);
    }
    __syncthreads();
    int own[kPer];
    int run = -1;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int o = s_owner[threadIdx.x * kPer + j];
      run         = o > run ? o : run;
      own[j]      = run;
    }
    int incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl = y > incl ? y : incl;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int before = -1;  // max over all previous threads
    for (int wv = 0; wv < wid; ++wv) before = s_warp[wv] > before ? s_warp[wv] : before;
    const int prev_lane = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane > 0) before = prev_lane > before ? prev_lane : before;
#pragma unroll
    for (int j = 0; j < kPer; ++j) s_owner[threadIdx.x * kPer + j] = own[j] > before ? own[j] : before;
    __syncthreads();
    for (int e = e0 + threadIdx.x; e < e1; e += kBlock) {
      const int k   = s_owner[e - e0];
      const int v   = IDENT ? k : frontier[k];
      const int beg = staged ? s_scan[k - k0] : scan[k];
      const long long pos = (long long)off[v] + (e - beg);
      op.edge(v, pos, idx[pos]);
    }
    __syncthreads();
  }
}

// per-algorithm scratch for the advance
struct advance_scratch_t {
  dbuf deg, scan, tmp, tile_k;
  size_t tmp_bytes{0};
  size_t tile_cap{0};  // tiles tile_k holds: a queue of distinct vertices never spans more than nnz edges
  void init(handle_impl const& h, int32_t nv, int64_t nnz)
  {
    deg  = make_dbuf<int32_t>((size_t)nv + 1, h.stream);
    scan = make_dbuf<int32_t>((size_t)nv + 1, h.stream);
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, deg.as<int32_t>(), scan.as<int32_t>(), nv + 1, h.stream);
    tmp      = dbuf(tmp_bytes, h.stream);
    tile_cap = (size_t)(std::min<int64_t>(std::max<int64_t>(nnz, 0), (1ll << 31) - 1) / kTileEdges + 1);
    tile_k   = make_dbuf<int2>(tile_cap, h.stream);
  }
};

// total_edges = sum of the degrees of the queue entries (known on the host from the previous level)
// ready_deg: degrees of the queue entries if the producer of the queue already wrote them (n + 1 readable elements; the
// exclusive scan never uses the last one), else nullptr
// degree sum of queue entries [0, n)
template <typename O>
__global__ void k_queue_degree_sum(O const* __restrict__ off, int32_t const* __restrict__ q, int32_t const* __restrict__ ready_deg,
                                   int n, unsigned long long* __restrict__ out)
{
  unsigned long long t = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    t += ready_deg ? (unsigned long long)(unsigned)ready_deg[i] : (unsigned long long)((long long)off[q[i] + 1] - (long long)off[q[i]]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0 && t) atomicAdd(out, t);
}

template <typename O, typename Op>
void advance(handle_impl const& h, advance_scratch_t& sc, O const* off, int32_t const* idx, int32_t const* queue, int n,
             unsigned long long total_edges, Op op, int32_t const* ready_deg = nullptr)
{
  if (n <= 0) return;
  B200_EXPECTS(total_edges < (1ull << 31) || n > 1, CUGRAPH_UNKNOWN_ERROR, "a single vertex with 2^31 or more edges");
  if (total_edges >= h.tune.advance_split_edges && n > 1) {
    // the tile numbering is 32-bit: a queue whose degrees sum to 2^31 or more (graphs with 64-bit offsets) is advanced in
    // halves, each with its own degree sum (one small reduction + read-back per split; only such graphs ever get here)
    const int n1 = n / 2;
    dbuf d_sum   = make_dbuf<unsigned long long>(1, h.stream);
    CUDA_TRY(cudaMemsetAsync(d_sum.data(), 0, sizeof(unsigned long long), h.stream));
    B200_LAUNCH(h, (k_queue_degree_sum<O>), grid_for(n1, 1, h.sm_count * 8), kBlock, 0, off, queue, ready_deg, n1,
                d_sum.as<unsigned long long>());
    const unsigned long long e1 = read_back(h, d_sum.as<unsigned long long>());
    advance<O, Op>(h, sc, off, idx, queue, n1, e1, op, ready_deg);
    advance<O, Op>(h, sc, off, idx, queue + n1, n - n1, total_edges - e1, op, ready_deg ? ready_deg + n1 : nullptr);
    return;
  }
  if (!ready_deg) {
    B200_LAUNCH(h, (k_queue_degrees<O>), (n + 1 + kBlock - 1) / kBlock, kBlock, 0, off, queue, n, sc.deg.as<int32_t>());
    ready_deg = sc.deg.as<int32_t>();
  }
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(sc.tmp.data(), sc.tmp_bytes, ready_deg, sc.scan.as<int32_t>(), n + 1, h.stream));
  h.launches += 1;
  if (total_edges == 0) return;
  const int n_tiles = (int)((total_edges + kTileEdges - 1) / kTileEdges);
  dbuf spill;  // only if the caller's queue held duplicates (more edges than the graph has)
  int2* tile_k = sc.tile_k.as<int2>();
  if ((size_t)n_tiles > sc.tile_cap) {
    spill  = make_dbuf<int2>((size_t)n_tiles, h.stream);
    tile_k = spill.as<int2>();
  }
  B200_LAUNCH(h, k_tile_owners, (n_tiles + kBlock - 1) / kBlock, kBlock, 0, sc.scan.as<int32_t>(), n, n_tiles, tile_k);
  int grid = (int)std::min<unsigned long long>((unsigned long long)n_tiles, (unsigned long long)h.sm_count * 8);
  B200_LAUNCH(h, (k_advance<O, Op, false>), grid, kBlock, 0, off, idx, queue, n, sc.scan.as<int32_t>(), tile_k, n_tiles, op);
}

__device__ __forceinline__ float atomic_min_nonneg(float* addr, float v)
{
  return __int_as_float(atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v)));
}
__device__ __forceinline__ double atomic_min_nonneg(double* addr, double v)
{
  return __longlong_as_double(atomicMin(reinterpret_cast<long long*>(addr), __double_as_longlong(v)));
}

}  // namespace
}  // namespace b200
