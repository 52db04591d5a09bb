// Graph staging on the GPU: edge list (external ids) -> degree-ordered internal ids -> compressed
// rows with sorted neighbours + the bin / chunk metadata the hot-path kernels consume.
// Replaces (behaviourally) cpp/src/c_api/graph_sg.cpp:89-330 -> create_graph_from_edgelist
// (cpp/src/structure/create_graph_from_edgelist_impl.cuh:1430-1688) -> renumber_edgelist
// (renumber_edgelist_impl.cuh:419-833).  Staging is one-time and untimed; device-wide sorts and
// scans use CUB (library code), everything else is hand-written.
#include "graph.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace b200 {

namespace {

constexpr int kBlock = 256;

inline int grid_for(int64_t n, int per_thread = 1)
{
  int64_t b = (n + (int64_t)kBlock * per_thread - 1) / ((int64_t)kBlock * per_thread);
  return (int)std::min<int64_t>(std::max<int64_t>(b, 1), 1 << 20);
}

// ---------------------------------------------------------------- small device utilities
template <typename T>
__global__ void k_minmax(T const* a, int64_t n, long long* mn, long long* mx)
{
  long long lmn = LLONG_MAX, lmx = LLONG_MIN;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    long long v = (long long)a[i];
    lmn = v < lmn ? v : lmn;
    lmx = v > lmx ? v : lmx;
  }
  for (int o = 16; o > 0; o >>= 1) {
    long long t = __shfl_xor_sync(0xffffffffu, lmn, o);
    lmn = t < lmn ? t : lmn;
    t = __shfl_xor_sync(0xffffffffu, lmx, o);
    lmx = t > lmx ? t : lmx;
  }
  if (is_commit_lane()) {
    atomicMin(mn, lmn);
    atomicMax(mx, lmx);
  }
}

template <typename T>
__global__ void k_mark(T const* a, int64_t n, int32_t* flags)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    flags[a[i]] = 1;
}

template <typename T>
__global__ void k_dense_sorted_ext(int32_t const* flags, int32_t const* rank, int64_t m, T* sorted_ext)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
    if (flags[i]) sorted_ext[rank[i]] = (T)i;
}

template <typename T>
__global__ void k_rank_dense(T const* a, int64_t n, int32_t const* rank_tab, int32_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = rank_tab[a[i]];
}

template <typename T>
__device__ __forceinline__ int32_t lower_bound_dev(T const* a, int32_t n, T key)
{
  int32_t lo = 0, hi = n;
  while (lo < hi) {
    int32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// out[i] = rank of a[i] in sorted_ext, or -1
template <typename T>
__global__ void k_rank_search(T const* a, int64_t n, T const* sorted_ext, int32_t nv, int32_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    T key     = a[i];
    int32_t p = lower_bound_dev(sorted_ext, nv, key);
    out[i]    = (p < nv && sorted_ext[p] == key) ? p : -1;
  }
}

template <typename T>
__global__ void k_rank_identity(T const* a, int64_t n, int32_t nv, int32_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    long long v = (long long)a[i];
    out[i]      = (v >= 0 && v < nv) ? (int32_t)v : -1;
  }
}

__global__ void k_compose(int32_t const* rank, int64_t n, int32_t const* int_of_rank, int32_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t r = rank[i];
    out[i]    = r < 0 ? -1 : int_of_rank[r];
  }
}

__global__ void k_degree(int32_t const* major, int64_t n, int32_t* deg)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(&deg[major[i]], 1);
}

__global__ void k_degree_keys(int32_t const* deg, int32_t nv, uint64_t* keys)
{
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += gridDim.x * blockDim.x)
    keys[i] = ((uint64_t)(0x7fffffffu - (uint32_t)deg[i]) << 32) | (uint32_t)i;
}

__global__ void k_perm_from_keys(uint64_t const* keys, int32_t nv, int32_t* rank_of_int, int32_t* int_of_rank)
{
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += gridDim.x * blockDim.x) {
    int32_t r      = (int32_t)(keys[i] & 0xffffffffu);
    rank_of_int[i] = r;
    int_of_rank[r] = i;
  }
}

template <typename T>
__global__ void k_gather_ext(T const* sorted_ext, int32_t const* rank_of_int, int32_t nv, T* ext_of_int)
{
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += gridDim.x * blockDim.x)
    ext_of_int[i] = sorted_ext ? sorted_ext[rank_of_int[i]] : (T)rank_of_int[i];
}

// key = (relabel(major) << bits) | relabel_minor(minor)
__global__ void k_pack_keys(int32_t const* major, int32_t const* minor, int64_t n,
                            int32_t const* relabel_major, int32_t const* relabel_minor, int bits, uint64_t* keys)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t a = (uint32_t)(relabel_major ? relabel_major[major[i]] : major[i]);
    uint32_t b = (uint32_t)(relabel_minor ? relabel_minor[minor[i]] : minor[i]);
    keys[i]    = ((uint64_t)a << bits) | b;
  }
}

__global__ void k_iota64(int64_t n, uint32_t* v)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    v[i] = (uint32_t)i;
}

// order-preserving map of non-negative / general floats to unsigned
__device__ __forceinline__ uint32_t ord(float f)
{
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint64_t ord(double f)
{
  uint64_t u = (uint64_t)__double_as_longlong(f);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

template <typename W, typename U>
__global__ void k_weight_keys(W const* w, int64_t n, U* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = ord(w[i]);
}

template <typename T>
__global__ void k_gather(T const* in, uint32_t const* perm, int64_t n, T* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = in[perm[i]];
}

__global__ void k_run_heads(uint64_t const* keys, int64_t n, uint8_t* head)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// sorted keys -> offsets: offsets[r] = first position whose major >= r (row-parallel binary search,
// robust to long runs of empty rows), and indices = low bits
template <typename O>
__global__ void k_offsets(uint64_t const* keys, int64_t n, int bits, int32_t n_rows, O* offsets)
{
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      int64_t mid = lo + ((hi - lo) >> 1);
      if ((int64_t)(keys[mid] >> bits) < r) lo = mid + 1; else hi = mid;
    }
    offsets[r] = (O)lo;
  }
}

__global__ void k_indices(uint64_t const* keys, int64_t n, int bits, int32_t* indices)
{
  uint64_t mask = (bits >= 64) ? ~0ull : ((1ull << bits) - 1ull);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    indices[i] = (int32_t)(keys[i] & mask);
}

// rows with degree >= thr form a prefix (degrees descending): count them by binary search
template <typename O>
__global__ void k_segments(O const* offsets, int32_t n_rows, int32_t* seg /* kNumSeg */)
{
  int k = threadIdx.x;
  if (k >= kNumSeg) return;
  int thr    = (k < kNumSeg - 1) ? (32 >> k) : 0;  // == kSegThreshold[k]
  int32_t lo = 0, hi = n_rows;  // first row with degree < thr
  while (lo < hi) {
    int32_t mid = lo + ((hi - lo) >> 1);
    long long d = (long long)(offsets[mid + 1] - offsets[mid]);
    if (d >= thr) lo = mid + 1; else hi = mid;
  }
  seg[k] = lo;
}

template <typename O>
__global__ void k_check_sorted_degree(O const* offsets, int32_t n_rows, int* bad)
{
  for (int32_t r = blockIdx.x * blockDim.x + threadIdx.x; r + 1 < n_rows; r += gridDim.x * blockDim.x) {
    long long d0 = (long long)(offsets[r + 1] - offsets[r]);
    long long d1 = (long long)(offsets[r + 2] - offsets[r + 1]);
    if (d1 > d0) *bad = 1;
  }
}

// chunk c covers edges [c*kWarpChunk, (c+1)*kWarpChunk) of the degree>=32 prefix
template <typename O>
__global__ void k_chunk_rows(O const* offsets, int32_t n_hi_rows, int32_t n_chunks, int32_t* first_row, int32_t* straddle)
{
  for (int32_t c = blockIdx.x * blockDim.x + threadIdx.x; c <= n_chunks; c += gridDim.x * blockDim.x) {
    if (c == n_chunks) {
      first_row[c] = n_hi_rows;
      straddle[c]  = 0;
      continue;
    }
    long long e = (long long)c * kWarpChunk;
    int32_t lo = 0, hi = n_hi_rows;  // first row with offsets[row] > e
    while (lo < hi) {
      int32_t mid = lo + ((hi - lo) >> 1);
      if ((long long)offsets[mid] <= e) lo = mid + 1; else hi = mid;
    }
    int32_t row  = lo - 1;
    first_row[c] = row;
    straddle[c]  = ((long long)offsets[row] < e) ? 1 : 0;
  }
}

// a row that straddles several consecutive chunk boundaries is listed once
__global__ void k_split_flags(int32_t const* first_row, int32_t const* straddle, int32_t n_chunks, int32_t* uniq)
{
  for (int32_t c = blockIdx.x * blockDim.x + threadIdx.x; c <= n_chunks; c += gridDim.x * blockDim.x) {
    int f = 0;
    if (c < n_chunks && straddle[c]) f = !(c > 0 && straddle[c - 1] && first_row[c - 1] == first_row[c]);
    uniq[c] = f;
  }
}

__global__ void k_split_rows(int32_t const* first_row, int32_t const* uniq, int32_t const* scan, int32_t n_chunks,
                             int32_t* split_rows)
{
  for (int32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += gridDim.x * blockDim.x)
    if (uniq[c]) split_rows[scan[c]] = first_row[c];
}

template <typename O>
__global__ void k_expand_rows(O const* offsets, int32_t n_rows, int32_t const* row_vertex, int32_t* major_of_edge)
{
  // one warp per row (simple; staging only)
  int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  int lane     = threadIdx.x & 31;
  int64_t nw   = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_rows; r += nw) {
    int32_t v = row_vertex ? row_vertex[r] : (int32_t)r;
    for (long long e = (long long)offsets[r] + lane; e < (long long)offsets[r + 1]; e += 32) major_of_edge[e] = v;
  }
}

template <typename T>
__global__ void k_iota_t(int32_t n, T* out)
{
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = (T)i;
}

template <typename T>
__global__ void k_int_to_ext(int32_t const* in, int64_t n, T const* ext_of_int, T* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t v = in[i];
    out[i]    = v < 0 ? (T)-1 : ext_of_int[v];
  }
}

template <typename T>
__global__ void k_permute(T const* in, int32_t const* perm, int32_t n, T* out)
{
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[perm[i]];
}

template <typename T>
__global__ void k_fill(T* a, int64_t n, T v)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = v;
}

template <typename T>
__global__ void k_scatter_values(int32_t const* idx, T const* vals, int64_t n, T* out, int* n_invalid)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t v = idx[i];
    if (v < 0) atomicAdd(n_invalid, 1); else out[v] = vals[i];
  }
}

template <typename T>
__global__ void k_self_loop_flags(T const* s, T const* d, int64_t n, uint8_t* keep)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    keep[i] = s[i] != d[i];
}

template <typename T>
__global__ void k_copy_cast(void const* in, cugraph_data_type_id_t in_type, int64_t n, T* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (in_type == INT32) out[i] = (T) reinterpret_cast<int32_t const*>(in)[i];
    else out[i] = (T) reinterpret_cast<int64_t const*>(in)[i];
  }
}

// ---------------------------------------------------------------- CUB wrappers
struct cub_tmp {
  dbuf buf;
  void* ptr{nullptr};
  size_t bytes{0};
};

template <typename K>
void sort_keys(handle_impl const& h, K const* in, K* out, int64_t n, int begin_bit, int end_bit)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, bytes, in, out, n, begin_bit, end_bit, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp.data(), bytes, in, out, n, begin_bit, end_bit, h.stream));
  h.launches += 4;
}

template <typename K, typename Val>
void sort_pairs(handle_impl const& h, K const* kin, K* kout, Val const* vin, Val* vout, int64_t n, int begin_bit, int end_bit)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, n, begin_bit, end_bit, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.data(), bytes, kin, kout, vin, vout, n, begin_bit, end_bit, h.stream));
  h.launches += 4;
}

void exclusive_scan_i32(handle_impl const& h, int32_t const* in, int32_t* out, int64_t n)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, in, out, n, h.stream));
  h.launches += 2;
}

template <typename T>
int64_t select_flagged(handle_impl const& h, T const* in, uint8_t const* flags, T* out, int64_t n)
{
  dbuf d_count(sizeof(int64_t), h.stream);
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, bytes, in, flags, out, d_count.as<int64_t>(), n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.data(), bytes, in, flags, out, d_count.as<int64_t>(), n, h.stream));
  h.launches += 2;
  int64_t cnt = 0;
  CUDA_TRY(cudaMemcpyAsync(&cnt, d_count.data(), sizeof(int64_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  return cnt;
}

template <typename T>
int64_t unique_sorted(handle_impl const& h, T const* in, T* out, int64_t n)
{
  dbuf d_count(sizeof(int64_t), h.stream);
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceSelect::Unique(nullptr, bytes, in, out, d_count.as<int64_t>(), n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceSelect::Unique(tmp.data(), bytes, in, out, d_count.as<int64_t>(), n, h.stream));
  h.launches += 2;
  int64_t cnt = 0;
  CUDA_TRY(cudaMemcpyAsync(&cnt, d_count.data(), sizeof(int64_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  return cnt;
}

int bits_for(int64_t n)
{
  int b = 1;
  while ((1ll << b) < n) ++b;
  return b;
}

// ---------------------------------------------------------------- compressed-row construction
// (major, minor[, w]) in internal ids -> csx.  `relabel_major` maps a vertex id to its physical row.
template <typename W>
void build_csx_typed(handle_impl const& h, csx_t& out, int32_t const* major, int32_t const* minor, W const* w,
                     int64_t n, int32_t nv, int32_t const* relabel_major, int32_t const* relabel_minor,
                     bool dedupe, bool keep_min_weight)
{
  phase_trace tr(h);
  int bits = bits_for(std::max<int64_t>(nv, 2));
  B200_EXPECTS(2 * bits <= 64, CUGRAPH_INVALID_INPUT, "too many vertices");
  dbuf keys  = make_dbuf<uint64_t>(n, h.stream);
  dbuf keys2 = make_dbuf<uint64_t>(n, h.stream);
  B200_LAUNCH(h, k_pack_keys, grid_for(n, 4), kBlock, 0, major, minor, n, relabel_major, relabel_minor, bits,
              keys.as<uint64_t>());
  dbuf wsorted;
  if (w == nullptr) {
    sort_keys<uint64_t>(h, keys.as<uint64_t>(), keys2.as<uint64_t>(), n, 0, 2 * bits);
  } else {
    dbuf perm  = make_dbuf<uint32_t>(n, h.stream);
    dbuf perm2 = make_dbuf<uint32_t>(n, h.stream);
    B200_EXPECTS(n < (1ll << 32), CUGRAPH_INVALID_INPUT, "weighted graphs are limited to 2^32 edges per GPU");
    B200_LAUNCH(h, k_iota64, grid_for(n, 4), kBlock, 0, n, perm.as<uint32_t>());
    if (dedupe && keep_min_weight) {
      // stable two-pass: order by weight first so that the run head after the key sort is the minimum
      using U = typename std::conditional<sizeof(W) == 4, uint32_t, uint64_t>::type;
      dbuf wk  = make_dbuf<U>(n, h.stream);
      dbuf wk2 = make_dbuf<U>(n, h.stream);
      B200_LAUNCH(h, (k_weight_keys<W, U>), grid_for(n, 4), kBlock, 0, w, n, wk.as<U>());
      sort_pairs<U, uint32_t>(h, wk.as<U>(), wk2.as<U>(), perm.as<uint32_t>(), perm2.as<uint32_t>(), n, 0,
                              (int)sizeof(U) * 8);
      B200_LAUNCH(h, (k_gather<uint64_t>), grid_for(n, 4), kBlock, 0, keys.as<uint64_t>(), perm2.as<uint32_t>(), n,
                  keys2.as<uint64_t>());
      std::swap(keys, keys2);
      std::swap(perm, perm2);
    }
    sort_pairs<uint64_t, uint32_t>(h, keys.as<uint64_t>(), keys2.as<uint64_t>(), perm.as<uint32_t>(),
                                   perm2.as<uint32_t>(), n, 0, 2 * bits);
    wsorted = make_dbuf<W>(n, h.stream);
    B200_LAUNCH(h, (k_gather<W>), grid_for(n, 4), kBlock, 0, w, perm2.as<uint32_t>(), n, wsorted.as<W>());
  }
  keys.release();
  tr.mark("csx: pack + sort");
  int64_t m = n;
  if (dedupe && n > 0) {
    dbuf head = make_dbuf<uint8_t>(n, h.stream);
    B200_LAUNCH(h, k_run_heads, grid_for(n, 4), kBlock, 0, keys2.as<uint64_t>(), n, head.as<uint8_t>());
    dbuf kd = make_dbuf<uint64_t>(n, h.stream);
    m       = select_flagged<uint64_t>(h, keys2.as<uint64_t>(), head.as<uint8_t>(), kd.as<uint64_t>(), n);
    if (w != nullptr) {
      dbuf wd = make_dbuf<W>(n, h.stream);
      select_flagged<W>(h, wsorted.as<W>(), head.as<uint8_t>(), wd.as<W>(), n);
      wsorted = std::move(wd);
    }
    keys2 = std::move(kd);
  }
  out.n_rows  = nv;
  out.nnz     = m;
  out.offs64  = m >= h.tune.offs64_min_edges;
  out.indices = make_dbuf<int32_t>(m, h.stream);
  B200_LAUNCH(h, k_indices, grid_for(m, 4), kBlock, 0, keys2.as<uint64_t>(), m, bits, out.indices.as<int32_t>());
  if (out.offs64) {
    out.offsets = make_dbuf<int64_t>((size_t)nv + 1, h.stream);
    B200_LAUNCH(h, (k_offsets<int64_t>), grid_for((int64_t)nv + 1), kBlock, 0, keys2.as<uint64_t>(), m, bits, nv,
                out.offsets.as<int64_t>());
  } else {
    out.offsets = make_dbuf<int32_t>((size_t)nv + 1, h.stream);
    B200_LAUNCH(h, (k_offsets<int32_t>), grid_for((int64_t)nv + 1), kBlock, 0, keys2.as<uint64_t>(), m, bits, nv,
                out.offsets.as<int32_t>());
  }
  if (w != nullptr) {
    if (m == n) {
      out.weights = std::move(wsorted);
    } else {  // shrink to fit
      out.weights = make_dbuf<W>(m, h.stream);
      CUDA_TRY(cudaMemcpyAsync(out.weights.data(), wsorted.data(), m * sizeof(W), cudaMemcpyDeviceToDevice, h.stream));
    }
  }
  check_last("build_csx");
  tr.mark("csx: indices + offsets");
}

void build_csx(handle_impl const& h, csx_t& out, int32_t const* major, int32_t const* minor, void const* w,
               cugraph_data_type_id_t wtype, int64_t n, int32_t nv, int32_t const* relabel_major,
               int32_t const* relabel_minor, bool dedupe, bool keep_min_weight)
{
  if (w == nullptr || wtype == FLOAT32)
    build_csx_typed<float>(h, out, major, minor, (float const*)w, n, nv, relabel_major, relabel_minor, dedupe,
                           keep_min_weight);
  else
    build_csx_typed<double>(h, out, major, minor, (double const*)w, n, nv, relabel_major, relabel_minor, dedupe,
                            keep_min_weight);
}

template <typename O>
void finish_binning_typed(handle_impl const& h, csx_t& c)
{
  O const* off = c.offsets.as<O>();
  dbuf d_seg   = make_dbuf<int32_t>(kNumSeg + 2, h.stream);
  CUDA_TRY(cudaMemsetAsync(d_seg.data(), 0, sizeof(int32_t) * (kNumSeg + 2), h.stream));
  B200_LAUNCH(h, (k_check_sorted_degree<O>), grid_for(c.n_rows), kBlock, 0, off, c.n_rows, d_seg.as<int>() + kNumSeg);
  B200_LAUNCH(h, (k_segments<O>), 1, 32, 0, off, c.n_rows, d_seg.as<int32_t>());
  int32_t hseg[kNumSeg + 2];
  CUDA_TRY(cudaMemcpyAsync(hseg, d_seg.data(), sizeof(hseg), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  B200_EXPECTS(hseg[kNumSeg] == 0, CUGRAPH_UNKNOWN_ERROR, "internal: rows are not degree-descending");
  for (int k = 0; k < kNumSeg; ++k) c.seg[k] = hseg[k];
  c.seg[kNumSeg] = c.n_rows;
  c.degree_sorted = true;
  O nnz_hi = 0;
  if (c.seg[0] > 0) {
    CUDA_TRY(cudaMemcpyAsync(&nnz_hi, off + c.seg[0], sizeof(O), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
  }
  c.nnz_hi   = (int64_t)nnz_hi;
  c.n_chunks = (int32_t)((c.nnz_hi + kWarpChunk - 1) / kWarpChunk);
  c.chunk_first_row = make_dbuf<int32_t>((size_t)c.n_chunks + 1, h.stream);
  dbuf straddle     = make_dbuf<int32_t>((size_t)c.n_chunks + 1, h.stream);
  dbuf uniq         = make_dbuf<int32_t>((size_t)c.n_chunks + 1, h.stream);
  dbuf scan         = make_dbuf<int32_t>((size_t)c.n_chunks + 1, h.stream);
  B200_LAUNCH(h, (k_chunk_rows<O>), grid_for(c.n_chunks + 1), kBlock, 0, off, c.seg[0], c.n_chunks,
              c.chunk_first_row.as<int32_t>(), straddle.as<int32_t>());
  B200_LAUNCH(h, k_split_flags, grid_for(c.n_chunks + 1), kBlock, 0, c.chunk_first_row.as<int32_t>(),
              straddle.as<int32_t>(), c.n_chunks, uniq.as<int32_t>());
  exclusive_scan_i32(h, uniq.as<int32_t>(), scan.as<int32_t>(), (int64_t)c.n_chunks + 1);
  int32_t n_split = 0;
  CUDA_TRY(cudaMemcpyAsync(&n_split, scan.as<int32_t>() + c.n_chunks, sizeof(int32_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  c.n_split    = n_split;
  c.split_rows = make_dbuf<int32_t>((size_t)std::max(n_split, 1), h.stream);
  B200_LAUNCH(h, k_split_rows, grid_for(c.n_chunks + 1), kBlock, 0, c.chunk_first_row.as<int32_t>(),
              uniq.as<int32_t>(), scan.as<int32_t>(), c.n_chunks, c.split_rows.as<int32_t>());
  check_last("finish_binning");
  sync(h);
}

void finish_binning(handle_impl const& h, csx_t& c)
{
  if (c.offs64) finish_binning_typed<int64_t>(h, c); else finish_binning_typed<int32_t>(h, c);
}

}  // namespace

// expand a csx back into (vertex-of-row per edge)
dbuf expand_majors(handle_impl const& h, csx_t const& c)
{
  dbuf maj = make_dbuf<int32_t>(c.nnz, h.stream);
  int grid = grid_for((int64_t)c.n_rows * 32);
  if (c.offs64)
    B200_LAUNCH(h, (k_expand_rows<int64_t>), grid, kBlock, 0, c.offsets.as<int64_t>(), c.n_rows,
                c.row_vertex.as<int32_t>(), maj.as<int32_t>());
  else
    B200_LAUNCH(h, (k_expand_rows<int32_t>), grid, kBlock, 0, c.offsets.as<int32_t>(), c.n_rows,
                c.row_vertex.as<int32_t>(), maj.as<int32_t>());
  return maj;
}

namespace {

struct staged_ids {
  int32_t nv{0};
  dbuf sorted_ext;  // VT[nv] (renumber) or empty
  dbuf src_rank;    // int32[n]
  dbuf dst_rank;
};

// external ids -> rank ids (dense 0..V-1 in ascending external order)
template <typename VT>
staged_ids compute_ranks(handle_impl const& h, VT const* verts, int64_t n_verts, VT const* src, VT const* dst,
                             int64_t n, bool renumber)
{
  staged_ids r;
  r.src_rank = make_dbuf<int32_t>(n, h.stream);
  r.dst_rank = make_dbuf<int32_t>(n, h.stream);
  dbuf mm    = make_dbuf<long long>(2, h.stream);
  long long init[2] = {LLONG_MAX, LLONG_MIN};
  CUDA_TRY(cudaMemcpyAsync(mm.data(), init, sizeof(init), cudaMemcpyHostToDevice, h.stream));
  if (n > 0) {
    B200_LAUNCH(h, (k_minmax<VT>), std::min(grid_for(n, 8), 2048), kBlock, 0, src, n, mm.as<long long>(), mm.as<long long>() + 1);
    B200_LAUNCH(h, (k_minmax<VT>), std::min(grid_for(n, 8), 2048), kBlock, 0, dst, n, mm.as<long long>(), mm.as<long long>() + 1);
  }
  if (n_verts > 0)
    B200_LAUNCH(h, (k_minmax<VT>), std::min(grid_for(n_verts, 8), 2048), kBlock, 0, verts, n_verts, mm.as<long long>(),
                mm.as<long long>() + 1);
  long long hmm[2];
  CUDA_TRY(cudaMemcpyAsync(hmm, mm.data(), sizeof(hmm), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  long long mn = hmm[0], mx = hmm[1];
  if (n == 0 && n_verts == 0) {
    r.nv = 0;
    return r;
  }
  if (!renumber) {
    B200_EXPECTS(mn >= 0, CUGRAPH_INVALID_INPUT, "renumber=false requires non-negative vertex ids");
    B200_EXPECTS(mx < 0x7fffffffll, CUGRAPH_INVALID_INPUT, "vertex id out of range for renumber=false");
    // the reference sizes the graph by the vertex list when given, else by max id + 1
    r.nv = (int32_t)(mx + 1);
    B200_LAUNCH(h, (k_rank_identity<VT>), grid_for(n, 4), kBlock, 0, src, n, r.nv, r.src_rank.as<int32_t>());
    B200_LAUNCH(h, (k_rank_identity<VT>), grid_for(n, 4), kBlock, 0, dst, n, r.nv, r.dst_rank.as<int32_t>());
    return r;
  }
  long long span      = mx - mn + 1;
  long long dense_cap = std::max<long long>(1ll << 22, 8 * (2 * n + n_verts));
  if (mn >= 0 && mx + 1 <= dense_cap && mx < 0x7fffffffll) {
    int64_t m   = mx + 1;
    dbuf flags  = make_dbuf<int32_t>(m + 1, h.stream);
    dbuf rank   = make_dbuf<int32_t>(m + 1, h.stream);
    CUDA_TRY(cudaMemsetAsync(flags.data(), 0, sizeof(int32_t) * (m + 1), h.stream));
    if (n > 0) {
      B200_LAUNCH(h, (k_mark<VT>), grid_for(n, 4), kBlock, 0, src, n, flags.as<int32_t>());
      B200_LAUNCH(h, (k_mark<VT>), grid_for(n, 4), kBlock, 0, dst, n, flags.as<int32_t>());
    }
    if (n_verts > 0) B200_LAUNCH(h, (k_mark<VT>), grid_for(n_verts, 4), kBlock, 0, verts, n_verts, flags.as<int32_t>());
    exclusive_scan_i32(h, flags.as<int32_t>(), rank.as<int32_t>(), m + 1);
    int32_t nv = 0;
    CUDA_TRY(cudaMemcpyAsync(&nv, rank.as<int32_t>() + m, sizeof(int32_t), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    r.nv         = nv;
    r.sorted_ext = make_dbuf<VT>(nv, h.stream);
    B200_LAUNCH(h, (k_dense_sorted_ext<VT>), grid_for(m, 4), kBlock, 0, flags.as<int32_t>(), rank.as<int32_t>(), m,
                r.sorted_ext.as<VT>());
    B200_LAUNCH(h, (k_rank_dense<VT>), grid_for(n, 4), kBlock, 0, src, n, rank.as<int32_t>(), r.src_rank.as<int32_t>());
    B200_LAUNCH(h, (k_rank_dense<VT>), grid_for(n, 4), kBlock, 0, dst, n, rank.as<int32_t>(), r.dst_rank.as<int32_t>());
    sync(h);
    return r;
  }
  (void)span;
  // general path: sort the concatenation, unique, binary-search ranks
  int64_t tot = 2 * n + n_verts;
  dbuf cat    = make_dbuf<VT>(tot, h.stream);
  dbuf cat2   = make_dbuf<VT>(tot, h.stream);
  if (n > 0) {
    CUDA_TRY(cudaMemcpyAsync(cat.as<VT>(), src, n * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(cat.as<VT>() + n, dst, n * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
  }
  if (n_verts > 0)
    CUDA_TRY(cudaMemcpyAsync(cat.as<VT>() + 2 * n, verts, n_verts * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
  sort_keys<VT>(h, cat.as<VT>(), cat2.as<VT>(), tot, 0, (int)sizeof(VT) * 8);
  int64_t nv = unique_sorted<VT>(h, cat2.as<VT>(), cat.as<VT>(), tot);
  B200_EXPECTS(nv < 0x7fffffffll, CUGRAPH_INVALID_INPUT, "more than 2^31-1 vertices on one GPU");
  r.nv         = (int32_t)nv;
  r.sorted_ext = make_dbuf<VT>(nv, h.stream);
  CUDA_TRY(cudaMemcpyAsync(r.sorted_ext.data(), cat.data(), nv * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
  B200_LAUNCH(h, (k_rank_search<VT>), grid_for(n, 2), kBlock, 0, src, n, r.sorted_ext.as<VT>(), r.nv, r.src_rank.as<int32_t>());
  B200_LAUNCH(h, (k_rank_search<VT>), grid_for(n, 2), kBlock, 0, dst, n, r.sorted_ext.as<VT>(), r.nv, r.dst_rank.as<int32_t>());
  sync(h);
  return r;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// symmetrise on rank ids.  Semantics of the reference's symmetrize_edgelist(reciprocal=false)
// (cpp/src/structure/symmetrize_edgelist_impl.cuh:77-110): group edges by unordered endpoint pair;
// the i-th lightest "lower" (src>dst) edge is paired with the i-th lightest "upper" one and the pair
// becomes one undirected edge with the averaged weight; unpaired edges keep their weight; every
// resulting undirected edge is stored in both directions; self-loops are kept once.
// ---------------------------------------------------------------------------------------------
namespace {

__global__ void k_sym_keys(int32_t const* s, int32_t const* d, int64_t n, int bits, uint64_t* comp)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t a = (uint32_t)s[i], b = (uint32_t)d[i];
    uint32_t hi = a > b ? a : b, lo = a > b ? b : a;
    uint64_t dir = a > b ? 0ull : (a < b ? 1ull : 2ull);
    comp[i] = ((((uint64_t)hi << bits) | lo) << 2) | dir;
  }
}

__device__ __forceinline__ int64_t lb64(uint64_t const* a, int64_t n, uint64_t key)
{
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    int64_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// pass 0: count outputs per element; pass 1: write them
template <typename W>
__global__ void k_sym_emit(uint64_t const* comp, W const* w, int64_t n, int bits, int32_t const* scan, int pass,
                           int32_t* cnt, int32_t* os, int32_t* od, W* ow)
{
  uint64_t mask = (1ull << bits) - 1ull;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t c   = comp[i];
    uint64_t key = c >> 2;
    int dir      = (int)(c & 3ull);
    int32_t hi = (int32_t)(key >> bits), lo = (int32_t)(key & mask);
    int emit = 0;
    W wt     = w ? w[i] : (W)0;
    if (dir == 2) {
      emit = 1;
    } else {
      int64_t r0 = lb64(comp, n, key << 2);
      int64_t r1 = lb64(comp, n, (key << 2) | 1ull);
      int64_t r2 = lb64(comp, n, (key << 2) | 2ull);
      int64_t L = r1 - r0, U = r2 - r1;
      if (dir == 0) {
        int64_t j = i - r0;
        emit      = 2;
        if (w && j < U) wt = (W)((w[i] + w[r1 + j]) / (W)2);
      } else {
        int64_t j = i - r1;
        emit      = (j >= L) ? 2 : 0;
      }
    }
    if (pass == 0) {
      cnt[i] = emit;
    } else if (emit > 0) {
      int32_t o = scan[i];
      os[o] = hi; od[o] = lo;
      if (ow) ow[o] = wt;
      if (emit == 2) {
        os[o + 1] = lo; od[o + 1] = hi;
        if (ow) ow[o + 1] = wt;
      }
    }
  }
}

template <typename W>
void symmetrize_typed(handle_impl const& h, dbuf& src, dbuf& dst, dbuf& w, bool weighted, int64_t& n, int32_t nv)
{
  int bits = bits_for(std::max<int64_t>(nv, 2));
  B200_EXPECTS(2 * bits + 2 <= 64, CUGRAPH_INVALID_INPUT, "too many vertices to symmetrize");
  B200_EXPECTS(2 * n < (1ll << 31), CUGRAPH_INVALID_INPUT, "symmetrize: edge list too large for one GPU pass");
  dbuf comp = make_dbuf<uint64_t>(n, h.stream), comp2 = make_dbuf<uint64_t>(n, h.stream);
  B200_LAUNCH(h, k_sym_keys, grid_for(n, 4), kBlock, 0, src.as<int32_t>(), dst.as<int32_t>(), n, bits, comp.as<uint64_t>());
  dbuf wsorted;
  if (weighted) {
    using U = typename std::conditional<sizeof(W) == 4, uint32_t, uint64_t>::type;
    dbuf perm = make_dbuf<uint32_t>(n, h.stream), perm2 = make_dbuf<uint32_t>(n, h.stream);
    dbuf wk = make_dbuf<U>(n, h.stream), wk2 = make_dbuf<U>(n, h.stream);
    B200_LAUNCH(h, k_iota64, grid_for(n, 4), kBlock, 0, n, perm.as<uint32_t>());
    B200_LAUNCH(h, (k_weight_keys<W, U>), grid_for(n, 4), kBlock, 0, w.as<W>(), n, wk.as<U>());
    sort_pairs<U, uint32_t>(h, wk.as<U>(), wk2.as<U>(), perm.as<uint32_t>(), perm2.as<uint32_t>(), n, 0, (int)sizeof(U) * 8);
    B200_LAUNCH(h, (k_gather<uint64_t>), grid_for(n, 4), kBlock, 0, comp.as<uint64_t>(), perm2.as<uint32_t>(), n, comp2.as<uint64_t>());
    sort_pairs<uint64_t, uint32_t>(h, comp2.as<uint64_t>(), comp.as<uint64_t>(), perm2.as<uint32_t>(), perm.as<uint32_t>(), n, 0, 2 * bits + 2);
    wsorted = make_dbuf<W>(n, h.stream);
    B200_LAUNCH(h, (k_gather<W>), grid_for(n, 4), kBlock, 0, w.as<W>(), perm.as<uint32_t>(), n, wsorted.as<W>());
  } else {
    sort_keys<uint64_t>(h, comp.as<uint64_t>(), comp2.as<uint64_t>(), n, 0, 2 * bits + 2);
    std::swap(comp, comp2);
  }
  // comp now holds the sorted composite keys
  dbuf cnt = make_dbuf<int32_t>(n + 1, h.stream), scan = make_dbuf<int32_t>(n + 1, h.stream);
  CUDA_TRY(cudaMemsetAsync(cnt.as<int32_t>() + n, 0, sizeof(int32_t), h.stream));
  B200_LAUNCH(h, (k_sym_emit<W>), grid_for(n, 2), kBlock, 0, comp.as<uint64_t>(), weighted ? wsorted.as<W>() : (W const*)nullptr,
              n, bits, (int32_t const*)nullptr, 0, cnt.as<int32_t>(), (int32_t*)nullptr, (int32_t*)nullptr, (W*)nullptr);
  exclusive_scan_i32(h, cnt.as<int32_t>(), scan.as<int32_t>(), n + 1);
  int32_t m = 0;
  CUDA_TRY(cudaMemcpyAsync(&m, scan.as<int32_t>() + n, sizeof(int32_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  dbuf os = make_dbuf<int32_t>(m, h.stream), od = make_dbuf<int32_t>(m, h.stream);
  dbuf ow;
  if (weighted) ow = make_dbuf<W>(m, h.stream);
  B200_LAUNCH(h, (k_sym_emit<W>), grid_for(n, 2), kBlock, 0, comp.as<uint64_t>(), weighted ? wsorted.as<W>() : (W const*)nullptr,
              n, bits, scan.as<int32_t>(), 1, (int32_t*)nullptr, os.as<int32_t>(), od.as<int32_t>(),
              weighted ? ow.as<W>() : (W*)nullptr);
  check_last("symmetrize");
  src = std::move(os);
  dst = std::move(od);
  if (weighted) w = std::move(ow);
  n = m;
}

}  // namespace

void symmetrize_ranks(handle_impl const& h, dbuf& src, dbuf& dst, dbuf& w, cugraph_data_type_id_t wtype, int64_t& n,
                      int32_t nv)
{
  bool weighted = w.data() != nullptr;
  if (!weighted || wtype == FLOAT32) symmetrize_typed<float>(h, src, dst, w, weighted, n, nv);
  else symmetrize_typed<double>(h, src, dst, w, weighted, n, nv);
}

// ---------------------------------------------------------------------------------------------
// the staging entry point used by capi_graph.cu
// ---------------------------------------------------------------------------------------------
template <typename VT>
void stage_graph_typed(handle_impl const& h, graph_impl& g, device_array_view_impl const* verts,
                       device_array_view_impl const* src, device_array_view_impl const* dst,
                       device_array_view_impl const* wv, bool renumber, bool drop_self_loops, bool drop_multi_edges,
                       bool symmetrize)
{
  phase_trace tr(h);
  int64_t n = (int64_t)src->size;
  // working copies in VT (inputs may legally be any integer width equal to the graph's vertex type)
  dbuf s_ext = make_dbuf<VT>(n, h.stream), d_ext = make_dbuf<VT>(n, h.stream);
  if (n > 0) {
    CUDA_TRY(cudaMemcpyAsync(s_ext.data(), src->data, n * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(d_ext.data(), dst->data, n * sizeof(VT), cudaMemcpyDeviceToDevice, h.stream));
  }
  dbuf w;
  size_t wsz = g.weighted ? dtype_size(g.weight_type) : 0;
  if (g.weighted) {
    w = dbuf(n * wsz, h.stream);
    if (n > 0) CUDA_TRY(cudaMemcpyAsync(w.data(), wv->data, n * wsz, cudaMemcpyDeviceToDevice, h.stream));
  }
  if (drop_self_loops && n > 0) {
    dbuf keep = make_dbuf<uint8_t>(n, h.stream);
    B200_LAUNCH(h, (k_self_loop_flags<VT>), grid_for(n, 4), kBlock, 0, s_ext.as<VT>(), d_ext.as<VT>(), n, keep.as<uint8_t>());
    dbuf s2   = make_dbuf<VT>(n, h.stream), d2 = make_dbuf<VT>(n, h.stream);
    int64_t m = select_flagged<VT>(h, s_ext.as<VT>(), keep.as<uint8_t>(), s2.as<VT>(), n);
    select_flagged<VT>(h, d_ext.as<VT>(), keep.as<uint8_t>(), d2.as<VT>(), n);
    if (g.weighted) {
      dbuf w2(n * wsz, h.stream);
      if (wsz == 4) select_flagged<float>(h, w.as<float>(), keep.as<uint8_t>(), w2.as<float>(), n);
      else select_flagged<double>(h, w.as<double>(), keep.as<uint8_t>(), w2.as<double>(), n);
      w = std::move(w2);
    }
    s_ext = std::move(s2);
    d_ext = std::move(d2);
    n     = m;
  }
  tr.mark("stage: copies/self-loops");
  staged_ids ranks = compute_ranks<VT>(h, verts ? (VT const*)verts->data : nullptr, verts ? (int64_t)verts->size : 0,
                                 s_ext.as<VT>(), d_ext.as<VT>(), n, renumber);
  s_ext.release();
  d_ext.release();
  tr.mark("stage: ranks");
  int32_t nv = ranks.nv;
  g.n_vertices = nv;
  g.renumbered = renumber;

  // the reference removes multi-edges FIRST (keeping the minimum weight when the graph is declared symmetric) and symmetrizes
  // what is left (c_api/graph_sg.cpp:203-247): (u,v,1), (u,v,2), (v,u,5) -> (u,v,1), (v,u,5) -> one undirected edge of weight 3
  if (drop_multi_edges && n > 0) {
    csx_t tmp;
    int32_t const* mj = g.store_transposed ? ranks.dst_rank.as<int32_t>() : ranks.src_rank.as<int32_t>();
    int32_t const* mn = g.store_transposed ? ranks.src_rank.as<int32_t>() : ranks.dst_rank.as<int32_t>();
    build_csx(h, tmp, mj, mn, g.weighted ? w.data() : nullptr, g.weight_type, n, nv, nullptr, nullptr, true, g.is_symmetric);
    dbuf maj_d = expand_majors(h, tmp);
    n          = tmp.nnz;
    if (g.store_transposed) {
      ranks.dst_rank = std::move(maj_d);
      ranks.src_rank = std::move(tmp.indices);
    } else {
      ranks.src_rank = std::move(maj_d);
      ranks.dst_rank = std::move(tmp.indices);
    }
    if (g.weighted) w = std::move(tmp.weights);
  }
  if (symmetrize && n > 0) symmetrize_ranks(h, ranks.src_rank, ranks.dst_rank, w, g.weight_type, n, nv);

  int32_t const* major = g.store_transposed ? ranks.dst_rank.as<int32_t>() : ranks.src_rank.as<int32_t>();
  int32_t const* minor = g.store_transposed ? ranks.src_rank.as<int32_t>() : ranks.dst_rank.as<int32_t>();
  void const* wptr     = g.weighted ? w.data() : nullptr;

  // degree-descending internal order (ties: ascending rank) — renumber_edgelist_impl.cuh:732-738
  dbuf deg = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  CUDA_TRY(cudaMemsetAsync(deg.data(), 0, sizeof(int32_t) * std::max(nv, 1), h.stream));
  if (n > 0) B200_LAUNCH(h, k_degree, grid_for(n, 4), kBlock, 0, major, n, deg.as<int32_t>());
  dbuf dk = make_dbuf<uint64_t>(std::max(nv, 1), h.stream), dk2 = make_dbuf<uint64_t>(std::max(nv, 1), h.stream);
  dbuf rank_of_int = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  g.int_of_rank    = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  if (nv > 0) {
    B200_LAUNCH(h, k_degree_keys, grid_for(nv), kBlock, 0, deg.as<int32_t>(), nv, dk.as<uint64_t>());
    sort_keys<uint64_t>(h, dk.as<uint64_t>(), dk2.as<uint64_t>(), nv, 0, 64);
    B200_LAUNCH(h, k_perm_from_keys, grid_for(nv), kBlock, 0, dk2.as<uint64_t>(), nv, rank_of_int.as<int32_t>(),
                g.int_of_rank.as<int32_t>());
  }
  g.ext_of_int = make_dbuf<VT>(std::max(nv, 1), h.stream);
  if (nv > 0)
    B200_LAUNCH(h, (k_gather_ext<VT>), grid_for(nv), kBlock, 0, renumber ? ranks.sorted_ext.as<VT>() : (VT const*)nullptr,
                rank_of_int.as<int32_t>(), nv, g.ext_of_int.as<VT>());
  if (renumber) g.sorted_ext = std::move(ranks.sorted_ext);
  tr.mark("stage: degree order");

  g.primary = std::make_unique<csx_t>();
  build_csx(h, *g.primary, major, minor, wptr, g.weight_type, n, nv, g.int_of_rank.as<int32_t>(),
            g.int_of_rank.as<int32_t>(), false, false);
  g.n_edges = g.primary->nnz;
  tr.mark("stage: build_csx");
  finish_binning(h, *g.primary);
  sync(h);
  tr.mark("stage: binning");
}

void stage_graph(handle_impl const& h, graph_impl& g, device_array_view_impl const* verts,
                 device_array_view_impl const* src, device_array_view_impl const* dst, device_array_view_impl const* wv,
                 bool renumber, bool drop_self_loops, bool drop_multi_edges, bool symmetrize)
{
  if (g.vertex_type == INT32)
    stage_graph_typed<int32_t>(h, g, verts, src, dst, wv, renumber, drop_self_loops, drop_multi_edges, symmetrize);
  else
    stage_graph_typed<int64_t>(h, g, verts, src, dst, wv, renumber, drop_self_loops, drop_multi_edges, symmetrize);
}

// CSR input: expand offsets to a source list, then the common path
void expand_offsets_to_rows(handle_impl const& h, void const* offsets, cugraph_data_type_id_t otype, int64_t n_rows,
                            int64_t nnz, void* rows_out, cugraph_data_type_id_t vtype);

// ---------------------------------------------------------------------------------------------
// orientation accessors
// ---------------------------------------------------------------------------------------------
// (major, minor[, w]) -> compressed rows whose PHYSICAL order is descending degree (row_vertex maps a
// physical row back to its major id), binned and chunked for the pull kernels.  Used for the lazily
// built transpose of a CSR graph and for the rectangular edge blocks of the multi-GPU partition.
std::unique_ptr<csx_t> build_binned_rows(handle_impl const& h, int32_t const* major, int32_t const* minor, void const* w,
                                         cugraph_data_type_id_t wtype, int64_t n, int32_t nv)
{
  dbuf deg = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  CUDA_TRY(cudaMemsetAsync(deg.data(), 0, sizeof(int32_t) * std::max(nv, 1), h.stream));
  if (n > 0) B200_LAUNCH(h, k_degree, grid_for(n, 4), kBlock, 0, major, n, deg.as<int32_t>());
  dbuf dk = make_dbuf<uint64_t>(std::max(nv, 1), h.stream), dk2 = make_dbuf<uint64_t>(std::max(nv, 1), h.stream);
  auto c        = std::make_unique<csx_t>();
  c->row_vertex = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  dbuf row_of_v = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
  if (nv > 0) {
    B200_LAUNCH(h, k_degree_keys, grid_for(nv), kBlock, 0, deg.as<int32_t>(), nv, dk.as<uint64_t>());
    sort_keys<uint64_t>(h, dk.as<uint64_t>(), dk2.as<uint64_t>(), nv, 0, 64);
    B200_LAUNCH(h, k_perm_from_keys, grid_for(nv), kBlock, 0, dk2.as<uint64_t>(), nv, c->row_vertex.as<int32_t>(),
                row_of_v.as<int32_t>());
  }
  build_csx(h, *c, major, minor, w, wtype, n, nv, row_of_v.as<int32_t>(), nullptr, false, false);
  finish_binning(h, *c);
  return c;
}

csx_t const& pull_view(handle_impl const& h, graph_impl& g)
{
  if (g.store_transposed || g.is_symmetric) return *g.primary;
  if (!g.pull_alt) {
    // transpose the primary CSR; physical rows re-sorted by in-degree so that the binned kernels apply
    csx_t const& p = *g.primary;
    dbuf maj       = expand_majors(h, p);  // sources
    g.pull_alt     = build_binned_rows(h, p.indices.as<int32_t>(), maj.as<int32_t>(), g.weighted ? p.weights.data() : nullptr,
                                       g.weight_type, p.nnz, g.n_vertices);
  }
  return *g.pull_alt;
}

// rows = sources, indices = destinations, in a layout the sweep kernels accept (degree-descending physical rows): the
// primary orientation of a CSR graph, a re-sorted transpose of a CSC graph (the mirror image of pull_view)
csx_t const& out_sweep_view(handle_impl const& h, graph_impl& g)
{
  if (!g.store_transposed || g.is_symmetric) return *g.primary;
  if (!g.out_alt) {
    csx_t const& p = *g.primary;  // CSC: rows = destinations, indices = sources
    dbuf maj       = expand_majors(h, p);
    g.out_alt      = build_binned_rows(h, p.indices.as<int32_t>(), maj.as<int32_t>(), g.weighted ? p.weights.data() : nullptr,
                                       g.weight_type, p.nnz, g.n_vertices);
  }
  return *g.out_alt;
}

csx_t const& push_view(handle_impl const& h, graph_impl& g)
{
  if (!g.store_transposed || g.is_symmetric) return *g.primary;
  if (!g.push_alt) {
    csx_t const& p = *g.primary;  // CSC: rows = destinations, indices = sources
    dbuf maj       = expand_majors(h, p);
    auto c         = std::make_unique<csx_t>();
    build_csx(h, *c, p.indices.as<int32_t>(), maj.as<int32_t>(), g.weighted ? p.weights.data() : nullptr,
              g.weight_type, p.nnz, g.n_vertices, nullptr, nullptr, false, false);
    c->degree_sorted = false;
    for (int k = 0; k <= kNumSeg; ++k) c->seg[k] = 0;
    sync(h);
    g.push_alt = std::move(c);
  }
  return *g.push_alt;
}

// ---------------------------------------------------------------------------------------------
// piece stream of all non-empty rows (sweep_layout_t, consumed by sweep.cuh)
// ---------------------------------------------------------------------------------------------
namespace {

// ---- staging of the piece stream.  All passes are O(nnz + #segments):
//   1. head flags: an edge starts a (row, block) segment if it starts its row or its source lies in another
//      block than its predecessor's (neighbours are sorted by source id)
//   2. segments = compacted head positions; each is cut into pieces of <= 64 entries, a piece gets its kind
//      (S / Q / H = 1 / 2 / <= 4 entries, F1..F8 = that many lane slots of 8 entries)
//   3. pieces are ordered (stable radix sort) by (band, block, kind); a run of one (band, block, kind) is cut into groups
//      of 256 / 128 / 64 / 32 pieces and chunks of a few groups; band by band, chunks are dealt to the persistent CTAs as
//      contiguous, cost-balanced ranges, the part of one block inside a range is a phase
//   4. one warp per group writes its step-rows (32 lanes x 16 bytes of ids) and row slots

template <typename O>
__global__ void k_hot_row_starts(O const* __restrict__ off, int32_t n_cov, uint8_t* __restrict__ flag)
{
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_cov) flag[(size_t)off[r]] = 1;  // covered rows are never empty
}

__global__ void k_hot_heads(int32_t const* __restrict__ idx, long long nnz, int W, uint8_t* __restrict__ flag)
{
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nnz; e += (long long)gridDim.x * blockDim.x) {
    if (e > 0 && !flag[e] && idx[e] / W != idx[e - 1] / W) flag[e] = 1;
  }
}

constexpr int kHotPieceSlots   = 8;                          // slots per piece (= steps per group) at most
constexpr int kHotPieceEntries = kHotPieceSlots * kHotSlot;  // 64

// per segment: its row (binary search in the offsets) and how many pieces it yields
template <typename O>
__global__ void k_hot_segment_info(int32_t const* __restrict__ head_pos, int32_t n_segs, long long nnz,
                                   O const* __restrict__ off, int32_t n_cov, int32_t* __restrict__ seg_row,
                                   int32_t* __restrict__ seg_pieces)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_segs) return;
  if (k == n_segs) {
    seg_pieces[k] = 0;
    return;
  }
  const long long start = head_pos[k];
  const long long end   = (k + 1 < n_segs) ? (long long)head_pos[k + 1] : nnz;
  int lo = 0, hi = n_cov;  // last row r with off[r] <= start
  while (hi - lo > 1) {
    const int mid = lo + ((hi - lo) >> 1);
    if ((long long)off[mid] <= start) lo = mid; else hi = mid;
  }
  seg_row[k]    = lo;
  seg_pieces[k] = (int)((end - start + kHotPieceEntries - 1) / kHotPieceEntries);
}

__host__ __device__ __forceinline__ int piece_kind(int len)
{
  return len == 1 ? kKindS : (len == 2 ? kKindQ : (len <= 4 ? kKindH : kKindF1 + (len + kHotSlot - 1) / kHotSlot - 1));
}

// per segment: write its pieces (start edge, entries, row) and their key = (band * B + block) * kNumKinds + kind
__global__ void k_hot_emit_pieces(int32_t const* __restrict__ head_pos, int32_t n_segs, long long nnz,
                                  int32_t const* __restrict__ idx, int W, int B, int32_t band_rows,
                                  int32_t const* __restrict__ seg_row,
                                  int32_t const* __restrict__ piece_off, uint32_t* __restrict__ piece_key,
                                  int32_t* __restrict__ piece_start, int32_t* __restrict__ piece_len,
                                  int32_t* __restrict__ piece_row)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_segs) return;
  const long long start = head_pos[k];
  const long long end   = (k + 1 < n_segs) ? (long long)head_pos[k + 1] : nnz;
  const int row         = seg_row[k];
  const int bb          = (row / band_rows) * B + idx[start] / W;  // (band, block)
  int p                 = piece_off[k];
  for (long long s = start; s < end; s += kHotPieceEntries, ++p) {
    const int len  = (int)((end - s < kHotPieceEntries) ? end - s : kHotPieceEntries);
    piece_key[p]   = (uint32_t)(bb * kNumKinds + piece_kind(len));
    piece_start[p] = (int32_t)s;
    piece_len[p]   = len;
    piece_row[p]   = row;
  }
}

__global__ void k_hot_class_starts(uint32_t const* __restrict__ sorted_key, int32_t n_pieces, int n_keys,
                                   int32_t* __restrict__ class_start)
{
  const int key = blockIdx.x * blockDim.x + threadIdx.x;
  if (key > n_keys) return;
  int lo = 0, hi = n_pieces;  // first piece with sorted_key >= key
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if (sorted_key[mid] < (uint32_t)key) lo = mid + 1; else hi = mid;
  }
  class_start[key] = lo;
}

struct sweep_fill_t {  // build-time companion of a chunk: its pieces start at piece_begin, its (band, block, kind) run ends at piece_end
  int32_t piece_begin, piece_end, block, pad;
};

// Host-side plan of the sweep's work structure, from the piece counts per (band, block, kind) alone (class_start[key] =
// first piece of key = (band * B + block) * kNumKinds + kind, pieces ordered by key):
//   group = 256 / 128 / 64 / 32 pieces of one kind (S / Q / H / F), 1 or (F kinds) 1..8 step-rows
//   chunk = consecutive groups of one kind in one block of one band, at most kind_chunk_groups(kind)
//   range = contiguous chunks of one band per persistent CTA, balanced by an estimate of their load/store-unit time (the
//           sweep is bound by it: one cycle per 128-byte line of ids, per conflict-free 32 gathers, per sector of atomics);
//           every band is dealt to the same n_cta CTAs on its own (one sweep launch per band)
//   phase = the chunks of one block inside one range (a CTA loads the block's slice once per phase)
// Pure host code: exercised on CPU through cugraph_b200_debug_plan_sweep[_bands] (tests/test_sweep_plan*_cpu.py).
struct sweep_plan_t {
  std::vector<sweep_chunk_t> chunks;
  std::vector<sweep_fill_t> fills;
  std::vector<sweep_phase_t> phases;
  std::vector<int32_t> cta_phase;   // n_bands * n_cta + 1
  std::vector<int32_t> band_phase;  // n_bands + 1
  int64_t n_steprows{0}, n_rowslots{0};
  int n_cta{1};
};

inline double sweep_group_cost(int kind)
{
  // Load/store-unit cycles.  The atomics dominate: a scattered 64-bit RED costs about one cycle PER LANE whatever its
  // sectors (measured: plain stores or one sector per warp instead of scattered atomics made no difference), i.e.
  // ~1.2 cycles per piece; a step-row costs 4 lines of ids + 8 gathers at ~1.5 wavefronts.  The F8 pieces of hub rows are
  // summed by shuffles first (one RED per 32 pieces).
  return kind_steps(kind) * 14.0 + kind_pieces(kind) * (kind == kNumKinds - 1 ? 0.1 : 1.2) + 4.0;
}
constexpr double kPhaseCost = 2500.0;  // barrier + 192 KiB slice fill, in the same unit

bool plan_sweep(std::vector<int32_t> const& cstart, int n_bands, int B, int sm_count, sweep_plan_t& P)
{
  std::vector<double> cost;          // per chunk, the phase overhead on the first chunk of every block
  std::vector<size_t> band_chunk(1);  // chunks of band k: [band_chunk[k], band_chunk[k+1])
  for (int band = 0; band < n_bands; ++band) {
    for (int b = 0; b < B; ++b) {
      bool first = true;
      for (int kind = 0; kind < kNumKinds; ++kind) {
        const int key    = (band * B + b) * kNumKinds + kind;
        int32_t p        = cstart[key];
        const int32_t pe = cstart[key + 1];
        const int ppg = kind_pieces(kind), steps = kind_steps(kind), gmax = kind_chunk_groups(kind);
        while (p < pe) {
          const int groups = (int)std::min<int64_t>(gmax, ((int64_t)(pe - p) + ppg - 1) / ppg);
          if (P.n_steprows + (int64_t)groups * steps >= (1ll << 31) - 64 || P.n_rowslots + (int64_t)groups * ppg >= (1ll << 31) - 64)
            return false;  // 32-bit step-row / row-slot numbers
          P.chunks.push_back({(int32_t)P.n_steprows, (int32_t)P.n_rowslots, groups, kind});
          P.fills.push_back({p, pe, b, 0});
          cost.push_back(groups * sweep_group_cost(kind) + (first ? kPhaseCost : 0.0));
          first = false;
          P.n_steprows += (int64_t)groups * steps;
          P.n_rowslots += (int64_t)groups * ppg;
          p += groups * ppg;  // may pass pe inside the last group: the fill pads
        }
      }
    }
    band_chunk.push_back(P.chunks.size());
  }
  size_t most = 0;
  for (int band = 0; band < n_bands; ++band) most = std::max(most, band_chunk[band + 1] - band_chunk[band]);
  P.n_cta = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm_count, most));
  P.cta_phase.assign((size_t)n_bands * P.n_cta + 1, 0);
  P.band_phase.assign(n_bands + 1, 0);
  for (int band = 0; band < n_bands; ++band) {
    const size_t c_lo = band_chunk[band], n = band_chunk[band + 1] - c_lo;
    std::vector<double> pre(n + 1, 0.0);
    for (size_t c = 0; c < n; ++c) pre[c + 1] = pre[c] + cost[c_lo + c];
    P.band_phase[band] = (int32_t)P.phases.size();
    size_t c = 0;
    for (int cta = 0; cta < P.n_cta; ++cta) {
      const double target = pre[n] * (cta + 1) / P.n_cta;
      const size_t c0     = c;
      if (cta == P.n_cta - 1) c = n;
      else while (c < n && pre[c + 1] <= target) ++c;
      P.cta_phase[(size_t)band * P.n_cta + cta] = (int32_t)P.phases.size();
      for (size_t k = c_lo + c0; k < c_lo + c;) {  // split the range by block
        size_t e = k;
        while (e < c_lo + c && P.fills[e].block == P.fills[k].block) ++e;
        P.phases.push_back({P.fills[k].block, (int32_t)k, (int32_t)e, 0});
        k = e;
      }
    }
  }
  P.band_phase[n_bands]                  = (int32_t)P.phases.size();
  P.cta_phase[(size_t)n_bands * P.n_cta] = (int32_t)P.phases.size();
  return true;
}

// Bank-aware entry order inside the lane slots of the F kinds (4-byte values): order the entries of the 32 pieces of a group
// so that the k-th shared-memory gathers of the 32 lanes in every step (one LDS of the sweep kernel) fall into different
// banks.  Any assignment of a piece's entries to its (step, position) places is a valid layout (the sweep adds all of them
// into one sum per piece); padding may point at any of the kHotZeroPad zero columns, i.e. at any bank.  Greedy, place by
// place (bank_order_place below); a lane without a free bank waits for a later place while it has spare places left; all
// padding of a place shares one zero column on a free bank.  Sweep on RMAT-24: 0.373 ms without, 0.331 ms with this order.
// State per lane: bank_bits[b] = the piece's entries (bit e = entry e, <= 64 per piece) on bank b, `rem` = not placed yet,
// `have` = banks with an entry left.
struct bank_piece_t {
  unsigned long long bank_bits[32];
  unsigned long long rem;
  unsigned have;
  unsigned have2;  // banks with at least two entries left: used first, which keeps the number of distinct banks up
};

// one place of all 32 lanes: returns this lane's entry index (>= 0) or -1 - pad_bank for padding.
// PARALLEL greedy: every lane that still holds entries proposes a bank nobody has taken at this place (preferring banks of
// which its piece still holds several entries, search start rotated by lane and place); of the lanes proposing the same
// bank the one that comes first in an order rotating with the place wins, the others propose again — three rounds, then
// lanes that must place an entry now (no spare places left) take any bank.  (A version in which the 32 lanes took turns
// one after the other reached 1.5 wavefronts per load on RMAT-20 but cost 42 ms of staging at RMAT-24.)
constexpr int kBankRounds = 8;
__device__ __forceinline__ int bank_order_place(bank_piece_t& P, int places_left, int lane)
{
  unsigned taken = 0, taken2 = 0;  // banks used once / twice at this place (the same in every lane)
  int mine       = -1;
  const int spare = places_left - __popcll(P.rem);  // places beyond the ones the remaining entries need
  const int prio  = (lane + 11 * places_left) & 31;  // who wins a contested bank changes from place to place
  const int r0    = (lane + 5 * places_left) & 31;
#pragma unroll 1
  for (int round = 0; round < kBankRounds; ++round) {
    int want = -1;
    if (mine < 0 && P.rem != 0ull) {
      unsigned pick = P.have2 & ~taken;
      if (!pick) pick = P.have & ~taken;
      if (!pick && round >= kBankRounds - 2 && spare <= 0) {  // must place now: accept a conflict, on a bank used once if any
        pick = P.have & ~taken2;
        if (!pick && round == kBankRounds - 1) pick = P.have;
      }
      if (pick) {
        const unsigned rot = r0 ? ((pick >> r0) | (pick << (32 - r0))) : pick;
        want               = (__ffs(rot) - 1 + r0) & 31;
      }
    }
    // lanes with the same proposal: the smallest rotated priority wins (in the last round everybody proposing wins)
    const unsigned same = __match_any_sync(0xffffffffu, want);
    bool win            = want >= 0;
    if (win && round < kBankRounds - 1) {
      // winner = the lane of `same` whose prio is smallest: compare by scanning the (few) competitors
      unsigned others = same & ~(1u << lane);
      while (others) {
        const int o = __ffs(others) - 1;
        others &= others - 1;
        const int po = (o + 11 * places_left) & 31;
        if (po < prio) win = false;
      }
    }
    if (win) {
      mine = __ffsll((long long)(P.bank_bits[want] & P.rem)) - 1;
      P.rem &= ~(1ull << mine);
      const int left = __popcll(P.bank_bits[want] & P.rem);
      if (left < 2) P.have2 &= ~(1u << want);
      if (left < 1) P.have &= ~(1u << want);
    }
    const unsigned won = __reduce_or_sync(0xffffffffu, win ? (1u << want) : 0u);
    taken2 |= taken & won;
    taken |= won;
    if (!__any_sync(0xffffffffu, mine < 0 && P.rem != 0ull)) break;
  }
  if (mine >= 0) return mine;
  const int pad_bank = (~taken) ? __ffs(~taken) - 1 : 0;
  return -1 - pad_bank;
}

constexpr int kFillWarps = 6;  // = the largest kind_chunk_groups()

// one CTA per chunk, one warp per group
template <typename T, bool BANK>
__global__ void __launch_bounds__(kFillWarps * 32)
k_sweep_fill(sweep_chunk_t const* __restrict__ chunks, sweep_fill_t const* __restrict__ fills, int32_t const* __restrict__ perm,
             int32_t const* __restrict__ piece_start, int32_t const* __restrict__ piece_len,
             int32_t const* __restrict__ piece_row, int32_t const* __restrict__ idx, T const* __restrict__ w, int W,
             uint4* __restrict__ ids_out, T* __restrict__ w_out, int32_t* __restrict__ rows_out)
{
  const sweep_chunk_t ch = chunks[blockIdx.x];
  const sweep_fill_t fl  = fills[blockIdx.x];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  if (g >= ch.n_groups) return;
  const int col0 = fl.block * W;
  if (ch.kind < kKindF1) {  // S / Q / H: R pieces of E entries per lane; piece k of lane l is piece k * 32 + l of the group
    const int R = ch.kind == kKindS ? 8 : (ch.kind == kKindQ ? 4 : 2), E = 8 / R;
    const size_t slot = ((size_t)(unsigned)(ch.sr_begin + g) << 5) + lane;
    unsigned v[8];
    for (int k = 0; k < R; ++k) {
      const long long pi = (long long)fl.piece_begin + ((long long)g * 32 * R) + k * 32 + lane;
      int st = 0, ln = 0, row = -1;
      if (pi < fl.piece_end) {
        const int p = perm[pi];
        st          = piece_start[p];
        ln          = piece_len[p];
        row         = piece_row[p];
      }
      for (int e = 0; e < E; ++e) {
        v[k * E + e] = e < ln ? (unsigned)(idx[st + e] - col0) : (unsigned)W;
        if (w_out) w_out[slot * 8 + k * E + e] = e < ln ? w[st + e] : (T)0;
      }
      rows_out[(size_t)(unsigned)ch.row_begin + ((size_t)g * 32 + lane) * R + k] = row;
    }
    ids_out[slot] = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
    return;
  }
  const int C        = ch.kind - kKindF1 + 1;
  const long long pi = (long long)fl.piece_begin + (long long)g * 32 + lane;
  int st = 0, ln = 0, row = -1;
  if (pi < fl.piece_end) {
    const int p = perm[pi];
    st          = piece_start[p];
    ln          = piece_len[p];
    row         = piece_row[p];
  }
  rows_out[(size_t)(unsigned)ch.row_begin + (size_t)g * 32 + lane] = row;
  bank_piece_t bp;  // only used by the BANK instantiation
  if (BANK) {       // the whole warp takes part (lanes without a piece hold padding only)
    for (int b = 0; b < 32; ++b) bp.bank_bits[b] = 0ull;
    bp.have = bp.have2 = 0u;
    for (int e = 0; e < ln; ++e) {
      const int b = (idx[st + e] - col0) & 31;
      if (bp.bank_bits[b]) bp.have2 |= 1u << b;
      bp.bank_bits[b] |= 1ull << e;
      bp.have |= 1u << b;
    }
    bp.rem = ln >= 64 ? ~0ull : ((1ull << ln) - 1ull);
  }
  for (int j = 0; j < C; ++j) {
    const size_t slot = ((size_t)(unsigned)(ch.sr_begin + g * C + j) << 5) + lane;
    unsigned v[kHotSlot];
    if (BANK) {
#pragma unroll 1
      for (int k = 0; k < kHotSlot; ++k) {
        const int e = bank_order_place(bp, (C - j) * kHotSlot - k, lane);
        v[k]        = e >= 0 ? (unsigned)(idx[st + e] - col0) : (unsigned)(W + ((-1 - e - (W & 31)) & 31));
        if (w_out) w_out[slot * kHotSlot + k] = e >= 0 ? w[st + e] : (T)0;
      }
    } else {
#pragma unroll
      for (int k = 0; k < kHotSlot; ++k) {
        const int e   = j * kHotSlot + k;
        const bool in = e < ln;
        v[k]          = in ? (unsigned)(idx[st + e] - col0) : (unsigned)W;
        if (w_out) w_out[slot * kHotSlot + k] = in ? w[st + e] : (T)0;
      }
    }
    ids_out[slot] = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
  }
}

// ---- the tail layout (graph.cuh): runs of equal in-degree, tiles of 32 rows, lane-interleaved ids
// below[d] = first row of [row_lo, row_hi) whose in-degree is < d (rows are degree-descending), d = 0 .. kTailMaxDegree + 1
template <typename O>
__global__ void k_tail_run_bounds(O const* __restrict__ off, int32_t row_lo, int32_t row_hi, int32_t* __restrict__ below)
{
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d > kTailMaxDegree + 1) return;
  int lo = row_lo, hi = row_hi;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if ((long long)(off[mid + 1] - off[mid]) >= d) lo = mid + 1; else hi = mid;
  }
  below[d] = lo;
}

// one thread per lane of a tile
template <typename O, typename T>
__global__ void k_tail_fill(tail_run_t const* __restrict__ runs, int n_runs, O const* __restrict__ off,
                            int32_t const* __restrict__ idx, T const* __restrict__ w, int32_t pad_col,
                            int32_t* __restrict__ ids_out, T* __restrict__ w_out)
{
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)runs[n_runs].first_tile * kTailTile) return;
  const int tile = (int)(t / kTailTile), lane = (int)(t % kTailTile);
  int r = 0;
  while (tile >= runs[r + 1].first_tile) ++r;
  const tail_run_t R = runs[r];
  const int d        = R.degree;
  const int row      = R.first_row + (tile - R.first_tile) * kTailTile + lane;
  const bool live    = row < runs[r + 1].first_row;
  const long long e0 = live ? (long long)off[row] : 0;
  const long long o  = R.id_off + (long long)(tile - R.first_tile) * kTailTile * d + lane;
  for (int k = 0; k < d; ++k) {
    ids_out[o + (long long)k * kTailTile] = live ? idx[e0 + k] : pad_col;
    if (w_out) w_out[o + (long long)k * kTailTile] = live ? w[e0 + k] : (T)0;
  }
}

template <typename O>
void build_tail_layout(handle_impl const& h, csx_t const& c, int32_t nv, size_t es, sweep_layout_t& L)
{
  dbuf d_below = make_dbuf<int32_t>(kTailMaxDegree + 2, h.stream);
  B200_LAUNCH(h, (k_tail_run_bounds<O>), 1, 64, 0, c.offsets.as<O>(), L.n_str, L.n_cov, d_below.as<int32_t>());
  int32_t below[kTailMaxDegree + 2];
  CUDA_TRY(cudaMemcpyAsync(below, d_below.data(), sizeof(below), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  tail_run_t at{0, L.n_str, 0, 0, 0};  // the next run starts here
  for (int d = kTailMaxDegree; d >= 1; --d) {
    const int32_t lo = below[d + 1], hi = below[d];  // the rows of in-degree d
    if (hi <= lo) continue;
    B200_EXPECTS(lo == at.first_row, CUGRAPH_UNKNOWN_ERROR, "tail rows are not degree-descending");
    at.degree = d;
    L.tail_runs.push_back(at);
    const int32_t tiles = (hi - lo + kTailTile - 1) / kTailTile;
    at.first_row = hi;
    at.first_tile += tiles;
    at.first_unit += (tiles + tail_unit_tiles(d) - 1) / tail_unit_tiles(d);
    at.id_off += (int64_t)tiles * kTailTile * d;
  }
  B200_EXPECTS(at.first_row == L.n_cov, CUGRAPH_UNKNOWN_ERROR, "tail rows of in-degree >= the bound or 0");
  at.degree     = 0;
  L.n_tail_runs = (int)L.tail_runs.size();
  L.tail_runs.push_back(at);
  L.tail_run = make_dbuf<tail_run_t>(L.tail_runs.size(), h.stream);
  CUDA_TRY(cudaMemcpyAsync(L.tail_run.data(), L.tail_runs.data(), sizeof(tail_run_t) * L.tail_runs.size(), cudaMemcpyHostToDevice,
                           h.stream));
  L.tail_ids = make_dbuf<int32_t>((size_t)std::max<int64_t>(at.id_off, 1), h.stream);
  const bool weighted = c.weights.data() != nullptr;
  if (weighted) L.tail_w = dbuf((size_t)std::max<int64_t>(at.id_off, 1) * es, h.stream);
  const int64_t threads = (int64_t)at.first_tile * kTailTile;
  if (es == 4)
    B200_LAUNCH(h, (k_tail_fill<O, float>), grid_for(threads), kBlock, 0, L.tail_run.as<tail_run_t>(), L.n_tail_runs,
                c.offsets.as<O>(), c.indices.as<int32_t>(), c.weights.as<float>(), nv, L.tail_ids.as<int32_t>(), L.tail_w.as<float>());
  else
    B200_LAUNCH(h, (k_tail_fill<O, double>), grid_for(threads), kBlock, 0, L.tail_run.as<tail_run_t>(), L.n_tail_runs,
                c.offsets.as<O>(), c.indices.as<int32_t>(), c.weights.as<double>(), nv, L.tail_ids.as<int32_t>(), L.tail_w.as<double>());
  check_last("sweep tail layout");
  sync(h);  // the host run table is pageable
}

// Row bands: the sweep's fp64 REDs into acc[row] hit the L2 only while the rows they scatter over fit in it (measured on an
// H100 80GB HBM3 at 700 W, 50 MB of L2: a scattered RED.64 costs the same up to 24 MB of accumulators, 1.3x at 48 MB and
// 3.7x at 64 MB), so the stream rows are split into bands whose accumulators take at most kBandL2Share of the L2.  Half
// gave the fastest RMAT-24 sweep without a tail (3 bands, DESIGN.md §3.2); more bands add launch tails and slice loads.
// CUGRAPH_B200_SWEEP_BANDS forces a count (tests, A/B runs).
constexpr double kBandL2Share = 0.5;

int sweep_bands(handle_impl const& h, int32_t n_str)
{
  const int most = std::max(1, (int)(((int64_t)n_str + kBandRowAlign - 1) / kBandRowAlign));
  int P          = h.tune.sweep_bands;
  if (P <= 0) P = h.l2_bytes ? (int)std::ceil(8.0 * n_str / (kBandL2Share * (double)h.l2_bytes)) : 1;
  return std::min(std::max(P, 1), most);
}

// The piece stream holds the rows [0, seg[k]) for the bin k this returns: rows of in-degree >= kSegThreshold[k].
// By default the rows of in-degree < kSweepTailDegree leave it on graphs of at least kSweepTailMinEdges edges, and it holds
// every non-empty row on smaller ones.  CUGRAPH_B200_SWEEP_TAIL_DEGREE forces a bound on any graph (tests, A/B runs):
// 1 = no tail, other values are rounded down to a bin threshold.
int sweep_stream_bin(handle_impl const& h, csx_t const& c)
{
  int bound = h.tune.sweep_tail_degree;
  if (bound <= 0) bound = c.nnz >= kSweepTailMinEdges ? kSweepTailDegree : 1;
  int k = 0;
  while (kSegThreshold[k] > bound) ++k;  // kSegThreshold[kNumSeg - 2] = 1
  return k;
}

template <typename O>
std::unique_ptr<sweep_layout_t> build_sweep_layout(handle_impl const& h, csx_t const& c, int32_t nv, size_t es)
{
  phase_trace tr(h);
  const int W         = (int)(kHotSliceBytes / es) - kHotZeroPad;  // columns per block; the pad holds zeros
  const int32_t n_cov = c.seg[kNumSeg - 2];                         // rows of degree >= 1
  const int32_t n_str = c.seg[sweep_stream_bin(h, c)];              // rows of the stream; the tail is swept by k_sweep_tail
  if (n_str <= 0) return nullptr;                                   // no row reaches the bound: the plain sweep fits better
  const int B         = (int)(((int64_t)nv + W - 1) / W);
  int64_t nnz = 0;  // edges of the stream rows: a prefix of indices (rows are degree-descending)
  {
    O off_str;
    CUDA_TRY(cudaMemcpyAsync(&off_str, c.offsets.as<O>() + n_str, sizeof(O), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    nnz = (int64_t)off_str;
  }
  auto L              = std::make_unique<sweep_layout_t>();
  L->W = W; L->B = B; L->n_cov = n_cov; L->n_str = n_str; L->nnz = c.nnz;
  int32_t const* idx = c.indices.as<int32_t>();
  // equal bands of whole kBandRowAlign spans; rounding may leave fewer than asked for
  const int asked         = sweep_bands(h, n_str);
  const int32_t band_rows = (int32_t)((((int64_t)n_str + asked - 1) / asked + kBandRowAlign - 1) / kBandRowAlign * kBandRowAlign);
  const int n_bands       = (int)(((int64_t)n_str + band_rows - 1) / band_rows);
  L->n_bands              = n_bands;
  for (int b = 0; b <= n_bands; ++b) L->band_row.push_back((int32_t)std::min<int64_t>((int64_t)b * band_rows, n_str));

  // 1. segment heads
  dbuf flag = make_dbuf<uint8_t>(nnz, h.stream);
  CUDA_TRY(cudaMemsetAsync(flag.data(), 0, nnz, h.stream));
  B200_LAUNCH(h, (k_hot_row_starts<O>), grid_for(n_str), kBlock, 0, c.offsets.as<O>(), n_str, flag.as<uint8_t>());
  B200_LAUNCH(h, k_hot_heads, std::min(grid_for(nnz, 4), h.sm_count * 32), kBlock, 0, idx, (long long)nnz, W, flag.as<uint8_t>());
  dbuf head_pos = make_dbuf<int32_t>(nnz, h.stream);
  int64_t n_segs64;
  {
    dbuf d_count = make_dbuf<int64_t>(1, h.stream);
    thrust::counting_iterator<int32_t> iota(0);
    size_t bytes = 0;
    CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, bytes, iota, flag.as<uint8_t>(), head_pos.as<int32_t>(), d_count.as<int64_t>(),
                                        nnz, h.stream));
    dbuf tmp(bytes, h.stream);
    CUDA_TRY(cub::DeviceSelect::Flagged(tmp.data(), bytes, iota, flag.as<uint8_t>(), head_pos.as<int32_t>(),
                                        d_count.as<int64_t>(), nnz, h.stream));
    CUDA_TRY(cudaMemcpyAsync(&n_segs64, d_count.data(), sizeof(int64_t), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
  }
  flag.release();
  const int32_t n_segs = (int32_t)n_segs64;
  tr.mark("sweep layout: segment heads");

  // 2. pieces
  dbuf seg_row = make_dbuf<int32_t>(n_segs, h.stream), seg_pieces = make_dbuf<int32_t>((size_t)n_segs + 1, h.stream);
  dbuf piece_off = make_dbuf<int32_t>((size_t)n_segs + 1, h.stream);
  B200_LAUNCH(h, (k_hot_segment_info<O>), grid_for((int64_t)n_segs + 1), kBlock, 0, head_pos.as<int32_t>(), n_segs,
              (long long)nnz, c.offsets.as<O>(), n_str, seg_row.as<int32_t>(), seg_pieces.as<int32_t>());
  exclusive_scan_i32(h, seg_pieces.as<int32_t>(), piece_off.as<int32_t>(), (int64_t)n_segs + 1);
  int32_t n_pieces = 0;
  CUDA_TRY(cudaMemcpyAsync(&n_pieces, piece_off.as<int32_t>() + n_segs, sizeof(int32_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  seg_pieces.release();
  L->n_pieces = n_pieces;
  dbuf piece_key = make_dbuf<uint32_t>(n_pieces, h.stream), piece_key2 = make_dbuf<uint32_t>(n_pieces, h.stream);
  dbuf piece_start = make_dbuf<int32_t>(n_pieces, h.stream), piece_len = make_dbuf<int32_t>(n_pieces, h.stream);
  dbuf piece_row = make_dbuf<int32_t>(n_pieces, h.stream);
  B200_LAUNCH(h, k_hot_emit_pieces, grid_for(n_segs), kBlock, 0, head_pos.as<int32_t>(), n_segs, (long long)nnz, idx, W, B,
              band_rows, seg_row.as<int32_t>(), piece_off.as<int32_t>(), piece_key.as<uint32_t>(), piece_start.as<int32_t>(),
              piece_len.as<int32_t>(), piece_row.as<int32_t>());
  head_pos.release();
  seg_row.release();
  piece_off.release();
  tr.mark("sweep layout: pieces");

  // 3. order pieces by (band, block, kind)
  const int n_keys = n_bands * B * kNumKinds;
  dbuf perm = make_dbuf<uint32_t>(n_pieces, h.stream), perm2 = make_dbuf<uint32_t>(n_pieces, h.stream);
  B200_LAUNCH(h, k_iota64, grid_for(n_pieces, 4), kBlock, 0, (int64_t)n_pieces, perm.as<uint32_t>());
  sort_pairs<uint32_t, uint32_t>(h, piece_key.as<uint32_t>(), piece_key2.as<uint32_t>(), perm.as<uint32_t>(),
                                 perm2.as<uint32_t>(), n_pieces, 0, bits_for(n_keys + 1));
  dbuf class_start = make_dbuf<int32_t>((size_t)n_keys + 1, h.stream);
  B200_LAUNCH(h, k_hot_class_starts, grid_for(n_keys + 1), kBlock, 0, piece_key2.as<uint32_t>(), n_pieces, n_keys,
              class_start.as<int32_t>());
  std::vector<int32_t> cstart((size_t)n_keys + 1);
  CUDA_TRY(cudaMemcpyAsync(cstart.data(), class_start.data(), sizeof(int32_t) * cstart.size(), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  piece_key.release();
  piece_key2.release();
  perm.release();
  tr.mark("sweep layout: kind sort");
  if (tr.on) {  // layout statistics: pieces by kind, per range of blocks
    int edges[] = {0, 1, 4, 16, 64, 160, B};
    std::fprintf(stderr, "[sweep] B=%d W=%d rows=%d (tail %d rows, %lld edges) nnz=%lld segments=%d pieces=%d bands=%d of %d rows\n",
                 B, W, n_str, n_cov - n_str, (long long)(c.nnz - nnz), (long long)nnz, n_segs, n_pieces, n_bands, band_rows);
    for (int k = 0; k + 1 < 7; ++k) {
      const int b0 = std::min(edges[k], B), b1 = std::min(edges[k + 1], B);
      if (b1 <= b0) continue;
      std::fprintf(stderr, "[sweep] blocks [%d,%d) pieces by kind S Q H F1..F8:", b0, b1);
      for (int kind = 0; kind < kNumKinds; ++kind) {
        long long np = 0;
        for (int band = 0; band < n_bands; ++band)
          for (int b = b0; b < b1; ++b) np += cstart[(band * B + b) * kNumKinds + kind + 1] - cstart[(band * B + b) * kNumKinds + kind];
        std::fprintf(stderr, " %lld", np);
      }
      std::fprintf(stderr, "\n");
    }
  }

  // 4. chunks, CTA ranges, phases
  sweep_plan_t plan;
  if (!plan_sweep(cstart, n_bands, B, h.sm_count, plan)) return nullptr;  // step-row numbers overflow 31 bits
  L->band_phase = plan.band_phase;
  L->n_steprows = plan.n_steprows;
  L->n_rowslots = plan.n_rowslots;
  L->n_chunks   = (int32_t)plan.chunks.size();
  L->n_phases   = (int32_t)plan.phases.size();
  L->n_cta      = plan.n_cta;
  L->chunks     = make_dbuf<sweep_chunk_t>(std::max<size_t>(plan.chunks.size(), 1), h.stream);
  L->phases     = make_dbuf<sweep_phase_t>(std::max<size_t>(plan.phases.size(), 1), h.stream);
  L->cta_phase  = make_dbuf<int32_t>(plan.cta_phase.size(), h.stream);
  dbuf d_fills  = make_dbuf<sweep_fill_t>(std::max<size_t>(plan.fills.size(), 1), h.stream);
  if (!plan.chunks.empty()) {
    CUDA_TRY(cudaMemcpyAsync(L->chunks.data(), plan.chunks.data(), sizeof(sweep_chunk_t) * plan.chunks.size(), cudaMemcpyHostToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(L->phases.data(), plan.phases.data(), sizeof(sweep_phase_t) * plan.phases.size(), cudaMemcpyHostToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(d_fills.data(), plan.fills.data(), sizeof(sweep_fill_t) * plan.fills.size(), cudaMemcpyHostToDevice, h.stream));
  }
  CUDA_TRY(cudaMemcpyAsync(L->cta_phase.data(), plan.cta_phase.data(), sizeof(int32_t) * plan.cta_phase.size(), cudaMemcpyHostToDevice, h.stream));
  sync(h);  // the host vectors are pageable
  L->cursor = make_dbuf<int>(L->n_phases + 1, h.stream);  // the last one: the tail's
  CUDA_TRY(cudaMemsetAsync(L->cursor.data(), 0, sizeof(int) * (L->n_phases + 1), h.stream));

  // 5. step-rows and row slots
  L->ids  = make_dbuf<uint4>((size_t)std::max<int64_t>(L->n_steprows, 1) * 32, h.stream);
  L->rows = make_dbuf<int32_t>(std::max<int64_t>(L->n_rowslots, 1), h.stream);
  const bool weighted = c.weights.data() != nullptr;
  if (weighted) L->w = dbuf((size_t)std::max<int64_t>(L->n_steprows, 1) * 32 * kHotSlot * es, h.stream);
  L->bank_order = h.tune.sweep_bank_order && es == 4;  // a double spans two banks
  if (!plan.chunks.empty()) {
    const int grid = (int)plan.chunks.size();
    if (es == 4 && L->bank_order)
      B200_LAUNCH(h, (k_sweep_fill<float, true>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<float>(), W, L->ids.as<uint4>(), L->w.as<float>(), L->rows.as<int32_t>());
    else if (es == 4)
      B200_LAUNCH(h, (k_sweep_fill<float, false>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<float>(), W, L->ids.as<uint4>(), L->w.as<float>(), L->rows.as<int32_t>());
    else
      B200_LAUNCH(h, (k_sweep_fill<double, false>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<double>(), W, L->ids.as<uint4>(), L->w.as<double>(), L->rows.as<int32_t>());
  }
  check_last("sweep layout");
  sync(h);
  tr.mark("sweep layout: fill");
  if (n_str < n_cov) {
    build_tail_layout<O>(h, c, nv, es, *L);
    tr.mark("sweep layout: tail");
    if (tr.on) {
      std::fprintf(stderr, "[sweep] tail: %d runs, %d tiles, %d units, %.1f MB of ids\n", L->n_tail_runs,
                   L->tail_runs.back().first_tile, L->tail_runs.back().first_unit, (double)L->tail_runs.back().id_off * 4 / 1e6);
    }
  }
  if (tr.on) {
    std::fprintf(stderr, "[sweep] %lld step-rows = %.1f MB of ids, %lld row slots = %.1f MB, %d chunks, %d phases, %d CTAs\n",
                 (long long)L->n_steprows, (double)L->n_steprows * 512 / 1e6, (long long)L->n_rowslots,
                 (double)L->n_rowslots * 4 / 1e6, L->n_chunks, L->n_phases, L->n_cta);
    for (int band = 0; band < n_bands; ++band) {  // slice loads: a CTA loads a block's slice once per phase
      const int p0 = plan.band_phase[band], p1 = plan.band_phase[band + 1];
      const int c0 = p1 > p0 ? plan.phases[p0].chunk_begin : 0, c1 = p1 > p0 ? plan.phases[p1 - 1].chunk_end : 0;
      std::fprintf(stderr, "[sweep] band %d rows [%d,%d): %d pieces, %d chunks, %d phases = slice loads\n", band,
                   L->band_row[band], L->band_row[band + 1], cstart[(band + 1) * B * kNumKinds] - cstart[band * B * kNumKinds],
                   c1 - c0, p1 - p0);
    }
  }
  return L;
}

}  // namespace

// flat copy of plan_sweep's result for the debug C entries (CPU tests)
bool debug_plan_sweep(std::vector<int32_t> const& cstart, int n_bands, int B, int sm_count, int64_t totals[3],
                      std::vector<int32_t>& chunks4, std::vector<int32_t>& fills4, std::vector<int32_t>& phases4,
                      std::vector<int32_t>& cta_phase, std::vector<int32_t>& band_phase)
{
  sweep_plan_t P;
  if (!plan_sweep(cstart, n_bands, B, sm_count, P)) return false;
  totals[0] = P.n_steprows; totals[1] = P.n_rowslots; totals[2] = P.n_cta;
  for (auto const& x : P.chunks) chunks4.insert(chunks4.end(), {x.sr_begin, x.row_begin, x.n_groups, x.kind});
  for (auto const& x : P.fills) fills4.insert(fills4.end(), {x.piece_begin, x.piece_end, x.block, x.pad});
  for (auto const& x : P.phases) phases4.insert(phases4.end(), {x.block, x.chunk_begin, x.chunk_end, x.pad});
  cta_phase  = P.cta_phase;
  band_phase = P.band_phase;
  return true;
}

sweep_layout_t const* sweep_layout(handle_impl const& h, csx_t const& c, int32_t n_vertices, size_t elem_size)
{
  auto& slot  = (elem_size == 4) ? c.hot4 : c.hot8;
  auto& tried = (elem_size == 4) ? c.hot4_tried : c.hot8_tried;
  if (tried) return slot.get();
  tried = true;
  // 32-bit edge positions / step-row numbers; build_sweep_layout itself gives up (nullptr) if the step-rows overflow
  if (!c.degree_sorted || c.seg[kNumSeg - 2] <= 0 || c.nnz < h.tune.sweep_min_edges || c.offs64 || c.nnz >= (1ll << 31) - 4096)
    return nullptr;
  slot = build_sweep_layout<int32_t>(h, c, n_vertices, elem_size);
  return slot.get();
}

// ---------------------------------------------------------------------------------------------
// id translation
// ---------------------------------------------------------------------------------------------
void ext_to_int(handle_impl const& h, graph_impl const& g, void const* ext, size_t n, int32_t* out)
{
  if (n == 0) return;
  dbuf rank = make_dbuf<int32_t>(n, h.stream);
  int grid  = grid_for((int64_t)n, 2);
  if (g.vertex_type == INT32) {
    if (g.renumbered)
      B200_LAUNCH(h, (k_rank_search<int32_t>), grid, kBlock, 0, (int32_t const*)ext, (int64_t)n,
                  g.sorted_ext.as<int32_t>(), g.n_vertices, rank.as<int32_t>());
    else
      B200_LAUNCH(h, (k_rank_identity<int32_t>), grid, kBlock, 0, (int32_t const*)ext, (int64_t)n, g.n_vertices,
                  rank.as<int32_t>());
  } else {
    if (g.renumbered)
      B200_LAUNCH(h, (k_rank_search<int64_t>), grid, kBlock, 0, (int64_t const*)ext, (int64_t)n,
                  g.sorted_ext.as<int64_t>(), g.n_vertices, rank.as<int32_t>());
    else
      B200_LAUNCH(h, (k_rank_identity<int64_t>), grid, kBlock, 0, (int64_t const*)ext, (int64_t)n, g.n_vertices,
                  rank.as<int32_t>());
  }
  B200_LAUNCH(h, k_compose, grid, kBlock, 0, rank.as<int32_t>(), (int64_t)n, g.int_of_rank.as<int32_t>(), out);
  check_last("ext_to_int");
}

void int_to_ext(handle_impl const& h, graph_impl const& g, int32_t const* in, size_t n, void* ext_out)
{
  if (n == 0) return;
  int grid = grid_for((int64_t)n, 2);
  if (g.vertex_type == INT32)
    B200_LAUNCH(h, (k_int_to_ext<int32_t>), grid, kBlock, 0, in, (int64_t)n, g.ext_of_int.as<int32_t>(), (int32_t*)ext_out);
  else
    B200_LAUNCH(h, (k_int_to_ext<int64_t>), grid, kBlock, 0, in, (int64_t)n, g.ext_of_int.as<int64_t>(), (int64_t*)ext_out);
  check_last("int_to_ext");
}

dbuf reported_vertices(handle_impl const& h, graph_impl const& g)
{
  size_t es = dtype_size(g.vertex_type);
  dbuf out((size_t)g.n_vertices * es, h.stream);
  if (g.n_vertices == 0) return out;
  if (g.renumbered) {
    CUDA_TRY(cudaMemcpyAsync(out.data(), g.ext_of_int.data(), (size_t)g.n_vertices * es, cudaMemcpyDeviceToDevice, h.stream));
  } else if (g.vertex_type == INT32) {
    B200_LAUNCH(h, (k_iota_t<int32_t>), grid_for(g.n_vertices), kBlock, 0, g.n_vertices, out.as<int32_t>());
  } else {
    B200_LAUNCH(h, (k_iota_t<int64_t>), grid_for(g.n_vertices), kBlock, 0, g.n_vertices, out.as<int64_t>());
  }
  return out;
}

dbuf to_reported_order(handle_impl const& h, graph_impl const& g, void const* vals, size_t es)
{
  dbuf out((size_t)g.n_vertices * es, h.stream);
  if (g.n_vertices == 0) return out;
  if (g.renumbered) {
    CUDA_TRY(cudaMemcpyAsync(out.data(), vals, (size_t)g.n_vertices * es, cudaMemcpyDeviceToDevice, h.stream));
  } else if (es == 4) {
    B200_LAUNCH(h, (k_permute<uint32_t>), grid_for(g.n_vertices), kBlock, 0, (uint32_t const*)vals,
                g.int_of_rank.as<int32_t>(), g.n_vertices, out.as<uint32_t>());
  } else {
    B200_LAUNCH(h, (k_permute<uint64_t>), grid_for(g.n_vertices), kBlock, 0, (uint64_t const*)vals,
                g.int_of_rank.as<int32_t>(), g.n_vertices, out.as<uint64_t>());
  }
  return out;
}

template <typename T>
dbuf collect_vertex_values(handle_impl const& h, graph_impl const& g, device_array_view_impl const* verts,
                           device_array_view_impl const* vals, T fill)
{
  B200_EXPECTS(verts->size == vals->size, CUGRAPH_INVALID_INPUT, "vertex and value arrays differ in size");
  dbuf out = make_dbuf<T>(std::max(g.n_vertices, 1), h.stream);
  B200_LAUNCH(h, (k_fill<T>), grid_for(g.n_vertices), kBlock, 0, out.as<T>(), (int64_t)g.n_vertices, fill);
  if (verts->size == 0) return out;
  dbuf idx = make_dbuf<int32_t>(verts->size, h.stream);
  ext_to_int(h, g, verts->data, verts->size, idx.as<int32_t>());
  dbuf bad = make_dbuf<int>(1, h.stream);
  CUDA_TRY(cudaMemsetAsync(bad.data(), 0, sizeof(int), h.stream));
  B200_LAUNCH(h, (k_scatter_values<T>), grid_for((int64_t)verts->size), kBlock, 0, idx.as<int32_t>(), (T const*)vals->data,
              (int64_t)verts->size, out.as<T>(), bad.as<int>());
  int hbad = 0;
  CUDA_TRY(cudaMemcpyAsync(&hbad, bad.data(), sizeof(int), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  B200_EXPECTS(hbad == 0, CUGRAPH_INVALID_INPUT, "vertex list contains ids that are not vertices of the graph");
  return out;
}

template dbuf collect_vertex_values<float>(handle_impl const&, graph_impl const&, device_array_view_impl const*,
                                           device_array_view_impl const*, float);
template dbuf collect_vertex_values<double>(handle_impl const&, graph_impl const&, device_array_view_impl const*,
                                            device_array_view_impl const*, double);

}  // namespace b200

extern "C" cugraph_error_code_t cugraph_b200_debug_plan_sweep_bands(const int32_t* class_start, int n_bands, int n_blocks,
                                                                    int sm_count, int64_t* totals, int32_t* chunks,
                                                                    int32_t* fills, size_t chunks_capacity, size_t* n_chunks,
                                                                    int32_t* phases, size_t phases_capacity, size_t* n_phases,
                                                                    int32_t* cta_phase, size_t cta_capacity,
                                                                    int32_t* band_phase, cugraph_error_t** error)
{
  using namespace b200;
  return guarded(error, [&] {
    B200_EXPECTS(class_start && totals && chunks && fills && phases && cta_phase && band_phase && n_chunks && n_phases,
                 CUGRAPH_INVALID_INPUT, "null argument");
    B200_EXPECTS(n_bands >= 1 && n_blocks >= 0 && sm_count >= 1, CUGRAPH_INVALID_INPUT, "bad parameter");
    std::vector<int32_t> cstart(class_start, class_start + (size_t)n_bands * n_blocks * kNumKinds + 1);
    std::vector<int32_t> c4, f4, p4, r, bp;
    int64_t t[3];
    B200_EXPECTS(debug_plan_sweep(cstart, n_bands, n_blocks, sm_count, t, c4, f4, p4, r, bp), CUGRAPH_INVALID_INPUT,
                 "step-row numbers overflow 31 bits");
    B200_EXPECTS(c4.size() / 4 <= chunks_capacity && p4.size() / 4 <= phases_capacity && r.size() <= cta_capacity,
                 CUGRAPH_INVALID_INPUT, "output capacity too small");
    std::copy(t, t + 3, totals);
    std::copy(c4.begin(), c4.end(), chunks);
    std::copy(f4.begin(), f4.end(), fills);
    std::copy(p4.begin(), p4.end(), phases);
    std::copy(r.begin(), r.end(), cta_phase);
    std::copy(bp.begin(), bp.end(), band_phase);
    *n_chunks = c4.size() / 4;
    *n_phases = p4.size() / 4;
  });
}

extern "C" cugraph_error_code_t cugraph_b200_debug_plan_sweep(const int32_t* class_start, int n_blocks, int sm_count,
                                                              int64_t* totals, int32_t* chunks, int32_t* fills,
                                                              size_t chunks_capacity, size_t* n_chunks, int32_t* phases,
                                                              size_t phases_capacity, size_t* n_phases, int32_t* cta_phase,
                                                              size_t cta_capacity, cugraph_error_t** error)
{
  int32_t band_phase[2];
  return cugraph_b200_debug_plan_sweep_bands(class_start, 1, n_blocks, sm_count, totals, chunks, fills, chunks_capacity, n_chunks,
                                             phases, phases_capacity, n_phases, cta_phase, cta_capacity, band_phase, error);
}
