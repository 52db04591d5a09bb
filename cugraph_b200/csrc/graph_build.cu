// Graph staging on the GPU: edge list (external ids) -> degree-ordered internal ids -> compressed
// rows with sorted neighbours + the bin / chunk metadata the hot-path kernels consume.
// Replaces (behaviourally) cpp/src/c_api/graph_sg.cpp:89-330 -> create_graph_from_edgelist
// (cpp/src/structure/create_graph_from_edgelist_impl.cuh:1430-1688) -> renumber_edgelist
// (renumber_edgelist_impl.cuh:419-833).  Staging is one-time and untimed; device-wide sorts and
// scans use CUB (library code), everything else is hand-written.  The pull sweep's own layout of a csx
// (the piece stream) is built by sweep_layout.cu.
#include "graph.cuh"
#include "staging.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace b200 {

namespace {

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
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x)
    keys[i] = ((uint64_t)(0x7fffffffu - (uint32_t)deg[i]) << 32) | (uint32_t)i;
}

__global__ void k_perm_from_keys(uint64_t const* keys, int32_t nv, int32_t* rank_of_int, int32_t* int_of_rank)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t r      = (int32_t)(keys[i] & 0xffffffffu);
    rank_of_int[i] = r;
    int_of_rank[r] = (int32_t)i;
  }
}

template <typename T>
__global__ void k_gather_ext(T const* sorted_ext, int32_t const* rank_of_int, int32_t nv, T* ext_of_int)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x)
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
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r + 1 < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
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
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[perm[i]];
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

// ---------------------------------------------------------------- CUB wrappers (sort_keys: staging.cuh)
template <typename T>
int64_t unique_sorted(handle_impl const& h, T const* in, T* out, int64_t n)
{
  dbuf d_count(sizeof(int64_t), h.stream);
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceSelect::Unique(nullptr, bytes, in, out, d_count.as<int64_t>(), n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceSelect::Unique(tmp.data(), bytes, in, out, d_count.as<int64_t>(), n, h.stream));
  h.launches += 2;
  return read_back(h, d_count.as<int64_t>());
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
    B200_LAUNCH(h, k_iota<uint32_t>, grid_for(n, 4), kBlock, 0, perm.as<uint32_t>(), n);
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
  c.nnz_hi   = c.seg[0] > 0 ? (int64_t)read_back(h, off + c.seg[0]) : 0;
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
  const int32_t n_split = read_back(h, scan.as<int32_t>() + c.n_chunks);
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
    B200_LAUNCH(h, (k_minmax<VT>), grid_for(n, 8, 2048), kBlock, 0, src, n, mm.as<long long>(), mm.as<long long>() + 1);
    B200_LAUNCH(h, (k_minmax<VT>), grid_for(n, 8, 2048), kBlock, 0, dst, n, mm.as<long long>(), mm.as<long long>() + 1);
  }
  if (n_verts > 0)
    B200_LAUNCH(h, (k_minmax<VT>), grid_for(n_verts, 8, 2048), kBlock, 0, verts, n_verts, mm.as<long long>(),
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
    const int32_t nv = read_back(h, rank.as<int32_t>() + m);
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
    B200_LAUNCH(h, k_iota<uint32_t>, grid_for(n, 4), kBlock, 0, perm.as<uint32_t>(), n);
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
  const int32_t m = read_back(h, scan.as<int32_t>() + n);
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
// staging of one multi-GPU edge block.  Edge u -> v sits at position (row = slot of v, col = slot of u); with symmetrize the
// caller has also shuffled a reversed copy (flag 1) of every non-self-loop edge v -> u to that position, so the position
// holds the whole group of the unordered pair {u, v}.  The same rules as single-GPU staging then apply locally:
// multi-edges -> the minimum weight per (row, col, flag) (weight-key sort, stable key sort, run heads, as build_csx_typed);
// symmetrize -> symmetrize_typed's pairing, the i-th lightest flag-0 edge with the i-th lightest flag-1 edge, emitting
// only the orientation stored here (the position (row = u, col = v) sees the same group from the other side and emits
// the other one, with the bit-identical averaged weight).
// ---------------------------------------------------------------------------------------------
namespace {

__global__ void k_block_stage_keys(int32_t const* rows, int32_t const* cols, uint8_t const* rev, int64_t n, int bits,
                                   uint64_t* keys)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t pos = ((uint64_t)(uint32_t)rows[i] << bits) | (uint32_t)cols[i];
    keys[i]            = (pos << 1) | (rev && rev[i] ? 1ull : 0ull);
  }
}

// keep[i] and the weight of element i of the sorted group of its position: a flag-0 edge always stays, averaged with the
// flag-1 edge of the same rank when there is one; a flag-1 edge stays when it has no flag-0 partner
template <typename W>
__global__ void k_block_pair(uint64_t const* keys, W const* w, int64_t n, uint8_t* keep, W* w_out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t pos = keys[i] >> 1;
    const int64_t r0 = lb64(keys, n, pos << 1), r1 = lb64(keys, n, (pos << 1) | 1ull), r2 = lb64(keys, n, (pos << 1) + 2ull);
    if (keys[i] & 1ull) {
      keep[i] = (i - r1) >= (r1 - r0) ? 1 : 0;
      if (w) w_out[i] = w[i];
    } else {
      const int64_t j = i - r0;
      keep[i]         = 1;
      if (w) w_out[i] = j < r2 - r1 ? (W)((w[i] + w[r1 + j]) / (W)2) : w[i];
    }
  }
}

__global__ void k_block_unpack(uint64_t const* keys, int64_t n, int bits, int32_t* rows, int32_t* cols)
{
  const uint64_t mask = (1ull << bits) - 1ull;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    rows[i] = (int32_t)(keys[i] >> (bits + 1));
    cols[i] = (int32_t)((keys[i] >> 1) & mask);
  }
}

template <typename W>
int64_t stage_block_typed(handle_impl const& h, int bits, int32_t* rows, int32_t* cols, uint8_t const* rev, W* w, int64_t n,
                          bool drop_multi_edges, bool symmetrize)
{
  const int key_bits = 2 * bits + 1;
  dbuf keys = make_dbuf<uint64_t>(n, h.stream), keys2 = make_dbuf<uint64_t>(n, h.stream);
  B200_LAUNCH(h, k_block_stage_keys, grid_for(n, 4), kBlock, 0, rows, cols, symmetrize ? rev : nullptr, n, bits,
              keys.as<uint64_t>());
  dbuf ws;  // the weights in key order
  if (w == nullptr) {
    sort_keys<uint64_t>(h, keys.as<uint64_t>(), keys2.as<uint64_t>(), n, 0, key_bits);
  } else {
    // stable two-pass: by weight first, so that every group of equal keys is in ascending weight
    B200_EXPECTS(n < (1ll << 32), CUGRAPH_INVALID_INPUT, "weighted graphs are limited to 2^32 edges per GPU");
    using U   = typename std::conditional<sizeof(W) == 4, uint32_t, uint64_t>::type;
    dbuf perm = make_dbuf<uint32_t>(n, h.stream), perm2 = make_dbuf<uint32_t>(n, h.stream);
    dbuf wk = make_dbuf<U>(n, h.stream), wk2 = make_dbuf<U>(n, h.stream);
    B200_LAUNCH(h, k_iota<uint32_t>, grid_for(n, 4), kBlock, 0, perm.as<uint32_t>(), n);
    B200_LAUNCH(h, (k_weight_keys<W, U>), grid_for(n, 4), kBlock, 0, w, n, wk.as<U>());
    sort_pairs<U, uint32_t>(h, wk.as<U>(), wk2.as<U>(), perm.as<uint32_t>(), perm2.as<uint32_t>(), n, 0, (int)sizeof(U) * 8);
    wk.release();
    wk2.release();
    B200_LAUNCH(h, (k_gather<uint64_t>), grid_for(n, 4), kBlock, 0, keys.as<uint64_t>(), perm2.as<uint32_t>(), n,
                keys2.as<uint64_t>());
    sort_pairs<uint64_t, uint32_t>(h, keys2.as<uint64_t>(), keys.as<uint64_t>(), perm2.as<uint32_t>(), perm.as<uint32_t>(), n,
                                   0, key_bits);
    std::swap(keys, keys2);
    ws = make_dbuf<W>(n, h.stream);
    B200_LAUNCH(h, (k_gather<W>), grid_for(n, 4), kBlock, 0, w, perm.as<uint32_t>(), n, ws.as<W>());
  }
  // keys2 holds the sorted keys, ws their weights; each pass below selects the flagged ones into keys / wsel, then swaps
  int64_t m = n;
  dbuf flag = make_dbuf<uint8_t>(n, h.stream);
  auto select = [&](dbuf const& wsrc) {
    const int64_t k = select_flagged<uint64_t>(h, keys2.as<uint64_t>(), flag.as<uint8_t>(), keys.as<uint64_t>(), m);
    std::swap(keys, keys2);
    if (w != nullptr) {
      dbuf wsel = make_dbuf<W>(k, h.stream);
      select_flagged<W>(h, wsrc.as<W>(), flag.as<uint8_t>(), wsel.as<W>(), m);
      ws = std::move(wsel);
    }
    m = k;
  };
  if (drop_multi_edges) {
    B200_LAUNCH(h, k_run_heads, grid_for(m, 4), kBlock, 0, keys2.as<uint64_t>(), m, flag.as<uint8_t>());
    select(ws);
  }
  if (symmetrize && m > 0) {
    dbuf wp;
    if (w != nullptr) wp = make_dbuf<W>(m, h.stream);
    B200_LAUNCH(h, (k_block_pair<W>), grid_for(m, 2), kBlock, 0, keys2.as<uint64_t>(), w ? ws.as<W>() : (W const*)nullptr, m,
                flag.as<uint8_t>(), w ? wp.as<W>() : (W*)nullptr);
    select(wp);
  }
  if (m > 0) {
    B200_LAUNCH(h, k_block_unpack, grid_for(m, 4), kBlock, 0, keys2.as<uint64_t>(), m, bits, rows, cols);
    if (w != nullptr) CUDA_TRY(cudaMemcpyAsync(w, ws.data(), m * sizeof(W), cudaMemcpyDeviceToDevice, h.stream));
  }
  check_last("stage_block_edges");
  sync(h);
  return m;
}

}  // namespace

int64_t stage_block_edges(handle_impl const& h, int32_t n_rows, int32_t n_cols, int32_t* rows, int32_t* cols,
                          uint8_t const* reversed, void* w, cugraph_data_type_id_t wtype, int64_t n, bool drop_multi_edges,
                          bool symmetrize)
{
  const int bits = bits_for(std::max<int64_t>(std::max(n_rows, n_cols), 2));
  B200_EXPECTS(2 * bits + 1 <= 64, CUGRAPH_INVALID_INPUT, "too many slots to stage");
  B200_EXPECTS(!symmetrize || 2 * n < (1ll << 31), CUGRAPH_INVALID_INPUT, "symmetrize: edge list too large for one GPU pass");
  if (n == 0) return 0;
  // every slot in range: [min, max] of the rows and of the columns in one read-back
  dbuf mm = make_dbuf<long long>(4, h.stream);
  long long init[4] = {LLONG_MAX, LLONG_MIN, LLONG_MAX, LLONG_MIN};
  CUDA_TRY(cudaMemcpyAsync(mm.data(), init, sizeof(init), cudaMemcpyHostToDevice, h.stream));
  B200_LAUNCH(h, (k_minmax<int32_t>), grid_for(n, 8, 2048), kBlock, 0, rows, n, mm.as<long long>(), mm.as<long long>() + 1);
  B200_LAUNCH(h, (k_minmax<int32_t>), grid_for(n, 8, 2048), kBlock, 0, cols, n, mm.as<long long>() + 2,
              mm.as<long long>() + 3);
  long long hmm[4];
  CUDA_TRY(cudaMemcpyAsync(hmm, mm.data(), sizeof(hmm), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  B200_EXPECTS(hmm[0] >= 0 && hmm[1] < n_rows && hmm[2] >= 0 && hmm[3] < n_cols, CUGRAPH_INVALID_INPUT,
               "edge slots out of range of the block");
  if (w == nullptr || wtype == FLOAT32)
    return stage_block_typed<float>(h, bits, rows, cols, reversed, (float*)w, n, drop_multi_edges, symmetrize);
  return stage_block_typed<double>(h, bits, rows, cols, reversed, (double*)w, n, drop_multi_edges, symmetrize);
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

// rows = destinations, indices = sources, physical row r = vertex r (the mirror image of push_view): the primary
// orientation of a CSC graph, a transpose of a CSR graph built once.  The graph's own storage is never changed.
csx_t const& in_view(handle_impl const& h, graph_impl& g)
{
  if (g.store_transposed || g.is_symmetric) return *g.primary;
  if (!g.in_alt) {
    csx_t const& p = *g.primary;  // CSR: rows = sources, indices = destinations
    dbuf maj       = expand_majors(h, p);
    auto c         = std::make_unique<csx_t>();
    build_csx(h, *c, p.indices.as<int32_t>(), maj.as<int32_t>(), g.weighted ? p.weights.data() : nullptr,
              g.weight_type, p.nnz, g.n_vertices, nullptr, nullptr, false, false);
    c->degree_sorted = false;
    for (int k = 0; k <= kNumSeg; ++k) c->seg[k] = 0;
    sync(h);
    g.in_alt = std::move(c);
  }
  return *g.in_alt;
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
    B200_LAUNCH(h, k_iota<int32_t>, grid_for(g.n_vertices), kBlock, 0, out.as<int32_t>(), (int64_t)g.n_vertices);
  } else {
    B200_LAUNCH(h, k_iota<int64_t>, grid_for(g.n_vertices), kBlock, 0, out.as<int64_t>(), (int64_t)g.n_vertices);
  }
  return out;
}

void to_reported_order_into(handle_impl const& h, graph_impl const& g, void const* vals, size_t es, void* out)
{
  if (g.n_vertices == 0) return;
  if (g.renumbered) {
    CUDA_TRY(cudaMemcpyAsync(out, vals, (size_t)g.n_vertices * es, cudaMemcpyDeviceToDevice, h.stream));
  } else if (es == 4) {
    B200_LAUNCH(h, (k_permute<uint32_t>), grid_for(g.n_vertices), kBlock, 0, (uint32_t const*)vals,
                g.int_of_rank.as<int32_t>(), g.n_vertices, (uint32_t*)out);
  } else {
    B200_LAUNCH(h, (k_permute<uint64_t>), grid_for(g.n_vertices), kBlock, 0, (uint64_t const*)vals,
                g.int_of_rank.as<int32_t>(), g.n_vertices, (uint64_t*)out);
  }
}

dbuf to_reported_order(handle_impl const& h, graph_impl const& g, void const* vals, size_t es)
{
  dbuf out((size_t)g.n_vertices * es, h.stream);
  to_reported_order_into(h, g, vals, es, out.data());
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
  B200_EXPECTS(read_back(h, bad.as<int>()) == 0, CUGRAPH_INVALID_INPUT, "vertex list contains ids that are not vertices of the graph");
  return out;
}

template dbuf collect_vertex_values<float>(handle_impl const&, graph_impl const&, device_array_view_impl const*,
                                           device_array_view_impl const*, float);
template dbuf collect_vertex_values<double>(handle_impl const&, graph_impl const&, device_array_view_impl const*,
                                            device_array_view_impl const*, double);

}  // namespace b200
