// Internal vocabulary of the H100-native libcugraph_c: error plumbing, the resource handle,
// type-erased arrays, stream-ordered device buffers.  Nothing here is exported.
#pragma once

#include <cugraph_c/b200_ext.h>
#include <cugraph_c/graph_functions.h>
#include <cugraph_c/labeling_algorithms.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>

namespace b200 {

// ---------------------------------------------------------------------------------------------
// errors: C++ exceptions inside, cugraph_error_code_t + heap message at the C boundary
// (same contract as the reference's run_algorithm wrapper, cpp/src/c_api/utils.hpp:13-47).
// ---------------------------------------------------------------------------------------------
struct error_impl {
  std::string message;
};

struct capi_exception : public std::runtime_error {
  cugraph_error_code_t code;
  capi_exception(cugraph_error_code_t c, std::string const& m) : std::runtime_error(m), code(c) {}
};

#define B200_EXPECTS(cond, code, msg)                                  \
  do {                                                                 \
    if (!(cond)) throw ::b200::capi_exception((code), std::string(msg)); \
  } while (0)

#define CUDA_TRY(call)                                                                           \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      cudaGetLastError();                                                                        \
      throw ::b200::capi_exception(                                                              \
        e__ == cudaErrorMemoryAllocation ? CUGRAPH_ALLOC_ERROR : CUGRAPH_UNKNOWN_ERROR,          \
        std::string("CUDA error ") + cudaGetErrorName(e__) + " at " + __FILE__ + ":" +           \
          std::to_string(__LINE__) + ": " + cudaGetErrorString(e__));                            \
    }                                                                                            \
  } while (0)

template <typename F>
cugraph_error_code_t guarded(cugraph_error_t** error, F&& f)
{
  if (error) *error = nullptr;
  try {
    f();
    return CUGRAPH_SUCCESS;
  } catch (capi_exception const& e) {
    if (error) *error = reinterpret_cast<cugraph_error_t*>(new error_impl{e.what()});
    return e.code;
  } catch (std::bad_alloc const&) {
    if (error) *error = reinterpret_cast<cugraph_error_t*>(new error_impl{"host allocation failed"});
    return CUGRAPH_ALLOC_ERROR;
  } catch (std::exception const& e) {
    if (error) *error = reinterpret_cast<cugraph_error_t*>(new error_impl{e.what()});
    return CUGRAPH_UNKNOWN_ERROR;
  }
}

// ---------------------------------------------------------------------------------------------
// dtype helpers
// ---------------------------------------------------------------------------------------------
inline size_t dtype_size(cugraph_data_type_id_t t)
{
  switch (t) {
    case INT8:
    case UINT8:
    case BOOL: return 1;
    case INT16:
    case UINT16: return 2;
    case INT32:
    case UINT32:
    case FLOAT32: return 4;
    case INT64:
    case UINT64:
    case FLOAT64:
    case SIZE_T: return 8;
    default: return 0;
  }
}

// ---------------------------------------------------------------------------------------------
// schedule knobs (development / tests): environment variables read ONCE, when a handle is created.  Results never
// depend on them.
// ---------------------------------------------------------------------------------------------
struct tuning_t {
  long long sweep_min_edges{1ll << 22};  // CUGRAPH_B200_SWEEP_MIN_EDGES: graphs below it use the plain sweep (tests: 0)
  bool sweep_bank_order{true};           // CUGRAPH_B200_SWEEP_BANK_ORDER
  int sweep_bands{0};                    // CUGRAPH_B200_SWEEP_BANDS: row bands of the piece stream (0: sized to the L2)
  int sweep_tail_degree{0};              // CUGRAPH_B200_SWEEP_TAIL_DEGREE: rows below this in-degree leave the piece stream
                                         // (0: the default rule, 1: no tail, 2/4/8/16/32: that bound on any graph)
  int sweep_tail_sms{-1};                // CUGRAPH_B200_SWEEP_TAIL_SMS: SMs the tail sweep gets beside the piece stream (< 0: chosen
                                         // from the layout, 0: no split, the tail after the bands on every SM)
  double bfs_alpha{40.0}, bfs_beta{24.0};  // CUGRAPH_B200_BFS_ALPHA / _BETA (Beamer switch points; alpha 14 -> 40: -7 % per source on RMAT-24, r02_notes)
  bool sssp_adaptive{true};                // CUGRAPH_B200_SSSP_ADAPTIVE
  double sssp_delta_scale{1.0};            // CUGRAPH_B200_SSSP_DELTA_SCALE
  double sssp_start_div{64.0};             // CUGRAPH_B200_SSSP_START_DIV: the controller starts with delta / this
  bool sssp_small_rounds{true};            // CUGRAPH_B200_SSSP_SMALL_ROUNDS: small near queues are relaxed round after round by one CTA
  int sssp_split_rounds{1};                // CUGRAPH_B200_SSSP_SPLIT_ROUNDS
  unsigned long long sssp_split_min_edges{1ull << 20};  // CUGRAPH_B200_SSSP_SPLIT_MIN_EDGES
  unsigned long long advance_split_edges{1ull << 31};  // CUGRAPH_B200_ADVANCE_SPLIT_EDGES: frontiers with this many edges are advanced in halves (tests lower it)
  long long offs64_min_edges{1ll << 31};  // CUGRAPH_B200_OFFS64_MIN_EDGES: a csx with this many edges stores 64-bit offsets, in [0, 2^31]
                                          // (tests: 0; lazily built views follow the handle passed to the algorithm)
  bool bfs_trace{false}, sssp_trace{false}, build_trace{false}, scc_trace{false};  // CUGRAPH_B200_{BFS,SSSP,BUILD,SCC}_TRACE
  static tuning_t from_env()
  {
    tuning_t t;
    auto get = [](const char* k) { return std::getenv(k); };
    if (auto e = get("CUGRAPH_B200_SWEEP_MIN_EDGES")) t.sweep_min_edges = std::atoll(e);
    if (auto e = get("CUGRAPH_B200_SWEEP_BANK_ORDER")) t.sweep_bank_order = std::atoi(e) != 0;
    if (auto e = get("CUGRAPH_B200_SWEEP_BANDS")) t.sweep_bands = std::max(0, std::atoi(e));
    if (auto e = get("CUGRAPH_B200_SWEEP_TAIL_DEGREE")) t.sweep_tail_degree = std::max(0, std::atoi(e));
    if (auto e = get("CUGRAPH_B200_SWEEP_TAIL_SMS")) t.sweep_tail_sms = std::atoi(e);
    if (auto e = get("CUGRAPH_B200_BFS_ALPHA")) t.bfs_alpha = std::atof(e);
    if (auto e = get("CUGRAPH_B200_BFS_BETA")) t.bfs_beta = std::atof(e);
    if (auto e = get("CUGRAPH_B200_SSSP_ADAPTIVE")) t.sssp_adaptive = std::atoi(e) != 0;
    if (auto e = get("CUGRAPH_B200_SSSP_DELTA_SCALE")) t.sssp_delta_scale = std::atof(e);
    if (auto e = get("CUGRAPH_B200_SSSP_START_DIV")) t.sssp_start_div = std::max(1.0, std::atof(e));
    if (auto e = get("CUGRAPH_B200_SSSP_SMALL_ROUNDS")) t.sssp_small_rounds = std::atoi(e) != 0;
    if (auto e = get("CUGRAPH_B200_SSSP_SPLIT_ROUNDS")) t.sssp_split_rounds = std::max(1, std::atoi(e));
    if (auto e = get("CUGRAPH_B200_SSSP_SPLIT_MIN_EDGES")) t.sssp_split_min_edges = std::strtoull(e, nullptr, 10);
    if (auto e = get("CUGRAPH_B200_ADVANCE_SPLIT_EDGES")) t.advance_split_edges = std::min<unsigned long long>(std::max<unsigned long long>(std::strtoull(e, nullptr, 10), 2ull), 1ull << 31);
    if (auto e = get("CUGRAPH_B200_OFFS64_MIN_EDGES")) t.offs64_min_edges = std::min(std::max(std::atoll(e), 0ll), 1ll << 31);
    t.bfs_trace   = get("CUGRAPH_B200_BFS_TRACE") != nullptr;
    t.sssp_trace  = get("CUGRAPH_B200_SSSP_TRACE") != nullptr;
    t.build_trace = get("CUGRAPH_B200_BUILD_TRACE") != nullptr;
    t.scc_trace   = get("CUGRAPH_B200_SCC_TRACE") != nullptr;
    return t;
  }
};

// ---------------------------------------------------------------------------------------------
// resource handle: one device, one stream, the device's default stream-ordered pool.  A side stream and two events let one
// kernel run beside the work of `stream` (the pull sweep's tail, sweep.cuh): forked from `stream` by `fork`, joined back
// into it by `join` before anything after it is enqueued, so everything outside that fork is ordered on `stream` alone.
// ---------------------------------------------------------------------------------------------
struct handle_impl {
  tuning_t tune{};
  int device{0};
  cudaStream_t stream{nullptr};
  bool borrowed_stream{false};  // stream belongs to the caller (torch): never destroyed here
  cudaStream_t side{nullptr};   // the handle's own, borrowed stream or not
  cudaEvent_t fork{nullptr}, join{nullptr};
  int sm_count{132};
  size_t l2_bytes{0};
  mutable size_t launches{0};
  void* pinned{nullptr};  // 4 KiB pinned host scratch for scalar read-backs
};

inline handle_impl const& H(const cugraph_resource_handle_t* h)
{
  B200_EXPECTS(h != nullptr, CUGRAPH_INVALID_HANDLE, "resource handle is NULL");
  return *reinterpret_cast<handle_impl const*>(h);
}

// Beamer's direction switch of a direction-optimising BFS level (the reference: bfs_impl.cuh:291-297), with the handle's
// CUGRAPH_B200_BFS_ALPHA / _BETA.  n_f, m_f: vertices and out-edges of the current frontier; prev_n_f: vertices of the
// previous one (0 at the first level); m_u: edges into the unvisited vertices; n_unvisited: vertices not visited yet.
// Returns the direction of this level (true = bottom-up), given that of the last one.  Single-GPU BFS (run_bfs) and
// multi-GPU BFS (cugraph_b200_bfs_bottom_up) both decide with it.
inline bool bfs_bottom_up(handle_impl const& h, bool bottom_up, long long n_f, long long prev_n_f, unsigned long long m_f,
                          unsigned long long m_u, long long n_unvisited)
{
  if (!bottom_up && (double)m_f * h.tune.bfs_alpha > (double)m_u && n_f >= prev_n_f) return true;
  if (bottom_up && (double)n_f * h.tune.bfs_beta < (double)n_unvisited && n_f < prev_n_f) return false;
  return bottom_up;
}

// streams of live handles: buffers that outlive their handle (graphs, results) are freed
// synchronously instead of on a destroyed stream (capi_basic.cu)
bool stream_is_live(cudaStream_t s);
void register_stream(cudaStream_t s);
void unregister_stream(cudaStream_t s);

// Blocks behind dbuf (capi_basic.cu).  A freed block stays with its stream and serves the next request of (about) its
// size on that stream — stream order makes that safe exactly like cudaFreeAsync / cudaMallocAsync — so that a repeated
// workload (graph after graph of the same shape) makes no allocator calls at all: with the driver's pool alone identical
// staging steps took between milliseconds and seconds depending on what the pool had to map.  The cache of
// a stream is bounded (32 GiB, then handed back to the pool) and is released when the stream's handle is destroyed.
void* block_alloc(size_t bytes, cudaStream_t s, size_t* capacity);
void block_free(void* p, size_t capacity, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// stream-ordered owning device buffer (the rmm::device_buffer role)
// ---------------------------------------------------------------------------------------------
class dbuf {
 public:
  dbuf() = default;
  dbuf(size_t bytes, cudaStream_t s) : bytes_(bytes), stream_(s)
  {
    if (bytes_ > 0) p_ = block_alloc(bytes_, s, &cap_);
  }
  dbuf(dbuf const&)            = delete;
  dbuf& operator=(dbuf const&) = delete;
  dbuf(dbuf&& o) noexcept { swap(o); }
  dbuf& operator=(dbuf&& o) noexcept
  {
    if (this != &o) {
      release();
      swap(o);
    }
    return *this;
  }
  ~dbuf() { release(); }
  void release()
  {
    if (p_) block_free(p_, cap_, stream_);
    p_     = nullptr;
    bytes_ = cap_ = 0;
  }
  void* data() const { return p_; }
  template <typename T>
  T* as() const
  {
    return reinterpret_cast<T*>(p_);
  }
  size_t bytes() const { return bytes_; }
  cudaStream_t stream() const { return stream_; }

 private:
  void swap(dbuf& o)
  {
    std::swap(p_, o.p_);
    std::swap(bytes_, o.bytes_);
    std::swap(cap_, o.cap_);
    std::swap(stream_, o.stream_);
  }
  void* p_{nullptr};
  size_t bytes_{0};
  size_t cap_{0};  // what the block really holds (a reused block may be a little larger than asked for)
  cudaStream_t stream_{nullptr};
};

template <typename T>
inline dbuf make_dbuf(size_t n, cudaStream_t s)
{
  return dbuf(n * sizeof(T), s);
}

// ---------------------------------------------------------------------------------------------
// type-erased arrays (reference cpp/src/c_api/array.hpp:17-97)
// ---------------------------------------------------------------------------------------------
struct device_array_view_impl {
  void* data{nullptr};
  size_t size{0};
  cugraph_data_type_id_t type{INT32};
  size_t nbytes() const { return size * dtype_size(type); }
};

struct device_array_impl {
  dbuf buf;
  size_t size{0};
  cugraph_data_type_id_t type{INT32};
  device_array_view_impl* new_view() const { return new device_array_view_impl{buf.data(), size, type}; }
};

struct host_array_view_impl {
  void* data{nullptr};
  size_t size{0};
  cugraph_data_type_id_t type{INT32};
  size_t nbytes() const { return size * dtype_size(type); }
};

struct host_array_impl {
  void* data{nullptr};
  size_t size{0};
  cugraph_data_type_id_t type{INT32};
};

inline device_array_view_impl const* V(const cugraph_type_erased_device_array_view_t* v)
{
  return reinterpret_cast<device_array_view_impl const*>(v);
}

inline cugraph_type_erased_device_array_t* wrap_array(dbuf&& b, size_t n, cugraph_data_type_id_t t)
{
  auto* a = new device_array_impl{std::move(b), n, t};
  return reinterpret_cast<cugraph_type_erased_device_array_t*>(a);
}

// result objects (reference cpp/src/c_api/centrality_result.hpp:14-19, paths_result.hpp:12-16, labeling_result.hpp)
struct centrality_result_impl {
  device_array_impl* vertices{nullptr};
  device_array_impl* values{nullptr};
  size_t iterations{0};
  bool converged{false};
};

struct paths_result_impl {
  device_array_impl* vertices{nullptr};
  device_array_impl* distances{nullptr};
  device_array_impl* predecessors{nullptr};
};

// weakly / strongly connected components (components.cu, scc.cu)
struct labeling_result_impl {
  device_array_impl* vertices{nullptr};
  device_array_impl* labels{nullptr};
};

// ---------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------
constexpr int kBlock = 256;  // threads per CTA of the element-wise kernels

// CTAs of kBlock threads for n elements, per_thread elements each: at least one, never more than 2^20, and at most max_grid
// (usually a multiple of h.sm_count) for kernels that gain nothing from more.  A kernel launched on such a grid strides over it.
inline int grid_for(int64_t n, int per_thread = 1, int max_grid = 1 << 20)
{
  const int64_t b = (n + (int64_t)kBlock * per_thread - 1) / ((int64_t)kBlock * per_thread);
  return (int)std::min<int64_t>(std::max<int64_t>(b, 1), std::min(max_grid, 1 << 20));
}

// B200_LAUNCH_ON: on stream s of handle h (its stream or its side stream), counted like every launch
#ifndef B200_HOST_EMU
#define B200_LAUNCH_ON(h, s, kernel, grid, block, smem, ...)                     \
  do {                                                                           \
    if ((grid) > 0) {                                                            \
      kernel<<<(grid), (block), (smem), (s)>>>(__VA_ARGS__);                     \
      (h).launches++;                                                            \
    }                                                                            \
  } while (0)
// the lane of a warp that commits a warp-reduced value
__device__ __forceinline__ bool is_commit_lane() { return (threadIdx.x & 31) == 0; }
#else
// host emulation of the staging kernels (emu/cuda_runtime.h, tests/test_emu_staging_cpu.py): every thread of the
// launch runs to completion, one after the other; warp shuffles are identities, so every thread commits for itself.  Streams
// are in order here: a launch on the side stream runs where it is enqueued
#define B200_LAUNCH_ON(h, s, kernel, grid, block, smem, ...)                     \
  do {                                                                           \
    if ((grid) > 0) {                                                            \
      (void)(s);                                                                 \
      emu_launch((grid), (block), (size_t)(smem), [&] { kernel(__VA_ARGS__); }); \
      (h).launches++;                                                            \
    }                                                                            \
  } while (0)
inline bool is_commit_lane() { return true; }
#endif
#define B200_LAUNCH(h, kernel, grid, block, smem, ...) B200_LAUNCH_ON(h, (h).stream, kernel, grid, block, smem, __VA_ARGS__)

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

inline void check_last(const char* what)
{
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    throw capi_exception(CUGRAPH_UNKNOWN_ERROR,
                         std::string("kernel launch failed (") + what + "): " + cudaGetErrorString(e));
}

inline void sync(handle_impl const& h) { CUDA_TRY(cudaStreamSynchronize(h.stream)); }

// the value at d, once the work enqueued before it on the handle's stream has finished
template <typename T>
T read_back(handle_impl const& h, T const* d)
{
  T v{};
  CUDA_TRY(cudaMemcpyAsync(&v, d, sizeof(T), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  return v;
}

// Element-wise kernels shared by the translation units.  A __global__ template instantiated in several of them is only
// safe with internal linkage, so every translation unit gets its own copy.
namespace {

template <typename T>
__global__ void k_fill(T* __restrict__ a, int64_t n, T v)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = v;
}

template <typename T>
__global__ void k_iota(T* __restrict__ a, int64_t n)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = (T)i;
}

// *out += number of elements below 0
template <typename T>
__global__ void k_count_negative(T const* __restrict__ a, int64_t n, int* __restrict__ out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (a[i] < (T)0) atomicAdd(out, 1);
}

// the sum of v over the CTA, valid in warp 0; smem holds one double per warp
__device__ __forceinline__ double block_sum(double v, double* smem)
{
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x < 32) {
    t = (threadIdx.x < (blockDim.x >> 5)) ? smem[threadIdx.x] : 0.0;
    t = warp_sum(t);
  }
  __syncthreads();
  return t;
}

}  // namespace

// CUGRAPH_B200_BUILD_TRACE=1: print the time of every staging phase (stream-synchronised) to stderr
struct phase_trace {
  handle_impl const& h;
  bool on;
  cudaEvent_t e0{}, e1{};
  explicit phase_trace(handle_impl const& hh) : h(hh), on(hh.tune.build_trace)
  {
    if (on) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
      cudaEventRecord(e0, h.stream);
    }
  }
  void mark(const char* what)
  {
    if (!on) return;
    cudaEventRecord(e1, h.stream);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    std::fprintf(stderr, "[build] %-28s %8.3f ms\n", what, ms);
    std::swap(e0, e1);
  }
  ~phase_trace()
  {
    if (on) {
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
    }
  }
};


}  // namespace b200
