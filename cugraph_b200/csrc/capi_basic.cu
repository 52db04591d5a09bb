// C-ABI entry points that carry no graph logic: errors, resource handle, type-erased arrays.
// Boundary being replaced: cpp/src/c_api/{error,resource_handle,array}.cpp of the reference.
#include "graph.cuh"

#include <cstdlib>
#include <map>
#include <mutex>
#include <unordered_map>
#include <unordered_set>

namespace b200 {
namespace {
std::mutex g_stream_mutex;
// stream -> the number of live handles on it.  Counted: several handles may borrow one stream (every handle made on torch's
// current stream), and the stream stays live until the last of them is freed; a buffer of a stream that is no longer live
// is freed with a synchronous cudaFree, which must never happen while another handle still queues work that uses it.
std::unordered_map<cudaStream_t, int>& live_streams()
{
  static auto* s = new std::unordered_map<cudaStream_t, int>();  // leaked on purpose: used during exit
  return *s;
}
// Freed blocks per stream (see block_alloc in common.cuh).  Leaked on purpose like the stream set.
struct block_cache_t {
  std::multimap<size_t, void*> blocks;  // capacity -> block
  size_t total{0};
};
std::unordered_map<cudaStream_t, block_cache_t>& block_caches()
{
  static auto* c = new std::unordered_map<cudaStream_t, block_cache_t>();
  return *c;
}
constexpr size_t kBlockCacheCap = 32ull << 30;  // bytes kept per stream; beyond it the cache of that stream is returned to the pool

// caller holds g_stream_mutex
void flush_cache_locked(cudaStream_t s, block_cache_t& c, bool stream_alive)
{
  for (auto& b : c.blocks) {
    if (stream_alive) cudaFreeAsync(b.second, s);
    else cudaFree(b.second);
  }
  c.blocks.clear();
  c.total = 0;
}
}  // namespace

void* block_alloc(size_t bytes, cudaStream_t s, size_t* capacity)
{
  {
    std::lock_guard<std::mutex> lk(g_stream_mutex);
    auto it = block_caches().find(s);
    if (it != block_caches().end()) {
      auto b = it->second.blocks.lower_bound(bytes);
      if (b != it->second.blocks.end() && b->first <= bytes + bytes / 8 + 512) {
        void* p   = b->second;
        *capacity = b->first;
        it->second.total -= b->first;
        it->second.blocks.erase(b);
        return p;
      }
    }
  }
  void* p       = nullptr;
  cudaError_t e = cudaMallocAsync(&p, bytes, s);
  if (e != cudaSuccess) {  // give everything cached back and try once more
    (void)cudaGetLastError();
    {
      std::lock_guard<std::mutex> lk(g_stream_mutex);
      for (auto& kv : block_caches()) flush_cache_locked(kv.first, kv.second, live_streams().count(kv.first) != 0);
    }
    cudaDeviceSynchronize();
    e = cudaMallocAsync(&p, bytes, s);
  }
  CUDA_TRY(e);
  *capacity = bytes;
  return p;
}

void block_free(void* p, size_t capacity, cudaStream_t s)
{
  std::lock_guard<std::mutex> lk(g_stream_mutex);
  if (live_streams().count(s) == 0) {
    cudaFree(p);
    return;
  }
  block_cache_t& c = block_caches()[s];
  if (c.total + capacity > kBlockCacheCap) flush_cache_locked(s, c, true);
  if (capacity > kBlockCacheCap) {
    cudaFreeAsync(p, s);
    return;
  }
  c.blocks.emplace(capacity, p);
  c.total += capacity;
}

bool stream_is_live(cudaStream_t s)
{
  std::lock_guard<std::mutex> lk(g_stream_mutex);
  return live_streams().count(s) != 0;
}
void register_stream(cudaStream_t s)
{
  std::lock_guard<std::mutex> lk(g_stream_mutex);
  ++live_streams()[s];
}
void unregister_stream(cudaStream_t s)
{
  std::lock_guard<std::mutex> lk(g_stream_mutex);
  auto live = live_streams().find(s);
  if (live != live_streams().end() && --live->second > 0) return;  // another handle still works on this stream
  auto it = block_caches().find(s);
  if (it != block_caches().end()) {  // the caller synchronised the stream: the cached blocks are idle
    flush_cache_locked(s, it->second, true);
    block_caches().erase(it);
  }
  live_streams().erase(s);
}

namespace {
// releases what a handle owns; the stream must be idle and unregistered
struct handle_deleter {
  void operator()(handle_impl* h) const
  {
    if (h->pinned) cudaFreeHost(h->pinned);
    if (h->fork) cudaEventDestroy(h->fork);
    if (h->join) cudaEventDestroy(h->join);
    if (h->side) cudaStreamDestroy(h->side);
    if (h->stream && !h->borrowed_stream) cudaStreamDestroy(h->stream);
    delete h;
  }
};

// A handle on the current device.  borrowed: `stream` is the caller's, else the handle creates its own.  NULL, with the
// reason on stderr after the entry point's name, when a CUDA call fails.
cugraph_resource_handle_t* create_handle(const char* entry, cudaStream_t stream, bool borrowed)
{
  try {
    std::unique_ptr<handle_impl, handle_deleter> h(new handle_impl{});
    h->tune            = tuning_t::from_env();
    h->stream          = stream;
    h->borrowed_stream = borrowed;
    CUDA_TRY(cudaGetDevice(&h->device));
    if (!borrowed) CUDA_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&h->fork, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&h->join, cudaEventDisableTiming));
    cudaDeviceProp prop{};
    CUDA_TRY(cudaGetDeviceProperties(&prop, h->device));
    h->sm_count = prop.multiProcessorCount;
    h->l2_bytes = static_cast<size_t>(prop.l2CacheSize);
    CUDA_TRY(cudaMallocHost(&h->pinned, 4096));
    // keep freed blocks in the pool: algorithm calls allocate/free V- and E-sized scratch
    cudaMemPool_t pool;
    CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, h->device));
    uint64_t threshold = UINT64_MAX;
    CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    register_stream(h->stream);
    return reinterpret_cast<cugraph_resource_handle_t*>(h.release());
  } catch (std::exception const& e) {
    std::fprintf(stderr, "%s: %s\n", entry, e.what());
    return nullptr;
  }
}
}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

// ----------------------------------------------------------------------------- error.h:28-29
const char* cugraph_error_message(const cugraph_error_t* error)
{
  if (error == nullptr) return nullptr;
  return reinterpret_cast<error_impl const*>(error)->message.c_str();
}

void cugraph_error_free(cugraph_error_t* error)
{
  if (error != nullptr) delete reinterpret_cast<error_impl*>(error);
}

// ------------------------------------------------------------------- resource_handle.h:25-31
// NULL -> single-GPU handle on the current device.  Non-NULL (a raft handle in the reference) is refused: multi-GPU runs
// are driven by cugraph_b200.mg over handles from cugraph_b200_create_resource_handle_on_stream.
cugraph_resource_handle_t* cugraph_create_resource_handle(void* raft_handle)
{
  if (raft_handle != nullptr) {
    std::fprintf(stderr, "cugraph_create_resource_handle: multi-GPU goes through cugraph_b200.mg (torch.distributed) + the "
                         "cugraph_b200_block_* entry points\n");
    return nullptr;
  }
  return create_handle("cugraph_create_resource_handle", nullptr, false);
}

int cugraph_resource_handle_get_comm_size(const cugraph_resource_handle_t*) { return 1; }

int cugraph_resource_handle_get_rank(const cugraph_resource_handle_t*) { return 0; }

void cugraph_free_resource_handle(cugraph_resource_handle_t* handle)
{
  if (!handle) return;
  auto* h = reinterpret_cast<handle_impl*>(handle);
  cudaStreamSynchronize(h->stream);
  unregister_stream(h->stream);
  handle_deleter{}(h);
}

// ------------------------------------------------------------------------------ b200_ext.h
const char* cugraph_b200_version(void) { return "cugraph_b200 0.1 (sm_90a)"; }

cugraph_resource_handle_t* cugraph_b200_create_resource_handle_on_stream(void* cuda_stream)
{
  return create_handle("cugraph_b200_create_resource_handle_on_stream", reinterpret_cast<cudaStream_t>(cuda_stream), true);
}

void* cugraph_b200_handle_stream(const cugraph_resource_handle_t* handle)
{
  return handle ? reinterpret_cast<void*>(reinterpret_cast<handle_impl const*>(handle)->stream) : nullptr;
}

size_t cugraph_b200_handle_launch_count(const cugraph_resource_handle_t* handle)
{
  return handle ? reinterpret_cast<handle_impl const*>(handle)->launches : 0;
}

// -------------------------------------------------------------------------- array.h:43-121
cugraph_error_code_t cugraph_type_erased_device_array_create(const cugraph_resource_handle_t* handle,
                                                             size_t n_elems,
                                                             cugraph_data_type_id_t dtype,
                                                             cugraph_type_erased_device_array_t** array,
                                                             cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(array != nullptr, CUGRAPH_INVALID_INPUT, "array out-pointer is NULL");
    size_t es = dtype_size(dtype);
    B200_EXPECTS(es > 0, CUGRAPH_UNSUPPORTED_TYPE_COMBINATION, "invalid dtype");
    dbuf b(n_elems * es, h.stream);
    *array = wrap_array(std::move(b), n_elems, dtype);
  });
}

cugraph_error_code_t cugraph_type_erased_device_array_create_from_view(
  const cugraph_resource_handle_t* handle,
  const cugraph_type_erased_device_array_view_t* view,
  cugraph_type_erased_device_array_t** array,
  cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(view != nullptr && array != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* v = V(view);
    dbuf b(v->nbytes(), h.stream);
    if (v->nbytes() > 0)
      CUDA_TRY(cudaMemcpyAsync(b.data(), v->data, v->nbytes(), cudaMemcpyDeviceToDevice, h.stream));
    sync(h);
    *array = wrap_array(std::move(b), v->size, v->type);
  });
}

void cugraph_type_erased_device_array_free(cugraph_type_erased_device_array_t* p)
{
  if (p) delete reinterpret_cast<device_array_impl*>(p);
}

cugraph_type_erased_device_array_view_t* cugraph_type_erased_device_array_view(
  cugraph_type_erased_device_array_t* array)
{
  if (!array) return nullptr;
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(
    reinterpret_cast<device_array_impl*>(array)->new_view());
}

cugraph_error_code_t cugraph_type_erased_device_array_view_as_type(
  cugraph_type_erased_device_array_t* array,
  cugraph_data_type_id_t dtype,
  cugraph_type_erased_device_array_view_t** result_view,
  cugraph_error_t** error)
{
  // reinterpretation is only allowed between types of equal width (reference array.cpp)
  return guarded(error, [&] {
    B200_EXPECTS(array != nullptr && result_view != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* a = reinterpret_cast<device_array_impl*>(array);
    B200_EXPECTS(dtype_size(dtype) == dtype_size(a->type) && dtype_size(dtype) > 0,
                 CUGRAPH_INVALID_INPUT,
                 "Could not treat type_erased_device_array_t as requested type");
    *result_view = reinterpret_cast<cugraph_type_erased_device_array_view_t*>(
      new device_array_view_impl{a->buf.data(), a->size, dtype});
  });
}

// ------------------------------------------------------------------------- array.h:123-170
cugraph_type_erased_device_array_view_t* cugraph_type_erased_device_array_view_create(
  void* pointer, size_t n_elems, cugraph_data_type_id_t dtype)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(
    new device_array_view_impl{pointer, n_elems, dtype});
}

void cugraph_type_erased_device_array_view_free(cugraph_type_erased_device_array_view_t* p)
{
  if (p) delete reinterpret_cast<device_array_view_impl*>(p);
}

size_t cugraph_type_erased_device_array_view_size(const cugraph_type_erased_device_array_view_t* p)
{
  return p ? V(p)->size : 0;
}

cugraph_data_type_id_t cugraph_type_erased_device_array_view_type(
  const cugraph_type_erased_device_array_view_t* p)
{
  return p ? V(p)->type : NTYPES;
}

const void* cugraph_type_erased_device_array_view_pointer(const cugraph_type_erased_device_array_view_t* p)
{
  return p ? V(p)->data : nullptr;
}

// ------------------------------------------------------------------------- array.h:172-262
cugraph_error_code_t cugraph_type_erased_host_array_create(const cugraph_resource_handle_t* handle,
                                                           size_t n_elems,
                                                           cugraph_data_type_id_t dtype,
                                                           cugraph_type_erased_host_array_t** array,
                                                           cugraph_error_t** error)
{
  return guarded(error, [&] {
    (void)H(handle);
    B200_EXPECTS(array != nullptr, CUGRAPH_INVALID_INPUT, "array out-pointer is NULL");
    size_t es = dtype_size(dtype);
    B200_EXPECTS(es > 0, CUGRAPH_UNSUPPORTED_TYPE_COMBINATION, "invalid dtype");
    void* p = std::malloc(n_elems * es > 0 ? n_elems * es : 1);
    B200_EXPECTS(p != nullptr, CUGRAPH_ALLOC_ERROR, "host allocation failed");
    *array = reinterpret_cast<cugraph_type_erased_host_array_t*>(new host_array_impl{p, n_elems, dtype});
  });
}

void cugraph_type_erased_host_array_free(cugraph_type_erased_host_array_t* p)
{
  if (!p) return;
  auto* a = reinterpret_cast<host_array_impl*>(p);
  std::free(a->data);
  delete a;
}

cugraph_type_erased_host_array_view_t* cugraph_type_erased_host_array_view(
  cugraph_type_erased_host_array_t* array)
{
  if (!array) return nullptr;
  auto* a = reinterpret_cast<host_array_impl*>(array);
  return reinterpret_cast<cugraph_type_erased_host_array_view_t*>(
    new host_array_view_impl{a->data, a->size, a->type});
}

cugraph_type_erased_host_array_view_t* cugraph_type_erased_host_array_view_create(
  void* pointer, size_t n_elems, cugraph_data_type_id_t dtype)
{
  return reinterpret_cast<cugraph_type_erased_host_array_view_t*>(
    new host_array_view_impl{pointer, n_elems, dtype});
}

void cugraph_type_erased_host_array_view_free(cugraph_type_erased_host_array_view_t* p)
{
  if (p) delete reinterpret_cast<host_array_view_impl*>(p);
}

size_t cugraph_type_erased_host_array_size(const cugraph_type_erased_host_array_view_t* p)
{
  return p ? reinterpret_cast<host_array_view_impl const*>(p)->size : 0;
}

cugraph_data_type_id_t cugraph_type_erased_host_array_type(const cugraph_type_erased_host_array_view_t* p)
{
  return p ? reinterpret_cast<host_array_view_impl const*>(p)->type : NTYPES;
}

void* cugraph_type_erased_host_array_pointer(const cugraph_type_erased_host_array_view_t* p)
{
  return p ? reinterpret_cast<host_array_view_impl const*>(p)->data : nullptr;
}

// ------------------------------------------------------------------------- array.h:264-326
cugraph_error_code_t cugraph_type_erased_host_array_view_copy(
  const cugraph_resource_handle_t* handle,
  cugraph_type_erased_host_array_view_t* dst,
  const cugraph_type_erased_host_array_view_t* src,
  cugraph_error_t** error)
{
  return guarded(error, [&] {
    (void)H(handle);
    B200_EXPECTS(dst && src, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* d       = reinterpret_cast<host_array_view_impl*>(dst);
    auto const* s = reinterpret_cast<host_array_view_impl const*>(src);
    B200_EXPECTS(d->nbytes() == s->nbytes(), CUGRAPH_INVALID_INPUT,
                 "source and destination arrays are different sizes");
    std::memcpy(d->data, s->data, s->nbytes());
  });
}

cugraph_error_code_t cugraph_type_erased_device_array_view_copy_from_host(
  const cugraph_resource_handle_t* handle,
  cugraph_type_erased_device_array_view_t* dst,
  const byte_t* h_src,
  cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(dst != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* d = reinterpret_cast<device_array_view_impl*>(dst);
    if (d->nbytes() > 0) {
      B200_EXPECTS(h_src != nullptr, CUGRAPH_INVALID_INPUT, "host source is NULL");
      CUDA_TRY(cudaMemcpyAsync(d->data, h_src, d->nbytes(), cudaMemcpyHostToDevice, h.stream));
    }
    sync(h);
  });
}

cugraph_error_code_t cugraph_type_erased_device_array_view_copy_to_host(
  const cugraph_resource_handle_t* handle,
  byte_t* h_dst,
  const cugraph_type_erased_device_array_view_t* src,
  cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(src != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto const* s = V(src);
    if (s->nbytes() > 0) {
      B200_EXPECTS(h_dst != nullptr, CUGRAPH_INVALID_INPUT, "host destination is NULL");
      CUDA_TRY(cudaMemcpyAsync(h_dst, s->data, s->nbytes(), cudaMemcpyDeviceToHost, h.stream));
    }
    sync(h);
  });
}

cugraph_error_code_t cugraph_type_erased_device_array_view_copy(
  const cugraph_resource_handle_t* handle,
  cugraph_type_erased_device_array_view_t* dst,
  const cugraph_type_erased_device_array_view_t* src,
  cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(dst && src, CUGRAPH_INVALID_INPUT, "NULL argument");
    auto* d       = reinterpret_cast<device_array_view_impl*>(dst);
    auto const* s = V(src);
    B200_EXPECTS(d->nbytes() == s->nbytes(), CUGRAPH_INVALID_INPUT,
                 "source and destination arrays are different sizes");
    if (s->nbytes() > 0)
      CUDA_TRY(cudaMemcpyAsync(d->data, s->data, s->nbytes(), cudaMemcpyDeviceToDevice, h.stream));
    sync(h);
  });
}

}  // extern "C"
