// Vertex degrees of a graph (reference cpp/include/cugraph_c/graph_functions.h:284-394, cpp/src/c_api/degrees.cpp,
// graph_view_t::compute_in_degrees / compute_out_degrees, cpp/include/cugraph/graph_view.hpp): the stored orientation's row
// lengths are one kind of degree, a histogram of its neighbour ids the other.  Results for every vertex (reported order) or
// for a caller-given list of vertices, in the graph's edge type (= its vertex type here).
#include "graph.cuh"

namespace b200 {
namespace {

template <typename O>
__global__ void k_row_lengths(O const* __restrict__ off, int32_t n, int32_t* __restrict__ out)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    out[v] = (int32_t)((long long)off[v + 1] - (long long)off[v]);
}
__global__ void k_index_histogram(int32_t const* __restrict__ idx, long long nnz, int32_t* __restrict__ out)
{
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nnz; e += (long long)gridDim.x * blockDim.x)
    atomicAdd(out + idx[e], 1);
}
// out[i] = (T)deg[sel ? sel[i] : i]
template <typename T>
__global__ void k_pick_degrees(int32_t const* __restrict__ deg, int32_t const* __restrict__ sel, long long n, T* __restrict__ out)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = sel ? sel[i] : (int)i;
    out[i]      = v >= 0 ? (T)deg[v] : (T)0;
  }
}

struct degrees_result_impl {
  device_array_impl* vertices{nullptr};
  device_array_impl* in_degrees{nullptr};
  device_array_impl* out_degrees{nullptr};
  bool shared{false};  // symmetric graph: one array serves both
};

// degrees by internal id: [0] = of the stored rows (majors), [1] = of the neighbour ids (minors)
void internal_degrees(handle_impl const& h, graph_impl const& g, bool want_major, bool want_minor, dbuf& major, dbuf& minor)
{
  csx_t const& c   = *g.primary;
  const int32_t nv = g.n_vertices;
  const int grid   = grid_for(nv, 1, h.sm_count * 8);
  if (want_major) {
    major = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    if (nv > 0) {
      if (c.offs64) B200_LAUNCH(h, (k_row_lengths<int64_t>), grid, kBlock, 0, c.offsets.as<int64_t>(), nv, major.as<int32_t>());
      else B200_LAUNCH(h, (k_row_lengths<int32_t>), grid, kBlock, 0, c.offsets.as<int32_t>(), nv, major.as<int32_t>());
    }
  }
  if (want_minor) {
    minor = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    CUDA_TRY(cudaMemsetAsync(minor.data(), 0, sizeof(int32_t) * std::max(nv, 1), h.stream));
    if (c.nnz > 0)
      B200_LAUNCH(h, k_index_histogram, grid_for(c.nnz, 1, h.sm_count * 16), kBlock, 0,
                  c.indices.as<int32_t>(), (long long)c.nnz, minor.as<int32_t>());
  }
}

cugraph_error_code_t degrees_entry(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                   const cugraph_type_erased_device_array_view_t* source_vertices, bool want_in, bool want_out,
                                   cugraph_degrees_result_t** result, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    auto const* sv = V(source_vertices);
    if (sv) B200_EXPECTS(sv->type == g->vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and source_vertices must match");
    const int32_t nv = g->n_vertices;
    // rows of the primary orientation are destinations when the graph is stored transposed
    const bool major_is_in = g->store_transposed;
    // cugraph_degrees on a graph declared symmetric computes the in-degrees only and serves them as both (c_api/degrees.cpp);
    // the single-direction calls always compute what they are asked for
    const bool share      = want_in && want_out && g->is_symmetric;
    const bool need_in    = want_in;
    const bool need_out   = want_out && !share;
    const bool need_major = major_is_in ? need_in : need_out;
    const bool need_minor = major_is_in ? need_out : need_in;
    dbuf major, minor;
    internal_degrees(h, *g, need_major, need_minor, major, minor);
    // which vertices, in which order
    const size_t n = sv ? sv->size : (size_t)nv;
    dbuf sel;  // internal ids of the requested vertices; all vertices: internal id per reported position
    dbuf verts_out;
    if (sv) {
      sel = make_dbuf<int32_t>(std::max<size_t>(n, 1), h.stream);
      ext_to_int(h, *g, sv->data, n, sel.as<int32_t>());
      verts_out = dbuf(std::max<size_t>(n, 1) * dtype_size(g->vertex_type), h.stream);
      if (n > 0) CUDA_TRY(cudaMemcpyAsync(verts_out.data(), sv->data, n * dtype_size(g->vertex_type), cudaMemcpyDeviceToDevice, h.stream));
    } else {
      verts_out = reported_vertices(h, *g);
      sel       = make_dbuf<int32_t>(std::max<size_t>(n, 1), h.stream);
      ext_to_int(h, *g, verts_out.data(), n, sel.as<int32_t>());
    }
    auto pick = [&](dbuf const& deg) {
      dbuf out(std::max<size_t>(n, 1) * dtype_size(g->edge_type), h.stream);
      const int grid = grid_for((int64_t)n, 1, h.sm_count * 8);
      if (g->edge_type == INT64)
        B200_LAUNCH(h, (k_pick_degrees<int64_t>), grid, kBlock, 0, deg.as<int32_t>(), sel.as<int32_t>(), (long long)n, out.as<int64_t>());
      else
        B200_LAUNCH(h, (k_pick_degrees<int32_t>), grid, kBlock, 0, deg.as<int32_t>(), sel.as<int32_t>(), (long long)n, out.as<int32_t>());
      return new device_array_impl{std::move(out), n, g->edge_type};
    };
    auto res      = std::make_unique<degrees_result_impl>();
    res->vertices = new device_array_impl{std::move(verts_out), n, g->vertex_type};
    if (need_in) res->in_degrees = pick(major_is_in ? major : minor);
    if (need_out) res->out_degrees = pick(major_is_in ? minor : major);
    res->shared = share;
    check_last("degrees");
    sync(h);
    *result = reinterpret_cast<cugraph_degrees_result_t*>(res.release());
  });
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_in_degrees(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                        const cugraph_type_erased_device_array_view_t* source_vertices, bool_t do_expensive_check,
                                        cugraph_degrees_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return degrees_entry(handle, graph, source_vertices, true, false, result, error);
}
cugraph_error_code_t cugraph_out_degrees(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                         const cugraph_type_erased_device_array_view_t* source_vertices, bool_t do_expensive_check,
                                         cugraph_degrees_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return degrees_entry(handle, graph, source_vertices, false, true, result, error);
}
cugraph_error_code_t cugraph_degrees(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                     const cugraph_type_erased_device_array_view_t* source_vertices, bool_t do_expensive_check,
                                     cugraph_degrees_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return degrees_entry(handle, graph, source_vertices, true, true, result, error);
}

cugraph_type_erased_device_array_view_t* cugraph_degrees_result_get_vertices(cugraph_degrees_result_t* r)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<degrees_result_impl*>(r)->vertices->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_degrees_result_get_in_degrees(cugraph_degrees_result_t* r)
{
  auto* d = reinterpret_cast<degrees_result_impl*>(r);
  return d->in_degrees ? reinterpret_cast<cugraph_type_erased_device_array_view_t*>(d->in_degrees->new_view()) : nullptr;
}
cugraph_type_erased_device_array_view_t* cugraph_degrees_result_get_out_degrees(cugraph_degrees_result_t* r)
{
  auto* d = reinterpret_cast<degrees_result_impl*>(r);
  device_array_impl* a = d->shared ? d->in_degrees : d->out_degrees;  // symmetric: the same memory serves both
  return a ? reinterpret_cast<cugraph_type_erased_device_array_view_t*>(a->new_view()) : nullptr;
}
void cugraph_degrees_result_free(cugraph_degrees_result_t* r)
{
  if (!r) return;
  auto* d = reinterpret_cast<degrees_result_impl*>(r);
  delete d->vertices;
  delete d->in_degrees;
  delete d->out_degrees;
  delete d;
}

}  // extern "C"
