// Weakly connected components (reference cpp/src/components/weakly_connected_components_impl.cuh:271-860, C API
// cpp/src/c_api/weakly_connected_components.cpp, cpp/include/cugraph_c/labeling_algorithms.h:20-75).  The reference grows BFS
// trees from batches of roots and merges colliding trees; here: hooking + pointer jumping over the stored edges
// (every edge hooks the larger of its endpoints' roots under the smaller with an atomicMin, then every vertex's pointer is
// compressed to its root; repeat until no edge joins two roots — O(log V) rounds of one pass over the edges each).
// The label of a component is the external id of its vertex with the smallest internal id.
#include "graph.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ int find_root(int32_t* parent, int v)
{
  int p = ((volatile int32_t*)parent)[v];
  while (p != v) {  // path halving: pointers only ever decrease, so racing updates stay valid
    const int gp = ((volatile int32_t*)parent)[p];
    if (gp != p) parent[v] = gp;
    v = p;
    p = gp;
  }
  return v;
}

__device__ __forceinline__ void hook(int32_t* parent, int u, int v, int* changed)
{
  int ru = find_root(parent, u), rv = find_root(parent, v);
  while (ru != rv) {
    const int hi = ru > rv ? ru : rv, lo = ru > rv ? rv : ru;
    const int old = atomicMin(parent + hi, lo);  // hi is (was) a root: parent[hi] == hi unless somebody hooked it first
    if (old == hi) {
      *changed = 1;
      return;
    }
    ru = find_root(parent, old);  // somebody else hooked hi under `old`: join that tree with lo instead
    rv = lo;
  }
}

// rows of degree >= 32 (a prefix of the degree-ordered rows): a warp per row; the others: a thread per row
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_hook_hi(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t n_hi, int32_t* parent,
          int* changed)
{
  const int lane = threadIdx.x & 31;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < n_hi; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int u = row_vertex ? row_vertex[r] : (int)r;
    for (long long e = (long long)off[r] + lane; e < (long long)off[r + 1]; e += 32) hook(parent, u, idx[e], changed);
  }
}
template <typename O>
__global__ void __launch_bounds__(kBlock)
k_hook_low(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t const* __restrict__ row_vertex, int32_t r0, int32_t r1,
           int32_t* parent, int* changed)
{
  for (long long r = r0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; r < r1; r += (long long)gridDim.x * blockDim.x) {
    const int u = row_vertex ? row_vertex[r] : (int)r;
    for (long long e = (long long)off[r]; e < (long long)off[r + 1]; ++e) hook(parent, u, idx[e], changed);
  }
}
__global__ void k_compress(int32_t* parent, int32_t n)
{
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) parent[v] = find_root(parent, v);
}

template <typename O>
void wcc_rounds(handle_impl const& h, csx_t const& c, int32_t nv, int32_t* parent)
{
  dbuf d_changed = make_dbuf<int>(1, h.stream);
  const int32_t n_hi = c.degree_sorted ? c.seg[0] : 0;
  const int32_t n_ne = c.degree_sorted ? c.seg[kNumSeg - 2] : c.n_rows;
  const int vgrid    = grid_for(nv, 1, h.sm_count * 8);
  while (true) {
    CUDA_TRY(cudaMemsetAsync(d_changed.data(), 0, sizeof(int), h.stream));
    if (n_hi > 0)
      B200_LAUNCH(h, (k_hook_hi<O>), grid_for((int64_t)n_hi * 32, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(), c.indices.as<int32_t>(),
                  c.row_vertex.as<int32_t>(), n_hi, parent, d_changed.as<int>());
    if (n_ne > n_hi)
      B200_LAUNCH(h, (k_hook_low<O>), grid_for(n_ne - n_hi, 1, h.sm_count * 16), kBlock, 0, c.offsets.as<O>(),
                  c.indices.as<int32_t>(), c.row_vertex.as<int32_t>(), n_hi, n_ne, parent, d_changed.as<int>());
    B200_LAUNCH(h, k_compress, vgrid, kBlock, 0, parent, nv);
    if (!read_back(h, d_changed.as<int>())) break;
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_weakly_connected_components(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                         bool_t do_expensive_check, cugraph_labeling_result_t** result,
                                                         cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(g->is_symmetric, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: input graph should be symmetric for weakly connected components.");
    const int32_t nv = g->n_vertices;
    dbuf parent      = make_dbuf<int32_t>(std::max(nv, 1), h.stream);
    if (nv > 0) {
      B200_LAUNCH(h, k_iota<int32_t>, grid_for(nv, 1, h.sm_count * 8), kBlock, 0, parent.as<int32_t>(), (int64_t)nv);
      csx_t const& c = *g->primary;  // symmetric: either orientation holds every edge in both directions
      if (c.offs64) wcc_rounds<int64_t>(h, c, nv, parent.as<int32_t>());
      else wcc_rounds<int32_t>(h, c, nv, parent.as<int32_t>());
    }
    // labels: the root's external id, reported in the result's vertex order
    dbuf label_ext(std::max<size_t>(nv, 1) * dtype_size(g->vertex_type), h.stream);
    int_to_ext(h, *g, parent.as<int32_t>(), (size_t)nv, label_ext.data());
    auto res      = std::make_unique<labeling_result_impl>();
    res->vertices = new device_array_impl{reported_vertices(h, *g), (size_t)nv, g->vertex_type};
    res->labels   = new device_array_impl{to_reported_order(h, *g, label_ext.data(), dtype_size(g->vertex_type)), (size_t)nv, g->vertex_type};
    check_last("weakly_connected_components");
    sync(h);
    *result = reinterpret_cast<cugraph_labeling_result_t*>(res.release());
  });
}

cugraph_type_erased_device_array_view_t* cugraph_labeling_result_get_vertices(cugraph_labeling_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<labeling_result_impl*>(result)->vertices->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_labeling_result_get_labels(cugraph_labeling_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<labeling_result_impl*>(result)->labels->new_view());
}
void cugraph_labeling_result_free(cugraph_labeling_result_t* result)
{
  if (!result) return;
  auto* r = reinterpret_cast<labeling_result_impl*>(result);
  delete r->vertices;
  delete r->labels;
  delete r;
}

}  // extern "C"
