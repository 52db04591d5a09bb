// C-ABI graph construction.  Boundary replaced: cpp/src/c_api/graph_sg.cpp:699-… (create_sg,
// create_with_times_sg, create_sg_from_csr, graph_free) and graph_mg.cpp (create_mg, in mg.cu).
#include "graph.cuh"

#include <algorithm>
#include <vector>

namespace b200 {
void stage_graph(handle_impl const& h, graph_impl& g, device_array_view_impl const* verts,
                 device_array_view_impl const* src, device_array_view_impl const* dst, device_array_view_impl const* wv,
                 bool renumber, bool drop_self_loops, bool drop_multi_edges, bool symmetrize);

namespace {

template <typename O, typename VT>
__global__ void k_offsets_to_rows(O const* offsets, int64_t n_rows, VT* rows)
{
  int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  int lane     = threadIdx.x & 31;
  int64_t nw   = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_rows; r += nw)
    for (long long e = (long long)offsets[r] + lane; e < (long long)offsets[r + 1]; e += 32) rows[e] = (VT)r;
}

// do_expensive_check of the constructors (create_graph_from_edgelist_impl.cuh:803-830: check_symmetric :260-314,
// check_no_parallel_edge :316-334), evaluated on the staged adjacency instead of on sorted copies of the edge list: rows
// and neighbours are internal ids of one id space and every row's neighbours are ascending, so a parallel edge is two
// equal neighbours side by side and (r, c) has its reverse iff r is found in row c.  One warp per row.
// flags[0]: an edge without its reverse; flags[1]: a parallel edge.
template <typename O>
__global__ void k_expensive_check(O const* __restrict__ off, int32_t const* __restrict__ idx, int32_t n_rows, int check_sym,
                                  int check_dup, int* __restrict__ flags)
{
  const int lane = threadIdx.x & 31;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < n_rows;
       r += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long beg = (long long)off[r], end = (long long)off[r + 1];
    for (long long e = beg + lane; e < end; e += 32) {
      const int c = idx[e];
      if (check_dup && e > beg && idx[e - 1] == c) flags[1] = 1;
      if (check_sym) {
        long long lo = (long long)off[c], hi = (long long)off[c + 1];  // first position in row c with idx >= r
        while (lo < hi) {
          const long long mid = lo + ((hi - lo) >> 1);
          if (idx[mid] < (int)r) lo = mid + 1; else hi = mid;
        }
        if (lo >= (long long)off[c + 1] || idx[lo] != (int)r) flags[0] = 1;
      }
    }
  }
}

void expensive_check(handle_impl const& h, graph_impl const& g, bool check_sym, bool check_dup)
{
  csx_t const& c = *g.primary;
  if ((!check_sym && !check_dup) || c.nnz == 0) return;
  dbuf flags = make_dbuf<int>(2, h.stream);
  CUDA_TRY(cudaMemsetAsync(flags.data(), 0, 2 * sizeof(int), h.stream));
  const int grid = grid_for((int64_t)c.n_rows * 32, 1, h.sm_count * 32);
  if (c.offs64)
    B200_LAUNCH(h, (k_expensive_check<int64_t>), grid, kBlock, 0, c.offsets.as<int64_t>(), c.indices.as<int32_t>(), c.n_rows,
                check_sym ? 1 : 0, check_dup ? 1 : 0, flags.as<int>());
  else
    B200_LAUNCH(h, (k_expensive_check<int32_t>), grid, kBlock, 0, c.offsets.as<int32_t>(), c.indices.as<int32_t>(), c.n_rows,
                check_sym ? 1 : 0, check_dup ? 1 : 0, flags.as<int>());
  int hf[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(hf, flags.data(), sizeof(hf), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  check_last("expensive check");
  // the reference raises cugraph::logic_error here, which its C layer reports as CUGRAPH_UNKNOWN_ERROR (c_api/utils.hpp:43-46)
  B200_EXPECTS(hf[0] == 0, CUGRAPH_UNKNOWN_ERROR,
               "Invalid input arguments: graph_properties.is_symmetric is true but the input edge list is not symmetric.");
  B200_EXPECTS(hf[1] == 0, CUGRAPH_UNKNOWN_ERROR,
               "Invalid input arguments: graph_properties.is_multigraph is false but the input edge list has parallel edges.");
}

bool is_int_type(cugraph_data_type_id_t t) { return t == INT32 || t == INT64; }
bool is_float_type(cugraph_data_type_id_t t) { return t == FLOAT32 || t == FLOAT64; }

// shared validation + staging for the edge-list constructors
void create_sg_common(const cugraph_resource_handle_t* handle, const cugraph_graph_properties_t* properties,
                      const cugraph_type_erased_device_array_view_t* vertices,
                      const cugraph_type_erased_device_array_view_t* src,
                      const cugraph_type_erased_device_array_view_t* dst,
                      const cugraph_type_erased_device_array_view_t* weights,
                      const cugraph_type_erased_device_array_view_t* edge_ids,
                      const cugraph_type_erased_device_array_view_t* edge_type_ids,
                      const cugraph_type_erased_device_array_view_t* edge_start_times,
                      const cugraph_type_erased_device_array_view_t* edge_end_times, bool_t store_transposed,
                      bool_t renumber, bool_t drop_self_loops, bool_t drop_multi_edges, bool_t symmetrize,
                      bool_t do_expensive_check, cugraph_graph_t** graph)
{
  auto const& h = H(handle);
  B200_EXPECTS(graph != nullptr, CUGRAPH_INVALID_INPUT, "graph out-pointer is NULL");
  *graph = nullptr;
  B200_EXPECTS(properties != nullptr, CUGRAPH_INVALID_INPUT, "properties is NULL");
  B200_EXPECTS(src != nullptr && dst != nullptr, CUGRAPH_INVALID_INPUT, "src and dst are required");
  auto const* s  = V(src);
  auto const* d  = V(dst);
  auto const* w  = V(weights);
  auto const* vx = V(vertices);
  // the same checks, in the same order, as graph_sg.cpp:727-790
  B200_EXPECTS(s->size == d->size, CUGRAPH_INVALID_INPUT, "Invalid input arguments: src size != dst size.");
  B200_EXPECTS(s->type == d->type, CUGRAPH_INVALID_INPUT, "Invalid input arguments: src type != dst type.");
  B200_EXPECTS(vx == nullptr || vx->type == s->type, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: vertices type != src type.");
  B200_EXPECTS(w == nullptr || w->size == s->size, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: src size != weights size.");
  B200_EXPECTS(is_int_type(s->type), CUGRAPH_UNSUPPORTED_TYPE_COMBINATION, "vertex type must be INT32 or INT64");
  B200_EXPECTS(w == nullptr || is_float_type(w->type), CUGRAPH_UNSUPPORTED_TYPE_COMBINATION,
               "weight type must be FLOAT32 or FLOAT64");
  auto const* eid = V(edge_ids);
  auto const* ety = V(edge_type_ids);
  B200_EXPECTS(eid == nullptr || eid->size == s->size, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: src size != edge id prop size");
  B200_EXPECTS(ety == nullptr || ety->size == s->size, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: src size != edge type prop size");
  B200_EXPECTS(V(edge_start_times) == nullptr || V(edge_start_times)->size == s->size, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: src size != edge start time size");
  B200_EXPECTS(V(edge_end_times) == nullptr || V(edge_end_times)->size == s->size, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: src size != edge end time size");
  B200_EXPECTS(!(symmetrize && (eid || ety)), CUGRAPH_INVALID_INPUT,
               "symmetrize with edge ids / edge types is not supported");
  // graph_sg.cpp:737-742
  B200_EXPECTS(symmetrize != TRUE || properties->is_symmetric == TRUE, CUGRAPH_INVALID_INPUT,
               "Invalid input arguments: The graph property must be symmetric if 'symmetrize' is set to True.");

  auto g              = std::make_unique<graph_impl>();
  g->vertex_type      = s->type;
  g->edge_type        = s->type;  // is_vertex_edge_combo: both 32 or both 64 (graph_traits.hpp:36-40)
  g->weighted         = (w != nullptr);
  g->weight_type      = w ? w->type : FLOAT32;  // graph_sg.cpp:776-778
  g->is_symmetric     = properties->is_symmetric == TRUE || symmetrize == TRUE;
  g->is_multigraph    = properties->is_multigraph == TRUE;
  g->store_transposed = store_transposed == TRUE;
  g->device           = h.device;
  stage_graph(h, *g, vx, s, d, w, renumber == TRUE, drop_self_loops == TRUE, drop_multi_edges == TRUE,
              symmetrize == TRUE);
  // the reference checks the edge list it hands to the graph constructor, i.e. after the drop / symmetrize passes
  if (do_expensive_check == TRUE)
    expensive_check(h, *g, properties->is_symmetric == TRUE && symmetrize != TRUE,
                    properties->is_multigraph != TRUE && drop_multi_edges != TRUE);
  *graph = reinterpret_cast<cugraph_graph_t*>(g.release());
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_graph_create_sg(const cugraph_resource_handle_t* handle,
                                             const cugraph_graph_properties_t* properties,
                                             const cugraph_type_erased_device_array_view_t* vertices,
                                             const cugraph_type_erased_device_array_view_t* src,
                                             const cugraph_type_erased_device_array_view_t* dst,
                                             const cugraph_type_erased_device_array_view_t* weights,
                                             const cugraph_type_erased_device_array_view_t* edge_ids,
                                             const cugraph_type_erased_device_array_view_t* edge_type_ids,
                                             bool_t store_transposed, bool_t renumber, bool_t drop_self_loops,
                                             bool_t drop_multi_edges, bool_t symmetrize, bool_t do_expensive_check,
                                             cugraph_graph_t** graph, cugraph_error_t** error)
{
  return guarded(error, [&] {
    create_sg_common(handle, properties, vertices, src, dst, weights, edge_ids, edge_type_ids, nullptr, nullptr,
                     store_transposed, renumber, drop_self_loops, drop_multi_edges, symmetrize, do_expensive_check, graph);
  });
}

cugraph_error_code_t cugraph_graph_create_with_times_sg(
  const cugraph_resource_handle_t* handle, const cugraph_graph_properties_t* properties,
  const cugraph_type_erased_device_array_view_t* vertices, const cugraph_type_erased_device_array_view_t* src,
  const cugraph_type_erased_device_array_view_t* dst, const cugraph_type_erased_device_array_view_t* weights,
  const cugraph_type_erased_device_array_view_t* edge_ids, const cugraph_type_erased_device_array_view_t* edge_type_ids,
  const cugraph_type_erased_device_array_view_t* edge_start_time_ids,
  const cugraph_type_erased_device_array_view_t* edge_end_time_ids, bool_t store_transposed, bool_t renumber,
  bool_t drop_self_loops, bool_t drop_multi_edges, bool_t symmetrize, bool_t do_expensive_check,
  cugraph_graph_t** graph, cugraph_error_t** error)
{
  return guarded(error, [&] {
    create_sg_common(handle, properties, vertices, src, dst, weights, edge_ids, edge_type_ids, edge_start_time_ids,
                     edge_end_time_ids, store_transposed, renumber, drop_self_loops, drop_multi_edges, symmetrize,
                     do_expensive_check, graph);
  });
}

// CSR input (graph.h:177): rows are sources; expanded to an edge list and staged like any other.
cugraph_error_code_t cugraph_graph_create_sg_from_csr(
  const cugraph_resource_handle_t* handle, const cugraph_graph_properties_t* properties,
  const cugraph_type_erased_device_array_view_t* offsets, const cugraph_type_erased_device_array_view_t* indices,
  const cugraph_type_erased_device_array_view_t* weights, const cugraph_type_erased_device_array_view_t* edge_ids,
  const cugraph_type_erased_device_array_view_t* edge_type_ids, bool_t store_transposed, bool_t renumber,
  bool_t symmetrize, bool_t do_expensive_check, cugraph_graph_t** graph, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    B200_EXPECTS(offsets && indices, CUGRAPH_INVALID_INPUT, "offsets and indices are required");
    auto const* o = V(offsets);
    auto const* i = V(indices);
    B200_EXPECTS(o->size >= 1, CUGRAPH_INVALID_INPUT, "offsets must have at least one element");
    B200_EXPECTS(is_int_type(o->type) && is_int_type(i->type), CUGRAPH_UNSUPPORTED_TYPE_COMBINATION,
                 "offsets / indices must be INT32 or INT64");
    int64_t n_rows = (int64_t)o->size - 1;
    int64_t nnz    = (int64_t)i->size;
    dbuf rows(nnz * dtype_size(i->type), h.stream);
    int grid = (int)std::min<int64_t>(std::max<int64_t>((n_rows * 32 + 255) / 256, 1), 1 << 20);
    if (nnz > 0) {
      if (o->type == INT32 && i->type == INT32)
        B200_LAUNCH(h, (k_offsets_to_rows<int32_t, int32_t>), grid, 256, 0, (int32_t const*)o->data, n_rows, rows.as<int32_t>());
      else if (o->type == INT64 && i->type == INT64)
        B200_LAUNCH(h, (k_offsets_to_rows<int64_t, int64_t>), grid, 256, 0, (int64_t const*)o->data, n_rows, rows.as<int64_t>());
      else if (o->type == INT32 && i->type == INT64)
        B200_LAUNCH(h, (k_offsets_to_rows<int32_t, int64_t>), grid, 256, 0, (int32_t const*)o->data, n_rows, rows.as<int64_t>());
      else
        B200_LAUNCH(h, (k_offsets_to_rows<int64_t, int32_t>), grid, 256, 0, (int64_t const*)o->data, n_rows, rows.as<int32_t>());
      check_last("offsets_to_rows");
    }
    device_array_view_impl src_view{rows.data(), (size_t)nnz, i->type};
    // all ids 0..n_rows-1 are vertices of a CSR graph even when isolated
    dbuf vlist(n_rows * dtype_size(i->type), h.stream);
    device_array_view_impl vview{vlist.data(), (size_t)n_rows, i->type};
    {
      // reuse the expansion kernel trick: a sequence is offsets [0,1,2,...] expanded
      std::vector<char> host(n_rows * dtype_size(i->type));
      if (i->type == INT32) for (int64_t r = 0; r < n_rows; ++r) reinterpret_cast<int32_t*>(host.data())[r] = (int32_t)r;
      else for (int64_t r = 0; r < n_rows; ++r) reinterpret_cast<int64_t*>(host.data())[r] = r;
      if (n_rows > 0) CUDA_TRY(cudaMemcpyAsync(vlist.data(), host.data(), host.size(), cudaMemcpyHostToDevice, h.stream));
      sync(h);
    }
    create_sg_common(handle, properties, reinterpret_cast<cugraph_type_erased_device_array_view_t const*>(&vview),
                     reinterpret_cast<cugraph_type_erased_device_array_view_t const*>(&src_view), indices, weights,
                     edge_ids, edge_type_ids, nullptr, nullptr, store_transposed, renumber, FALSE, FALSE, symmetrize,
                     do_expensive_check, graph);
  });
}

void cugraph_graph_free(cugraph_graph_t* graph)
{
  if (!graph) return;
  delete reinterpret_cast<graph_impl*>(graph);
}

}  // extern "C"
