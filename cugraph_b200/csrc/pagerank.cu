// PageRank on one GPU + its C-ABI entry points.
// Replaces cpp/src/link_analysis/pagerank_impl.cuh:40-330 (driver) and cpp/src/c_api/pagerank.cpp.
//
// Per iteration the reference runs ~6 V-sized thrust passes and 2 blocking scalar read-backs
// (pagerank_impl.cuh:225-318).  Here an iteration is: pull sweep (sweep.cu), whose row epilogue does the vertex pass
// (diff, dangling sum, next x = pr/out_w) where it writes each row, into the other of two x buffers -> 1-thread finalize
// that advances the device-resident loop state.  Personalized calls add their scatter after the sweep and so keep the
// separate vertex pass.  The host enqueues iterations in batches and only reads the `done` flag between batches; kernels
// of iterations past convergence are no-ops, so the iteration count and result are exactly those of a check-every-iteration
// loop.
#include "centrality_ops.cuh"
#include "graph.cuh"
#include "staging.cuh"

#include <algorithm>
#include <cmath>

namespace b200 {
namespace {

__global__ void k_out_degree(int32_t const* __restrict__ indices, long long nnz, int32_t* __restrict__ deg)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(deg + indices[i], 1);
}

template <typename T>
__global__ void k_out_weight(int32_t const* __restrict__ indices, T const* __restrict__ w, long long nnz, double* __restrict__ sums)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(sums + indices[i], (double)w[i]);
}

template <typename S, typename T>
__global__ void k_cast(S const* in, int32_t n, T* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (T)in[i];
}

// fused vertex pass: diff += |new-old| ; dangling += new where out_w==0 ; x = new / (out_w or 1).  The prologue's, and the
// iterations' of personalized calls; the others have the sweep's row epilogue do it (sweep_epilogue_t)
template <typename T>
__global__ void __launch_bounds__(kBlock)
k_vertex_pass(T const* __restrict__ pr_new, T const* __restrict__ pr_old, T const* __restrict__ out_w,
              T* __restrict__ x, int32_t n, pr_state_t* __restrict__ st)
{
  if (st->done) return;
  __shared__ double smem[8];
  double diff = 0.0, dang = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    T nv = pr_new[i];
    T ow = out_w[i];
    if (pr_old) diff += fabs((double)nv - (double)pr_old[i]);
    if (ow == (T)0) dang += (double)nv;
    x[i] = (ow == (T)0) ? nv : nv / ow;
  }
  diff = block_sum(diff, smem);
  dang = block_sum(dang, smem);
  if (threadIdx.x == 0) {
    if (pr_old) atomicAdd(&st->diff, diff);
    atomicAdd(&st->dangling, dang);
  }
}

// advance the loop state (pagerank_impl.cuh:256-259, 320-329)
__global__ void k_finalize(pr_state_t* st, double alpha, double epsilon, int n_vertices, int personalized,
                           int count_iteration, int max_iterations)
{
  if (st->done) return;
  double base    = st->dangling * alpha + (1.0 - alpha);
  st->init       = personalized ? 0.0 : base / (double)n_vertices;
  st->pers_scale = base;
  if (count_iteration) {
    st->iter += 1;
    st->last_diff = st->diff;
    if (st->diff < epsilon || st->iter >= max_iterations) st->done = 1;
  }
  st->diff     = 0.0;
  st->dangling = 0.0;
}

template <typename T>
__global__ void k_personalize(int32_t const* __restrict__ pv, T const* __restrict__ pvals, int32_t n, double pers_sum,
                              T* __restrict__ y, pr_state_t const* __restrict__ st)
{
  if (st->done) return;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[pv[i]] = (T)((double)y[pv[i]] + st->pers_scale * ((double)pvals[i] / pers_sum));
}

// entries equal to their predecessor in a sorted array
__global__ void k_count_repeats(int32_t const* __restrict__ sorted, int32_t n, int* __restrict__ out)
{
  for (int64_t i = 1 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (sorted[i] == sorted[i - 1]) atomicAdd(out, 1);
}

struct pr_args {
  device_array_view_impl const* pre_v{nullptr};
  device_array_view_impl const* pre_w{nullptr};
  device_array_view_impl const* init_v{nullptr};
  device_array_view_impl const* init_val{nullptr};
  device_array_view_impl const* pers_v{nullptr};
  device_array_view_impl const* pers_val{nullptr};
  double alpha{0.85};
  double epsilon{1e-5};
  size_t max_iterations{100};
  bool expensive{false};
};

template <typename T>
void pagerank_typed(handle_impl const& h, graph_impl& g, pr_args const& a, centrality_result_impl& res)
{
  phase_trace tr(h);
  const int32_t nv = g.n_vertices;
  // argument checks of pagerank_impl.cuh:79-88
  B200_EXPECTS(a.alpha >= 0.0 && a.alpha <= 1.0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: alpha should be in [0.0, 1.0].");
  B200_EXPECTS(a.epsilon >= 0.0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: epsilon should be non-negative.");
  if (nv == 0) {
    res.vertices   = new device_array_impl{dbuf(0, h.stream), 0, g.vertex_type};
    res.values     = new device_array_impl{dbuf(0, h.stream), 0, g.weight_type};
    res.iterations = 0;
    res.converged  = true;
    return;
  }
  csx_t const& c = pull_view(h, g);
  B200_EXPECTS(c.degree_sorted, CUGRAPH_UNKNOWN_ERROR, "internal: pull view is not binned");
  const bool weighted = g.weighted;

  // out-weight sums (pagerank_impl.cuh:180-198).  A property of the graph: computed once per graph
  // (the reference recomputes it on every call with a push-model prim, one atomic per edge).
  dbuf out_w_user;
  T const* out_w = nullptr;
  if (a.pre_w) {
    out_w_user = collect_vertex_values<T>(h, g, a.pre_v, a.pre_w, (T)0);
    out_w      = out_w_user.as<T>();
  } else {
    if (c.out_w.data() == nullptr) {
      dbuf ow = make_dbuf<T>(nv, h.stream);
      if (weighted) {
        dbuf sums = make_dbuf<double>(nv, h.stream);
        CUDA_TRY(cudaMemsetAsync(sums.data(), 0, sizeof(double) * nv, h.stream));
        if (c.nnz > 0)
          B200_LAUNCH(h, (k_out_weight<T>), grid_for(c.nnz, 1, h.sm_count * 16), kBlock, 0, c.indices.as<int32_t>(),
                      c.weights.as<T>(), (long long)c.nnz, sums.as<double>());
        B200_LAUNCH(h, (k_cast<double, T>), grid_for(nv), kBlock, 0, sums.as<double>(), nv, ow.as<T>());
      } else {
        dbuf deg = make_dbuf<int32_t>(nv, h.stream);
        CUDA_TRY(cudaMemsetAsync(deg.data(), 0, sizeof(int32_t) * nv, h.stream));
        if (c.nnz > 0)
          B200_LAUNCH(h, k_out_degree, grid_for(c.nnz, 1, h.sm_count * 16), kBlock, 0, c.indices.as<int32_t>(),
                      (long long)c.nnz, deg.as<int32_t>());
        B200_LAUNCH(h, (k_cast<int32_t, T>), grid_for(nv), kBlock, 0, deg.as<int32_t>(), nv, ow.as<T>());
      }
      sync(h);
      c.out_w = std::move(ow);
    }
    out_w = c.out_w.as<T>();
  }
  tr.mark("pagerank: pull view + out-weights");
  // the expensive input checks of pagerank_impl.cuh:90-175, in its order
  if (a.expensive && a.pre_w) {
    dbuf neg = make_dbuf<int>(1, h.stream);
    CUDA_TRY(cudaMemsetAsync(neg.data(), 0, sizeof(int), h.stream));
    B200_LAUNCH(h, (k_count_negative<T>), grid_for(nv), kBlock, 0, out_w, (int64_t)nv, neg.as<int>());
    B200_EXPECTS(read_back(h, neg.as<int>()) == 0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: outgoing edge weight sum values should be non-negative.");
  }
  if (a.expensive && weighted && c.nnz > 0) {
    dbuf neg = make_dbuf<int>(1, h.stream);
    CUDA_TRY(cudaMemsetAsync(neg.data(), 0, sizeof(int), h.stream));
    B200_LAUNCH(h, (k_count_negative<T>), grid_for(c.nnz, 1, h.sm_count * 16), kBlock, 0, c.weights.as<T>(), c.nnz, neg.as<int>());
    B200_EXPECTS(read_back(h, neg.as<int>()) == 0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: input edge weights should have non-negative values.");
  }

  // personalization (pagerank_impl.cuh:200-214): ids -> internal, sum must be positive
  dbuf pers_idx, pers_vals;
  int32_t n_pers  = 0;
  double pers_sum = 0.0;
  if (a.pers_v) {
    B200_EXPECTS(a.pers_val && a.pers_v->size == a.pers_val->size, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: if personalization.has_value() is true, the size of vertices and values should match");
    B200_EXPECTS(a.pers_v->size > 0, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: if personalizations.has_value() is true, the input personalization vector size should not be 0.");
    n_pers   = (int32_t)a.pers_v->size;
    pers_idx = make_dbuf<int32_t>(n_pers, h.stream);
    ext_to_int(h, g, a.pers_v->data, n_pers, pers_idx.as<int32_t>());
    struct pers_check_t {  // all read back with one copy
      double sum;
      int n_invalid;
      int n_negative;   // the expensive check only, as the two below
      int n_repeated;
    };
    dbuf chk = make_dbuf<pers_check_t>(1, h.stream);
    auto* dchk = chk.as<pers_check_t>();
    CUDA_TRY(cudaMemsetAsync(dchk, 0, sizeof(pers_check_t), h.stream));
    B200_LAUNCH(h, (k_count_negative<int32_t>), grid_for(n_pers), kBlock, 0, pers_idx.as<int32_t>(), (int64_t)n_pers, &dchk->n_invalid);
    B200_LAUNCH(h, (k_norm<T>), grid_for(n_pers, 1, 1024), kBlock, 0, (T const*)a.pers_val->data, n_pers, 1, &dchk->sum);
    dbuf sorted;
    if (a.expensive) {
      B200_LAUNCH(h, (k_count_negative<T>), grid_for(n_pers), kBlock, 0, (T const*)a.pers_val->data, (int64_t)n_pers,
                  &dchk->n_negative);
      // without this check a repeated vertex reaches k_personalize, whose read-modify-writes of y then race
      sorted = make_dbuf<int32_t>(n_pers, h.stream);
      sort_keys<int32_t>(h, pers_idx.as<int32_t>(), sorted.as<int32_t>(), n_pers, 0, 32);
      B200_LAUNCH(h, k_count_repeats, grid_for(n_pers), kBlock, 0, sorted.as<int32_t>(), n_pers, &dchk->n_repeated);
    }
    const pers_check_t hchk = read_back(h, dchk);
    B200_EXPECTS(hchk.n_invalid == 0, CUGRAPH_INVALID_INPUT, "Invalid input argument: peresonalization vertices have invalid vertex IDs.");
    B200_EXPECTS(hchk.n_negative == 0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: peresonalization values should be non-negative.");
    B200_EXPECTS(hchk.n_repeated == 0, CUGRAPH_UNKNOWN_ERROR,
                 "Invalid input argument: personalization vertices should not contain duplicate entries.");
    pers_sum = hchk.sum;
    B200_EXPECTS(pers_sum > 0.0, CUGRAPH_UNKNOWN_ERROR, "Invalid input argument: sum of personalization valuese should be positive.");
  }

  // state.  Two x buffers: the sweep's row epilogue writes the next x while the sweep still reads this one.  A personalized
  // call adds its scatter to y after the sweep, so its next x is made by a vertex pass after that, into the same buffer: it
  // needs one.  (Folding the scatter into the epilogue would need a dense V-sized personalization vector read per row,
  // about what the vertex pass costs.)
  const bool fused = n_pers == 0;
  dbuf pr_a = make_dbuf<T>(nv, h.stream), pr_b = make_dbuf<T>(nv, h.stream);
  dbuf x = make_sweep_x<T>(h, nv), x_alt;
  if (fused) x_alt = make_sweep_x<T>(h, nv);
  sweep_scratch_t sc;
  sc.init(h, c);
  pr_state_t* st = sc.st();

  if (a.init_val) {
    // the C API copies the guess as-is (cpp/src/c_api/pagerank.cpp:179-203, no normalisation)
    dbuf guess = collect_vertex_values<T>(h, g, a.init_v, a.init_val, (T)0);
    CUDA_TRY(cudaMemcpyAsync(pr_a.data(), guess.data(), sizeof(T) * nv, cudaMemcpyDeviceToDevice, h.stream));
    sync(h);
  } else {
    B200_LAUNCH(h, (k_fill<T>), grid_for(nv), kBlock, 0, pr_a.as<T>(), nv, (T)((T)1 / (T)nv));
  }

  tr.mark("pagerank: state setup");
  const int vgrid = grid_for(nv, 1, h.sm_count * 8);
  const int max_it = (int)std::min<size_t>(a.max_iterations, 0x7fffffff);
  // prologue: x and dangling sum of the starting vector, init for sweep 1
  B200_LAUNCH(h, (k_vertex_pass<T>), vgrid, kBlock, 0, pr_a.as<T>(), (T const*)nullptr, out_w, x.as<T>(), nv, st);
  B200_LAUNCH(h, k_finalize, 1, 1, 0, st, a.alpha, a.epsilon, nv, n_pers > 0 ? 1 : 0, 0, max_it);

  T* cur = pr_a.as<T>();
  T* nxt = pr_b.as<T>();
  T* xc  = x.as<T>();
  T* xn  = fused ? x_alt.as<T>() : nullptr;
  pr_state_t* hst = reinterpret_cast<pr_state_t*>(h.pinned);
  int enqueued    = 0;
  int iters       = 0;
  const int batch = (a.epsilon > 0.0) ? 8 : 64;
  while (true) {  // the reference's loop body runs at least once (pagerank_impl.cuh:224-327: test after iter++)
    int todo = std::min(batch, std::max(max_it, 1) - enqueued);
    for (int k = 0; k < todo; ++k) {
      if (fused) {
        // diff only where it is read: epsilon = 0 never stops on it and last_diff is not returned.  Nor, then, is y read
        // before the result: at epsilon = 0 the run ends after exactly max(max_it, 1) iterations, and only the last one
        // writes y (4 bytes per vertex less in every other sweep); the others write the next x alone
        const bool last = enqueued + 1 >= std::max(max_it, 1);
        sweep_epilogue_t<T> epi{out_w, xn, a.epsilon > 0.0 ? cur : nullptr};
        pull_sweep<T>(h, c, nv, xc, a.epsilon > 0.0 || last ? nxt : nullptr, sc, a.alpha, true, false, epi);
        std::swap(xc, xn);
      } else {
        pull_sweep<T>(h, c, nv, xc, nxt, sc, a.alpha);
        B200_LAUNCH(h, (k_personalize<T>), grid_for(n_pers), kBlock, 0, pers_idx.as<int32_t>(), (T const*)a.pers_val->data,
                    n_pers, pers_sum, nxt, st);
        B200_LAUNCH(h, (k_vertex_pass<T>), vgrid, kBlock, 0, nxt, cur, out_w, xc, nv, st);
      }
      B200_LAUNCH(h, k_finalize, 1, 1, 0, st, a.alpha, a.epsilon, nv, n_pers > 0 ? 1 : 0, 1, max_it);
      std::swap(cur, nxt);
      ++enqueued;
    }
    check_last("pagerank iteration");
    CUDA_TRY(cudaMemcpyAsync(hst, st, sizeof(pr_state_t), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    iters = hst->iter;
    if (hst->done || enqueued >= std::max(max_it, 1)) break;
  }
  tr.mark("pagerank: iterations (+ layout staging on the first call)");
  // after `iters` real iterations the newest vector sits in pr_a when iters is even, pr_b when odd
  T* final_pr = (iters % 2 == 0) ? pr_a.as<T>() : pr_b.as<T>();

  res.vertices   = new device_array_impl{reported_vertices(h, g), (size_t)nv, g.vertex_type};
  res.values     = new device_array_impl{to_reported_order(h, g, final_pr, sizeof(T)), (size_t)nv, g.weight_type};
  res.iterations = (size_t)iters;
  res.converged  = (size_t)iters < a.max_iterations;  // pagerank_impl.cuh:329
  sync(h);
  tr.mark("pagerank: result gather");
}

cugraph_error_code_t pagerank_entry(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, pr_args a,
                                    bool require_convergence, cugraph_centrality_result_t** result,
                                    cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    // type checks of cpp/src/c_api/pagerank.cpp:262-293
    if (a.pre_v) {
      B200_EXPECTS(a.pre_v->type == g->vertex_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and precomputed_vertex_out_weight_vertices must match");
      B200_EXPECTS(a.pre_w && a.pre_w->type == g->weight_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and precomputed_vertex_out_weight_sums must match");
    }
    if (a.init_v) {
      B200_EXPECTS(a.init_v->type == g->vertex_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and initial_guess_vertices must match");
      B200_EXPECTS(a.init_val && a.init_val->type == g->weight_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and initial_guess_values must match");
    }
    if (a.pers_v) {
      B200_EXPECTS(a.pers_v->type == g->vertex_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and personalization_vector must match");
      B200_EXPECTS(a.pers_val && a.pers_val->type == g->weight_type, CUGRAPH_INVALID_INPUT,
                   "vertex type of graph and personalization_vector must match");
    }
    if (!a.pre_w) a.pre_v = nullptr;
    if (!a.init_val) a.init_v = nullptr;
    auto res = std::make_unique<centrality_result_impl>();
    if (g->weight_type == FLOAT32) pagerank_typed<float>(h, *g, a, *res);
    else pagerank_typed<double>(h, *g, a, *res);
    bool converged = res->converged;
    *result        = reinterpret_cast<cugraph_centrality_result_t*>(res.release());
    // cpp/src/c_api/pagerank.cpp:306-313: the result object is still returned
    B200_EXPECTS(!require_convergence || converged, CUGRAPH_UNKNOWN_ERROR, "PageRank failed to converge.");
  });
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

cugraph_type_erased_device_array_view_t* cugraph_centrality_result_get_vertices(cugraph_centrality_result_t* result)
{
  auto* r = reinterpret_cast<centrality_result_impl*>(result);
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(r->vertices->new_view());
}

cugraph_type_erased_device_array_view_t* cugraph_centrality_result_get_values(cugraph_centrality_result_t* result)
{
  auto* r = reinterpret_cast<centrality_result_impl*>(result);
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(r->values->new_view());
}

size_t cugraph_centrality_result_get_num_iterations(cugraph_centrality_result_t* result)
{
  return reinterpret_cast<centrality_result_impl*>(result)->iterations;
}

bool_t cugraph_centrality_result_converged(cugraph_centrality_result_t* result)
{
  return reinterpret_cast<centrality_result_impl*>(result)->converged ? TRUE : FALSE;
}

void cugraph_centrality_result_free(cugraph_centrality_result_t* result)
{
  if (!result) return;
  auto* r = reinterpret_cast<centrality_result_impl*>(result);
  delete r->vertices;
  delete r->values;
  delete r;
}

#define PR_ARGS_COMMON                                                                          \
  pr_args a;                                                                                    \
  a.pre_v          = V(precomputed_vertex_out_weight_vertices);                                 \
  a.pre_w          = V(precomputed_vertex_out_weight_sums);                                     \
  a.init_v         = V(initial_guess_vertices);                                                 \
  a.init_val       = V(initial_guess_values);                                                   \
  a.alpha          = alpha;                                                                     \
  a.epsilon        = epsilon;                                                                   \
  a.max_iterations = max_iterations;                                                            \
  a.expensive      = do_expensive_check == TRUE;

cugraph_error_code_t cugraph_pagerank(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                      const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
                                      const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
                                      const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
                                      const cugraph_type_erased_device_array_view_t* initial_guess_values, double alpha,
                                      double epsilon, size_t max_iterations, bool_t do_expensive_check,
                                      cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  PR_ARGS_COMMON
  return pagerank_entry(handle, graph, a, true, result, error);
}

cugraph_error_code_t cugraph_pagerank_allow_nonconvergence(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values, double alpha, double epsilon,
  size_t max_iterations, bool_t do_expensive_check, cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  PR_ARGS_COMMON
  return pagerank_entry(handle, graph, a, false, result, error);
}

cugraph_error_code_t cugraph_personalized_pagerank(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  const cugraph_type_erased_device_array_view_t* personalization_vertices,
  const cugraph_type_erased_device_array_view_t* personalization_values, double alpha, double epsilon,
  size_t max_iterations, bool_t do_expensive_check, cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  PR_ARGS_COMMON
  a.pers_v   = V(personalization_vertices);
  a.pers_val = V(personalization_values);
  return pagerank_entry(handle, graph, a, true, result, error);
}

cugraph_error_code_t cugraph_personalized_pagerank_allow_nonconvergence(
  const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_vertices,
  const cugraph_type_erased_device_array_view_t* precomputed_vertex_out_weight_sums,
  const cugraph_type_erased_device_array_view_t* initial_guess_vertices,
  const cugraph_type_erased_device_array_view_t* initial_guess_values,
  const cugraph_type_erased_device_array_view_t* personalization_vertices,
  const cugraph_type_erased_device_array_view_t* personalization_values, double alpha, double epsilon,
  size_t max_iterations, bool_t do_expensive_check, cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  PR_ARGS_COMMON
  a.pers_v   = V(personalization_vertices);
  a.pers_val = V(personalization_values);
  return pagerank_entry(handle, graph, a, false, result, error);
}

// ------------------------------------------------------------------------ b200_ext.h bench hook
cugraph_error_code_t cugraph_b200_time_pull_spmv(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                 size_t iterations, double* ms_per_sweep,
                                                 double* algorithmic_bytes_per_sweep, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(g->weight_type == FLOAT32, CUGRAPH_NOT_IMPLEMENTED, "time_pull_spmv: float32 graphs only");
    csx_t const& c = pull_view(h, *g);
    int32_t nv     = g->n_vertices;
    dbuf x = make_sweep_x<float>(h, nv), y = make_dbuf<float>(nv, h.stream);
    B200_LAUNCH(h, (k_fill<float>), grid_for(nv), kBlock, 0, x.as<float>(), nv, 1.0f / (float)nv);
    sweep_scratch_t sc;
    sc.init(h, c);
    auto sweep = [&] { pull_sweep<float>(h, c, nv, x.as<float>(), y.as<float>(), sc, 0.85); };
    for (int k = 0; k < 3; ++k) sweep();
    cudaEvent_t e0, e1;
    CUDA_TRY(cudaEventCreate(&e0));
    CUDA_TRY(cudaEventCreate(&e1));
    CUDA_TRY(cudaEventRecord(e0, h.stream));
    for (size_t k = 0; k < iterations; ++k) sweep();
    CUDA_TRY(cudaEventRecord(e1, h.stream));
    CUDA_TRY(cudaEventSynchronize(e1));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    check_last("time_pull_spmv");
    if (ms_per_sweep) *ms_per_sweep = (double)ms / (double)std::max<size_t>(iterations, 1);
    // SURVEY §8d: E*4 [indices] (+E*4 weights) + (V+1)*sizeof(offset) + V*4 [x] + V*4 [y]
    if (algorithmic_bytes_per_sweep)
      *algorithmic_bytes_per_sweep = (double)c.nnz * 4.0 * (g->weighted ? 2.0 : 1.0) +
                                     (double)(nv + 1) * (c.offs64 ? 8.0 : 4.0) + (double)nv * 8.0;
  });
}

}  // extern "C"
