// Katz centrality and HITS on the pull sweep — the sibling algorithms that run on the same primitive as PageRank
// (per_v_transform_reduce_incoming_e / _outgoing_e with reduce_op::plus; reference cpp/src/centrality/katz_centrality_impl.cuh:34-196,
// cpp/src/link_analysis/hits_impl.cuh:29-206, C API cpp/src/c_api/katz.cpp, cpp/src/c_api/hits.cpp).  Each is a host loop
// over pull_sweep (sweep.cu: the shared-memory piece stream when the graph has one) and the owner-step kernels of
// centrality_ops.cuh over all vertices: the single-GPU form of its MGGraph loop (mg.py), without the collectives.  Each
// iteration reads its scalars back once, for the convergence test.
#include "centrality_ops.cuh"
#include "graph.cuh"

#include <array>
#include <cmath>
#include <limits>

namespace b200 {
namespace {

// ------------------------------------------------------------------------------------------
// Katz: x <- alpha * A^T x + beta until sum |x_new - x_old| < epsilon; then x / ||x||_2 (the C API always normalises,
// c_api/katz.cpp:116-129, and — faithfully — passes betas = nullptr whatever the caller gave, katz.cpp:151-152)
// ------------------------------------------------------------------------------------------
template <typename T>
void katz_typed(handle_impl const& h, graph_impl& g, double alpha, double beta, double epsilon, size_t max_iterations,
                centrality_result_impl& res)
{
  const int32_t nv = g.n_vertices;
  csx_t const& c   = pull_view(h, g);
  dbuf x = make_sweep_x<T>(h, nv), y = make_dbuf<T>(std::max(nv, 1), h.stream);  // x: zeros (katz_centrality_impl.cuh:88-93)
  sweep_scratch_t sc;
  sc.init(h, c);
  // the sweep adds beta before its one rounding to T (adding it in the step would round twice), so the step adds 0
  sc.set_init(h, beta);
  dbuf d2      = make_dbuf<double>(2, h.stream);  // diff, sum x^2
  size_t iter  = 0;
  double sumsq = 0.0;
  while (nv > 0) {
    pull_sweep<T>(h, c, nv, x.as<T>(), y.as<T>(), sc, alpha);
    CUDA_TRY(cudaMemsetAsync(d2.data(), 0, 2 * sizeof(double), h.stream));
    B200_LAUNCH(h, (k_katz_step<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, y.as<T>(), x.as<T>(), nv, 0.0, d2.as<double>());
    const std::array<double, 2> r = read_back(h, d2.as<std::array<double, 2>>());
    sumsq                         = r[1];
    ++iter;
    if ((T)r[0] < (T)epsilon) break;
    B200_EXPECTS(iter < max_iterations, CUGRAPH_UNKNOWN_ERROR, "Katz Centrality failed to converge.");
  }
  if (nv > 0) {  // x holds the final values, and sumsq their sum of squares (from the last step)
    const double l2 = std::sqrt(sumsq);
    B200_EXPECTS(l2 > 0.0, CUGRAPH_UNKNOWN_ERROR, "L2 norm of the computed Katz Centrality values should be positive.");
    B200_LAUNCH(h, (k_scale<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, x.as<T>(), nv, 1.0 / l2);
  }
  res.vertices   = new device_array_impl{reported_vertices(h, g), (size_t)nv, g.vertex_type};
  res.values     = new device_array_impl{to_reported_order(h, g, x.data(), sizeof(T)), (size_t)nv, g.weight_type};
  res.iterations = iter;
  res.converged  = true;
  check_last("katz");
  sync(h);
}

// ------------------------------------------------------------------------------------------
// Eigenvector centrality (eigenvector_centrality_impl.cuh:34-150): x <- (A^T x + x) / ||A^T x + x||_2 from x = 1 / V, until
// sum |x_new - x_old| < V * epsilon
// ------------------------------------------------------------------------------------------
template <typename T>
void eigenvector_typed(handle_impl const& h, graph_impl& g, double epsilon, size_t max_iterations, centrality_result_impl& res)
{
  const int32_t nv = g.n_vertices;
  csx_t const& c   = pull_view(h, g);
  dbuf x = make_sweep_x<T>(h, nv), y = make_dbuf<T>(std::max(nv, 1), h.stream);
  if (nv > 0) B200_LAUNCH(h, (k_fill<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, x.as<T>(), (int64_t)nv, (T)(1.0 / (double)nv));
  sweep_scratch_t sc;
  sc.init(h, c);
  dbuf d2     = make_dbuf<double>(2, h.stream);  // sum y^2, diff
  size_t iter = 0;
  while (nv > 0) {
    pull_sweep<T>(h, c, nv, x.as<T>(), y.as<T>(), sc, 1.0);
    CUDA_TRY(cudaMemsetAsync(d2.data(), 0, 2 * sizeof(double), h.stream));
    B200_LAUNCH(h, (k_eig_add<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, y.as<T>(), x.as<T>(), nv, d2.as<double>());
    B200_LAUNCH(h, (k_eig_scale<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, y.as<T>(), x.as<T>(), nv, d2.as<double>(),
                d2.as<double>() + 1);
    const double diff = read_back(h, d2.as<double>() + 1);
    ++iter;
    if ((T)diff < (T)nv * (T)epsilon) break;
    B200_EXPECTS(iter < max_iterations, CUGRAPH_UNKNOWN_ERROR, "Eigenvector Centrality failed to converge.");
  }
  res.vertices   = new device_array_impl{reported_vertices(h, g), (size_t)nv, g.vertex_type};
  res.values     = new device_array_impl{to_reported_order(h, g, x.data(), sizeof(T)), (size_t)nv, g.weight_type};
  res.iterations = iter;
  res.converged  = true;
  check_last("eigenvector_centrality");
  sync(h);
}

// ------------------------------------------------------------------------------------------
// HITS (hits_impl.cuh:49-191): authorities = sum over in-edges of the hubs, hubs = sum over out-edges of the
// authorities, both divided by their maximum; until sum |hubs - previous hubs| < V * epsilon; edge weights are not used
// ------------------------------------------------------------------------------------------
struct hits_result_impl {
  device_array_impl* vertices{nullptr};
  device_array_impl* hubs{nullptr};
  device_array_impl* authorities{nullptr};
  double hub_score_differences{0.0};
  size_t number_of_iterations{0};
};

// v /= sum v (the initial guess, and both results with `normalize`)
template <typename T>
void normalize_by(handle_impl const& h, T* v, int32_t nv, dbuf& d)
{
  CUDA_TRY(cudaMemsetAsync(d.data(), 0, sizeof(double), h.stream));
  B200_LAUNCH(h, (k_norm<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, v, nv, 1, d.as<double>());
  const double norm = read_back(h, d.as<double>());
  B200_EXPECTS((T)norm > (T)0, CUGRAPH_UNKNOWN_ERROR, "Norm is required to be a positive value.");
  B200_LAUNCH(h, (k_scale<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, v, nv, 1.0 / norm);
}

template <typename T>
void hits_typed(handle_impl const& h, graph_impl& g, double epsilon, size_t max_iterations, device_array_view_impl const* guess_v,
                device_array_view_impl const* guess_val, bool normalize, bool do_expensive_check, hits_result_impl& res)
{
  const int32_t nv   = g.n_vertices;
  csx_t const& c_in  = pull_view(h, g);       // rows = destinations: authorities <- hubs
  csx_t const& c_out = out_sweep_view(h, g);  // rows = sources: hubs <- authorities
  dbuf hubs_a = make_sweep_x<T>(h, nv), hubs_b = make_sweep_x<T>(h, nv), auth = make_sweep_x<T>(h, nv);
  dbuf d3 = make_dbuf<double>(3, h.stream);  // hub max, authority max, diff
  B200_EXPECTS(epsilon >= 0.0, CUGRAPH_INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.");
  double diff = std::numeric_limits<T>::max();
  size_t iter = max_iterations;
  if (nv > 0) {
    const T tolerance = (T)nv * (T)epsilon;
    if (guess_v) {
      dbuf gv = collect_vertex_values<T>(h, g, guess_v, guess_val, (T)0);
      CUDA_TRY(cudaMemcpyAsync(hubs_a.data(), gv.data(), sizeof(T) * nv, cudaMemcpyDeviceToDevice, h.stream));
      if (do_expensive_check) {
        dbuf neg = make_dbuf<int>(1, h.stream);
        CUDA_TRY(cudaMemsetAsync(neg.data(), 0, sizeof(int), h.stream));
        B200_LAUNCH(h, (k_count_negative<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, hubs_a.as<T>(), (int64_t)nv, neg.as<int>());
        B200_EXPECTS(read_back(h, neg.as<int>()) == 0, CUGRAPH_INVALID_INPUT, "Invalid input argument: initial guess values should be non-negative.");
      }
      normalize_by<T>(h, hubs_a.as<T>(), nv, d3);
    } else {
      B200_LAUNCH(h, (k_fill<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, hubs_a.as<T>(), (int64_t)nv, (T)(1.0 / (double)nv));
    }
    sweep_scratch_t sc_in, sc_out;
    sc_in.init(h, c_in);
    sc_out.init(h, c_out);
    T* prev = hubs_a.as<T>();
    T* curr = hubs_b.as<T>();
    iter    = 0;
    while (true) {
      pull_sweep<T>(h, c_in, nv, prev, auth.as<T>(), sc_in, 1.0, false);
      pull_sweep<T>(h, c_out, nv, auth.as<T>(), curr, sc_out, 1.0, false);
      CUDA_TRY(cudaMemsetAsync(d3.data(), 0, 3 * sizeof(double), h.stream));
      B200_LAUNCH(h, (k_hits_max<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, curr, auth.as<T>(), nv, d3.as<double>());
      B200_LAUNCH(h, (k_hits_scale<T>), grid_for(nv, 1, h.sm_count * 8), kBlock, 0, curr, auth.as<T>(), prev, nv, d3.as<double>(),
                  d3.as<double>() + 2);
      const std::array<double, 3> r = read_back(h, d3.as<std::array<double, 3>>());
      B200_EXPECTS((T)r[0] > (T)0 && (T)r[1] > (T)0, CUGRAPH_UNKNOWN_ERROR, "Norm is required to be a positive value.");
      diff = (double)(T)r[2];
      std::swap(prev, curr);
      ++iter;
      if ((T)diff < tolerance) break;
      B200_EXPECTS(iter < max_iterations, CUGRAPH_UNKNOWN_ERROR, "HITS failed to converge.");
    }
    if (normalize) {
      normalize_by<T>(h, prev, nv, d3);
      normalize_by<T>(h, auth.as<T>(), nv, d3);
    }
    res.hubs        = new device_array_impl{to_reported_order(h, g, prev, sizeof(T)), (size_t)nv, g.weight_type};
    res.authorities = new device_array_impl{to_reported_order(h, g, auth.data(), sizeof(T)), (size_t)nv, g.weight_type};
  } else {
    res.hubs        = new device_array_impl{dbuf(0, h.stream), 0, g.weight_type};
    res.authorities = new device_array_impl{dbuf(0, h.stream), 0, g.weight_type};
  }
  res.vertices              = new device_array_impl{reported_vertices(h, g), (size_t)nv, g.vertex_type};
  res.hub_score_differences = diff;
  res.number_of_iterations  = iter;
  check_last("hits");
  sync(h);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

cugraph_error_code_t cugraph_katz_centrality(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                             const cugraph_type_erased_device_array_view_t* betas, double alpha, double beta,
                                             double epsilon, size_t max_iterations, bool_t do_expensive_check,
                                             cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  (void)betas;  // the reference's C entry point drops them (c_api/katz.cpp:151-152 constructs its functor with nullptr)
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(alpha >= 0.0 && alpha <= 1.0, CUGRAPH_INVALID_INPUT, "Invalid input argument: alpha should be in [0.0, 1.0].");
    B200_EXPECTS(epsilon >= 0.0, CUGRAPH_INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.");
    auto res = std::make_unique<centrality_result_impl>();
    if (g->weight_type == FLOAT32) katz_typed<float>(h, *g, alpha, beta, epsilon, max_iterations, *res);
    else katz_typed<double>(h, *g, alpha, beta, epsilon, max_iterations, *res);
    *result = reinterpret_cast<cugraph_centrality_result_t*>(res.release());
  });
}

cugraph_error_code_t cugraph_eigenvector_centrality(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, double epsilon,
                                                    size_t max_iterations, bool_t do_expensive_check,
                                                    cugraph_centrality_result_t** result, cugraph_error_t** error)
{
  (void)do_expensive_check;
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    B200_EXPECTS(epsilon >= 0.0, CUGRAPH_INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.");
    auto res = std::make_unique<centrality_result_impl>();
    if (g->weight_type == FLOAT32) eigenvector_typed<float>(h, *g, epsilon, max_iterations, *res);
    else eigenvector_typed<double>(h, *g, epsilon, max_iterations, *res);
    *result = reinterpret_cast<cugraph_centrality_result_t*>(res.release());
  });
}

cugraph_error_code_t cugraph_hits(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, double epsilon,
                                  size_t max_iterations, const cugraph_type_erased_device_array_view_t* initial_hubs_guess_vertices,
                                  const cugraph_type_erased_device_array_view_t* initial_hubs_guess_values, bool_t normalize,
                                  bool_t do_expensive_check, cugraph_hits_result_t** result, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(result != nullptr, CUGRAPH_INVALID_INPUT, "result out-pointer is NULL");
    *result = nullptr;
    auto const* gv = V(initial_hubs_guess_vertices);
    auto const* gx = V(initial_hubs_guess_values);
    if (gv) {
      B200_EXPECTS(gx != nullptr && gx->size == gv->size, CUGRAPH_INVALID_INPUT, "initial hubs guess needs vertices and values of equal size");
      B200_EXPECTS(gv->type == g->vertex_type, CUGRAPH_INVALID_INPUT, "vertex type of graph and initial_hubs_guess_vertices must match");
      B200_EXPECTS(gx->type == g->weight_type, CUGRAPH_INVALID_INPUT, "weight type of graph and initial_hubs_guess_values must match");
    }
    auto res = std::make_unique<hits_result_impl>();
    if (g->weight_type == FLOAT32)
      hits_typed<float>(h, *g, epsilon, max_iterations, gv, gx, normalize == TRUE, do_expensive_check == TRUE, *res);
    else
      hits_typed<double>(h, *g, epsilon, max_iterations, gv, gx, normalize == TRUE, do_expensive_check == TRUE, *res);
    *result = reinterpret_cast<cugraph_hits_result_t*>(res.release());
  });
}

cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_vertices(cugraph_hits_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<hits_result_impl*>(result)->vertices->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_hubs(cugraph_hits_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<hits_result_impl*>(result)->hubs->new_view());
}
cugraph_type_erased_device_array_view_t* cugraph_hits_result_get_authorities(cugraph_hits_result_t* result)
{
  return reinterpret_cast<cugraph_type_erased_device_array_view_t*>(reinterpret_cast<hits_result_impl*>(result)->authorities->new_view());
}
double cugraph_hits_result_get_hub_score_differences(cugraph_hits_result_t* result)
{
  return reinterpret_cast<hits_result_impl*>(result)->hub_score_differences;
}
size_t cugraph_hits_result_get_number_of_iterations(cugraph_hits_result_t* result)
{
  return reinterpret_cast<hits_result_impl*>(result)->number_of_iterations;
}
void cugraph_hits_result_free(cugraph_hits_result_t* result)
{
  if (!result) return;
  auto* r = reinterpret_cast<hits_result_impl*>(result);
  delete r->vertices;
  delete r->hubs;
  delete r->authorities;
  delete r;
}

}  // extern "C"
