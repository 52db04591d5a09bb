// The pull sweep behind one entry point (pull_sweep, graph.cuh): which kernels run for a graph, and the scratch they need; the
// layout they read is built by sweep_layout.cu.  The only translation unit that includes the sweep kernels (sweep.cuh,
// spmv.cuh), so each is compiled once.
#include "sweep.cuh"

namespace b200 {
namespace {

// rows that may need an fp64 accumulator in a sweep: the piece stream covers every row
inline int32_t acc_rows(csx_t const& c) { return std::max(c.n_rows, 1); }

// ---- debug: compare the configured sweep with the plain reference sweep, row by row
template <typename T>
__global__ void k_fill_pattern(T* x, int32_t n)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    x[i] = (T)(0.5 + (double)(((unsigned)i * 2654435761u) >> 16) / 65536.0);
}

// packed (relative difference bits << 32 | row): atomicMax keeps the worst row of each class
template <typename T>
__global__ void k_compare_rows(int32_t const* __restrict__ row_vertex, T const* __restrict__ a, T const* __restrict__ b,
                               int32_t n_rows, int32_t n_hi, double tol, unsigned long long* __restrict__ worst /*[2]*/,
                               unsigned long long* __restrict__ n_bad /*[2]*/)
{
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    const int v     = row_vertex ? row_vertex[r] : (int)r;
    const double va = (double)a[v], vb = (double)b[v];
    const double den = fmax(fabs(va), 1e-300);
    const float rel  = (float)fmin(fabs(va - vb) / den, 1e30);
    const int cls    = r < n_hi ? 0 : 1;
    atomicMax(worst + cls, ((unsigned long long)__float_as_uint(rel) << 32) | (unsigned)r);
    if (rel > tol) atomicAdd(n_bad + cls, 1ull);
  }
}

}  // namespace

void sweep_scratch_t::init(handle_impl const& h, csx_t const& c)
{
  acc = make_dbuf<double>(acc_rows(c), h.stream);
  CUDA_TRY(cudaMemsetAsync(acc.data(), 0, sizeof(double) * acc_rows(c), h.stream));
  state = make_dbuf<pr_state_t>(1, h.stream);
  CUDA_TRY(cudaMemsetAsync(state.data(), 0, sizeof(pr_state_t), h.stream));
}

void sweep_scratch_t::set_init(handle_impl const& h, double init)
{
  pr_state_t hs{};
  hs.init = init;
  CUDA_TRY(cudaMemcpyAsync(state.data(), &hs, sizeof(pr_state_t), cudaMemcpyHostToDevice, h.stream));
  sync(h);  // hs is a stack variable
}

size_t padded_x_elems(int32_t n_vertices, size_t elem_size)
{
  const size_t slice = kHotSliceBytes / elem_size;
  const size_t W     = slice - kHotZeroPad;
  return ((size_t)n_vertices / W + 2) * slice;
}

template <typename T>
dbuf make_sweep_x(handle_impl const& h, int32_t n_vertices)
{
  const size_t n = padded_x_elems(n_vertices, sizeof(T));
  dbuf x         = make_dbuf<T>(n, h.stream);
  CUDA_TRY(cudaMemsetAsync(x.data(), 0, n * sizeof(T), h.stream));
  return x;
}

template <typename T>
void pull_sweep(handle_impl const& h, csx_t const& c, int32_t n_vertices, T const* x, T* y, sweep_scratch_t& sc, double alpha,
                bool use_weights, bool covered_rows_only, sweep_epilogue_t<T> const& epi)
{
  double* acc = sc.acc.as<double>();
  B200_EXPECTS(!epi.x_next || (epi.out_w && !covered_rows_only && epi.x_next != x), CUGRAPH_UNKNOWN_ERROR,
               "internal: a row epilogue needs out_w, every row and an x_next apart from x");
  B200_EXPECTS(y || (epi.x_next && !epi.y_old), CUGRAPH_UNKNOWN_ERROR, "internal: a sweep without y needs an epilogue");
  const row_epi_t<T> e{epi.out_w, epi.x_next, epi.y_old, sc.st()};
  if (sweep_layout_t const* L = sweep_layout(h, c, n_vertices, sizeof(T)))
    launch_sweep<T>(h, c, *L, x, y, acc, alpha, sc.st(), use_weights, covered_rows_only, e);
  else if (c.offs64)  // the plain sweep writes every row
    launch_pull_sweep<int64_t, T>(h, c, x, y, acc, alpha, sc.st(), use_weights, e);
  else
    launch_pull_sweep<int32_t, T>(h, c, x, y, acc, alpha, sc.st(), use_weights, e);
}

void prepare_pull_sweep(handle_impl const& h, csx_t const& c, int32_t nv, size_t es) { sweep_layout(h, c, nv, es); }

template dbuf make_sweep_x<float>(handle_impl const&, int32_t);
template dbuf make_sweep_x<double>(handle_impl const&, int32_t);
template void pull_sweep(handle_impl const&, csx_t const&, int32_t, float const*, float*, sweep_scratch_t&, double, bool, bool,
                         sweep_epilogue_t<float> const&);
template void pull_sweep(handle_impl const&, csx_t const&, int32_t, double const*, double*, sweep_scratch_t&, double, bool, bool,
                         sweep_epilogue_t<double> const&);

}  // namespace b200

using namespace b200;

extern "C" {

// Debug hook: y of the sweep PageRank would use on this graph (the shared-memory piece stream when the graph has one)
// against the plain sweep (k_spmv_hi + k_spmv_low, an independent implementation) on the same pseudo-random x.  out[0..3] = degree >= 32 rows:
// max relative difference, its row, that row's degree, rows above 1e-5; out[4..7] = the same for the degree < 32 rows.
cugraph_error_code_t cugraph_b200_debug_compare_sweeps(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph,
                                                       double* out, cugraph_error_t** error)
{
  return guarded(error, [&] {
    auto const& h = H(handle);
    auto* g       = G(graph);
    B200_EXPECTS(out != nullptr, CUGRAPH_INVALID_INPUT, "out is NULL");
    B200_EXPECTS(g->weight_type == FLOAT32, CUGRAPH_NOT_IMPLEMENTED, "single-GPU float32 graphs only");
    csx_t const& c = pull_view(h, *g);
    B200_EXPECTS(!c.offs64, CUGRAPH_NOT_IMPLEMENTED, "32-bit offsets only");
    const int32_t nv = g->n_vertices;
    dbuf x = make_sweep_x<float>(h, nv), y0 = make_dbuf<float>(nv, h.stream), y1 = make_dbuf<float>(nv, h.stream);
    B200_LAUNCH(h, (k_fill_pattern<float>), grid_for(nv), kBlock, 0, x.as<float>(), nv);
    sweep_scratch_t sc;
    sc.init(h, c);
    launch_pull_sweep<int32_t, float>(h, c, x.as<float>(), y0.as<float>(), sc.acc.as<double>(), 0.85, sc.st());
    pull_sweep<float>(h, c, nv, x.as<float>(), y1.as<float>(), sc, 0.85);
    dbuf res = make_dbuf<unsigned long long>(4, h.stream);
    CUDA_TRY(cudaMemsetAsync(res.data(), 0, 4 * sizeof(unsigned long long), h.stream));
    B200_LAUNCH(h, (k_compare_rows<float>), grid_for(c.n_rows), kBlock, 0, c.row_vertex.as<int32_t>(), y0.as<float>(), y1.as<float>(), c.n_rows, c.seg[0], 1e-5,
                res.as<unsigned long long>(), res.as<unsigned long long>() + 2);
    unsigned long long hres[4];
    CUDA_TRY(cudaMemcpyAsync(hres, res.data(), sizeof(hres), cudaMemcpyDeviceToHost, h.stream));
    sync(h);
    for (int k = 0; k < 2; ++k) {
      const unsigned bits = (unsigned)(hres[k] >> 32);
      float rel;
      std::memcpy(&rel, &bits, sizeof(rel));
      const int32_t row = (int32_t)(hres[k] & 0xffffffffu);
      int32_t offs[2]   = {0, 0};
      if (c.n_rows > 0)
        CUDA_TRY(cudaMemcpy(offs, c.offsets.as<int32_t>() + row, sizeof(offs), cudaMemcpyDeviceToHost));
      out[4 * k + 0] = rel;
      out[4 * k + 1] = row;
      out[4 * k + 2] = offs[1] - offs[0];
      out[4 * k + 3] = (double)hres[2 + k];
    }
    check_last("debug_compare_sweeps");
  });
}

}  // extern "C"
