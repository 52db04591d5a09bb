// Accessors for the CPU emulation build (libcugraph_c_emu.so): test infrastructure only, see emu/cuda_runtime.h.
#include "sweep_layout.cuh"

#include <algorithm>
#include <vector>

namespace b200 {
alignas(128) unsigned char smem_raw[256 * 1024];  // the dynamic shared memory of the one CTA that runs at a time
}  // namespace b200

using namespace b200;

#define EMU_EXPORT extern "C" __attribute__((visibility("default")))

// the schedule knobs are read from the environment when a handle is created; tests change the environment between cases
EMU_EXPORT void emu_reload_tuning(cugraph_resource_handle_t* handle)
{
  if (handle) reinterpret_cast<handle_impl*>(handle)->tune = tuning_t::from_env();
}

// primary orientation: pointers into the ("device" = host) arrays
EMU_EXPORT int emu_graph_primary(cugraph_graph_t* graph, int64_t* ints /*[8]: n_rows,nnz,offs64,nnz_hi,n_vertices,weighted,wsize,0*/,
                                 int32_t* seg /*[8]*/, void** ptrs /*[5]: offsets,indices,weights,ext_of_int,row_vertex*/)
{
  auto* g        = reinterpret_cast<graph_impl*>(graph);
  csx_t const& c = *g->primary;
  ints[0] = c.n_rows; ints[1] = c.nnz; ints[2] = c.offs64; ints[3] = c.nnz_hi; ints[4] = g->n_vertices;
  ints[5] = g->weighted; ints[6] = (int64_t)dtype_size(g->weight_type); ints[7] = 0;
  for (int k = 0; k <= kNumSeg; ++k) seg[k] = c.seg[k];
  ptrs[0] = c.offsets.data(); ptrs[1] = c.indices.data(); ptrs[2] = c.weights.data(); ptrs[3] = g->ext_of_int.data();
  ptrs[4] = c.row_vertex.data();
  return 0;
}

// piece stream of the primary orientation (built on first use)
EMU_EXPORT int emu_sweep_layout(const cugraph_resource_handle_t* handle, cugraph_graph_t* graph, int64_t* ints /*[12]*/,
                                void** ptrs /*[6]: ids, w, rows, chunks, phases, cta_phase*/)
{
  auto const& h  = H(handle);
  auto* g        = reinterpret_cast<graph_impl*>(graph);
  csx_t const& c = *g->primary;
  const size_t es = g->weighted ? dtype_size(g->weight_type) : 4;
  sweep_layout_t const* L = nullptr;
  try {
    L = sweep_layout(h, c, g->n_vertices, es);
  } catch (std::exception const& e) {
    std::fprintf(stderr, "emu_sweep_layout: %s\n", e.what());
    return 2;
  }
  if (!L) return 1;
  ints[0] = L->W; ints[1] = L->B; ints[2] = L->n_cov; ints[3] = L->nnz; ints[4] = L->n_steprows; ints[5] = L->n_rowslots;
  ints[6] = L->n_chunks; ints[7] = L->n_phases; ints[8] = (int64_t)L->n_bands * L->n_cta; ints[9] = L->bank_order; ints[10] = (int64_t)es;
  ints[11] = L->n_pieces;
  ptrs[0] = L->ids.data(); ptrs[1] = L->w.data(); ptrs[2] = L->rows.data(); ptrs[3] = L->chunks.data();
  ptrs[4] = L->phases.data(); ptrs[5] = L->cta_phase.data();
  return 0;
}

// the layout emu_sweep_layout built for elements of `es` bytes, or nullptr: the accessors below read it, never build it
static sweep_layout_t const* built_layout(cugraph_graph_t* graph, size_t es)
{
  csx_t const& c = *reinterpret_cast<graph_impl*>(graph)->primary;
  return c.sweep ? c.sweep->of(es).layout.get() : nullptr;
}

// row bands of that piece stream (call emu_sweep_layout first): returns n_bands and its CTAs per band (*n_cta);
// band_row / band_phase receive n_bands + 1 entries each when they hold at least `capacity`
EMU_EXPORT int emu_sweep_bands(cugraph_graph_t* graph, size_t es, int* n_cta, int32_t* band_row, int32_t* band_phase, size_t capacity)
{
  sweep_layout_t const* L = built_layout(graph, es);
  if (!L) return 0;
  *n_cta = L->n_cta;
  if ((size_t)L->n_bands + 1 <= capacity) {
    std::copy(L->band_row.begin(), L->band_row.end(), band_row);
    std::copy(L->band_phase.begin(), L->band_phase.end(), band_phase);
  }
  return L->n_bands;
}

// rows [0, n_str) of that piece stream are in it, the non-empty rows behind them are its tail; -1 without a layout
EMU_EXPORT int32_t emu_sweep_stream_rows(cugraph_graph_t* graph, size_t es)
{
  sweep_layout_t const* L = built_layout(graph, es);
  return L ? L->n_str : -1;
}

// tail layout of that piece stream: returns its runs (0 without a tail, -1 without a layout); runs receives n_runs + 1 x
// {degree, first_row, first_tile, first_unit, id_off} when it holds `capacity` entries, ptrs[2] = tail_ids, tail_w
EMU_EXPORT int emu_sweep_tail(cugraph_graph_t* graph, size_t es, int64_t* runs, size_t capacity, void** ptrs)
{
  sweep_layout_t const* L = built_layout(graph, es);
  if (!L) return -1;
  if (L->tail_runs.size() <= capacity)
    for (size_t k = 0; k < L->tail_runs.size(); ++k) {
      tail_run_t const& r = L->tail_runs[k];
      int64_t* o          = runs + 5 * k;
      o[0] = r.degree; o[1] = r.first_row; o[2] = r.first_tile; o[3] = r.first_unit; o[4] = r.id_off;
    }
  ptrs[0] = L->tail_ids.data();
  ptrs[1] = L->tail_w.data();
  return L->n_tail_runs;
}

EMU_EXPORT size_t emu_padded_x_elems(int32_t nv, size_t es) { return padded_x_elems(nv, es); }

// forget the cached layouts of the primary orientation (so that another set of knobs can be staged)
EMU_EXPORT void emu_reset_layouts(cugraph_graph_t* graph)
{
  reinterpret_cast<graph_impl*>(graph)->primary->sweep.reset();
}
