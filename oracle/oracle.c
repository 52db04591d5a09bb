/*
 * oracle.c — CPU restatement of the reference's sequential test oracles for the PageRank / BFS /
 * SSSP hot path.  TEST INFRASTRUCTURE ONLY: nothing under cugraph_b200/ may link or call this.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it.
 *
 * Pinned against: the reference's C-API golden vectors (cpp/tests/c_api/{pagerank,bfs,sssp}_test.c)
 * and the pylibcugraph karate goldens (python/pylibcugraph/pylibcugraph/tests/test_pagerank.py),
 * see tests/test_oracle_golden.py.  The reference library itself cannot be built here (needs
 * raft/rmm/cuco/CCCL-3, none vendored) so there is no oracle/_ref.
 *
 * Each function cites the reference code it follows.  Plain C99, no dependencies; OpenMP pragmas
 * (optional, -fopenmp) parallelise only loops whose iterations are independent, so results do not
 * depend on the thread count except for the reductions that say so.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

int oracle_num_threads(void)
{
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ------------------------------------------------------------------------------------------
 * COO -> compressed sparse (counting sort by major, stable; minors then sorted per row).
 * Follows what the reference's staging produces for the algorithms: offsets[major], minors
 * sorted within a row (cpp/src/structure/create_graph_from_edgelist_impl.cuh:1528-1657,
 * sort_adjacency_list).  Weights travel with their edge.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t minor;
  double w;
} oracle_pair_t;

static int cmp_pair(const void* a, const void* b)
{
  const oracle_pair_t* x = (const oracle_pair_t*)a;
  const oracle_pair_t* y = (const oracle_pair_t*)b;
  if (x->minor != y->minor) return (x->minor < y->minor) ? -1 : 1;
  if (x->w != y->w) return (x->w < y->w) ? -1 : 1;
  return 0;
}

int oracle_coo_to_csx(int64_t num_edges,
                      int32_t num_vertices,
                      const int32_t* major,
                      const int32_t* minor,
                      const double* w /* may be NULL */,
                      int64_t* offsets /* [V+1] out */,
                      int32_t* indices /* [E] out */,
                      double* w_out /* [E] out or NULL */)
{
  memset(offsets, 0, sizeof(int64_t) * ((size_t)num_vertices + 1));
  for (int64_t e = 0; e < num_edges; ++e) {
    if (major[e] < 0 || major[e] >= num_vertices || minor[e] < 0 || minor[e] >= num_vertices)
      return -1;
    offsets[major[e] + 1]++;
  }
  for (int32_t v = 0; v < num_vertices; ++v)
    offsets[v + 1] += offsets[v];
  int64_t* cursor = (int64_t*)malloc(sizeof(int64_t) * ((size_t)num_vertices + 1));
  if (!cursor) return -2;
  memcpy(cursor, offsets, sizeof(int64_t) * ((size_t)num_vertices + 1));
  for (int64_t e = 0; e < num_edges; ++e) {
    int64_t p  = cursor[major[e]]++;
    indices[p] = minor[e];
    if (w_out) w_out[p] = w ? w[e] : 1.0;
  }
  free(cursor);
#pragma omp parallel
  {
    oracle_pair_t* tmp = NULL;
    int64_t cap        = 0;
#pragma omp for schedule(dynamic, 1024)
    for (int32_t v = 0; v < num_vertices; ++v) {
      int64_t lo = offsets[v], hi = offsets[v + 1], n = hi - lo;
      if (n < 2) continue;
      if (n > cap) {
        free(tmp);
        cap = n * 2;
        tmp = (oracle_pair_t*)malloc(sizeof(oracle_pair_t) * (size_t)cap);
      }
      for (int64_t i = 0; i < n; ++i) {
        tmp[i].minor = indices[lo + i];
        tmp[i].w     = w_out ? w_out[lo + i] : 0.0;
      }
      qsort(tmp, (size_t)n, sizeof(oracle_pair_t), cmp_pair);
      for (int64_t i = 0; i < n; ++i) {
        indices[lo + i] = tmp[i].minor;
        if (w_out) w_out[lo + i] = tmp[i].w;
      }
    }
    free(tmp);
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * PageRank — follows pagerank_reference, cpp/tests/link_analysis/pagerank_test.cpp:33-121
 * (CSC input: offsets over destinations, indices = sources), cross-checked against the GPU
 * driver cpp/src/link_analysis/pagerank_impl.cuh:224-329 for the loop-exit rule:
 *   iter++ ; stop if diff_sum < epsilon, else stop if iter >= max_iterations ;
 *   converged = iter < max_iterations.
 * Arithmetic is double throughout (result_t = double instantiation of the reference oracle).
 * precomputed out-weight sums / initial guess / personalization follow the driver's semantics
 * (pagerank_impl.cuh:180-198, 289-309; c_api/pagerank.cpp:179-226: the C API does NOT normalise
 * the initial guess, it copies it).
 * ------------------------------------------------------------------------------------------ */
int oracle_pagerank(const int64_t* offsets /* CSC [V+1] */,
                    const int32_t* indices /* sources [E] */,
                    const double* weights /* [E] or NULL */,
                    int32_t num_vertices,
                    const double* precomputed_out_w /* [V] or NULL */,
                    const int32_t* pers_vertices /* or NULL */,
                    const double* pers_values,
                    int32_t pers_size,
                    int has_initial_guess /* pageranks[] holds it */,
                    double alpha,
                    double epsilon,
                    int64_t max_iterations,
                    double* pageranks /* [V] in/out */,
                    int64_t* iterations_out,
                    int* converged_out)
{
  const int32_t V = num_vertices;
  if (V == 0) {
    if (iterations_out) *iterations_out = 0;
    if (converged_out) *converged_out = 1;
    return 0;
  }
  if (!has_initial_guess) {
    for (int32_t i = 0; i < V; ++i)
      pageranks[i] = 1.0 / (double)V;
  }
  double pers_sum = 0.0;
  if (pers_vertices) {
    for (int32_t i = 0; i < pers_size; ++i)
      pers_sum += pers_values[i];
    if (!(pers_sum > 0.0)) return -1;
  }
  double* out_w = (double*)calloc((size_t)V, sizeof(double));
  double* old   = (double*)malloc(sizeof(double) * (size_t)V);
  if (!out_w || !old) return -2;
  if (precomputed_out_w) {
    memcpy(out_w, precomputed_out_w, sizeof(double) * (size_t)V);
  } else {
    for (int32_t i = 0; i < V; ++i)
      for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j)
        out_w[indices[j]] += weights ? weights[j] : 1.0;
  }
  int64_t iter = 0;
  while (1) {
    memcpy(old, pageranks, sizeof(double) * (size_t)V);
    double dangling = 0.0;
    for (int32_t i = 0; i < V; ++i)
      if (out_w[i] == 0.0) dangling += old[i];
    const double unvarying = pers_vertices ? 0.0 : (dangling * alpha + (1.0 - alpha)) / (double)V;
#pragma omp parallel for schedule(dynamic, 4096)
    for (int32_t i = 0; i < V; ++i) {
      double acc = 0.0;
      for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) {
        int32_t nbr = indices[j];
        double w    = weights ? weights[j] : 1.0;
        acc += alpha * old[nbr] * (w / out_w[nbr]);
      }
      pageranks[i] = acc + unvarying;
    }
    if (pers_vertices) {
      for (int32_t i = 0; i < pers_size; ++i)
        pageranks[pers_vertices[i]] +=
          (dangling * alpha + (1.0 - alpha)) * (pers_values[i] / pers_sum);
    }
    double diff = 0.0;
    for (int32_t i = 0; i < V; ++i)
      diff += fabs(pageranks[i] - old[i]);
    iter++;
    if (diff < epsilon) break;
    if (iter >= max_iterations) break;
  }
  free(out_w);
  free(old);
  if (iterations_out) *iterations_out = iter;
  if (converged_out) *converged_out = (iter < max_iterations);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * BFS — follows bfs_reference, cpp/tests/traversal/bfs_test.cpp:33-70 (CSR input), generalised
 * to several sources (cugraph_bfs accepts a source list; every source starts at depth 0,
 * cpp/src/traversal/bfs_impl.cuh:270-285).  Unreached: distance INT32_MAX, predecessor -1.
 * ------------------------------------------------------------------------------------------ */
int oracle_bfs(const int64_t* offsets,
               const int32_t* indices,
               int32_t num_vertices,
               const int32_t* sources,
               int32_t num_sources,
               int32_t depth_limit,
               int32_t* distances,
               int32_t* predecessors)
{
  const int32_t V = num_vertices;
  for (int32_t i = 0; i < V; ++i) {
    distances[i]    = INT32_MAX;
    predecessors[i] = -1;
  }
  int32_t* cur = (int32_t*)malloc(sizeof(int32_t) * (size_t)(V > 0 ? V : 1));
  int32_t* nxt = (int32_t*)malloc(sizeof(int32_t) * (size_t)(V > 0 ? V : 1));
  if (!cur || !nxt) return -2;
  int32_t ncur = 0, nnxt = 0, depth = 0;
  for (int32_t s = 0; s < num_sources; ++s) {
    if (sources[s] < 0 || sources[s] >= V) {
      free(cur);
      free(nxt);
      return -1;
    }
    if (distances[sources[s]] != 0) {
      distances[sources[s]] = 0;
      cur[ncur++]           = sources[s];
    }
  }
  while (ncur > 0) {
    nnxt = 0;
    for (int32_t k = 0; k < ncur; ++k) {
      int32_t row = cur[k];
      for (int64_t j = offsets[row]; j != offsets[row + 1]; ++j) {
        int32_t nbr = indices[j];
        if (distances[nbr] == INT32_MAX) {
          distances[nbr]    = depth + 1;
          predecessors[nbr] = row;
          nxt[nnxt++]       = nbr;
        }
      }
    }
    int32_t* t = cur;
    cur        = nxt;
    nxt        = t;
    ncur       = nnxt;
    ++depth;
    if (depth >= depth_limit) break;
  }
  free(cur);
  free(nxt);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * SSSP — follows sssp_reference (Dijkstra with cutoff), cpp/tests/traversal/sssp_test.cpp:34-74.
 * `use_float` selects the weight_t the additions are performed in (float or double) so that
 * distances are bit-comparable with a GPU run in the same type.  Binary heap with lazy deletion
 * in place of std::priority_queue (same pop order on (distance, vertex)).
 * Unreached: distance FLT_MAX / DBL_MAX, predecessor -1.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  double d;
  int32_t v;
} heap_item_t;

static int heap_less(heap_item_t a, heap_item_t b)
{
  return (a.d < b.d) || (a.d == b.d && a.v < b.v);
}

int oracle_sssp(const int64_t* offsets,
                const int32_t* indices,
                const double* weights,
                int32_t num_vertices,
                int32_t source,
                double cutoff,
                int use_float,
                double* distances,
                int32_t* predecessors)
{
  const int32_t V  = num_vertices;
  const double inf = use_float ? (double)FLT_MAX : DBL_MAX;
  if (source < 0 || source >= V) return -1;
  if (cutoff > inf) cutoff = inf;
  /* the cutoff is compared in weight_t: the reference rounds it first (cpp/src/c_api/sssp.cpp:109,
   * static_cast<weight_t>(cutoff_)).  A double cutoff above a float distance d that rounds down to d must
   * leave the vertex at d unreached.  (Clamped first: the conversion is only defined within float's range.) */
  if (use_float) cutoff = (double)(float)cutoff;
  for (int32_t i = 0; i < V; ++i) {
    distances[i]    = inf;
    predecessors[i] = -1;
  }
  int64_t cap       = 1024, n = 0;
  heap_item_t* heap = (heap_item_t*)malloc(sizeof(heap_item_t) * (size_t)cap);
  if (!heap) return -2;
  distances[source] = 0.0;
  heap[n++]         = (heap_item_t){0.0, source};
  while (n > 0) {
    heap_item_t top = heap[0];
    heap[0]         = heap[--n];
    {
      int64_t i = 0;
      while (1) {
        int64_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < n && heap_less(heap[l], heap[m])) m = l;
        if (r < n && heap_less(heap[r], heap[m])) m = r;
        if (m == i) break;
        heap_item_t t = heap[i];
        heap[i]       = heap[m];
        heap[m]       = t;
        i             = m;
      }
    }
    if (top.d > distances[top.v]) continue;
    for (int64_t j = offsets[top.v]; j != offsets[top.v + 1]; ++j) {
      int32_t nbr = indices[j];
      double nd   = use_float ? (double)((float)top.d + (float)weights[j]) : top.d + weights[j];
      double thr  = distances[nbr] < cutoff ? distances[nbr] : cutoff;
      if (nd < thr) {
        distances[nbr]    = nd;
        predecessors[nbr] = top.v;
        if (n == cap) {
          cap *= 2;
          heap = (heap_item_t*)realloc(heap, sizeof(heap_item_t) * (size_t)cap);
          if (!heap) return -2;
        }
        int64_t i = n++;
        heap[i]   = (heap_item_t){nd, nbr};
        while (i > 0) {
          int64_t p = (i - 1) / 2;
          if (!heap_less(heap[i], heap[p])) break;
          heap_item_t t = heap[i];
          heap[i]       = heap[p];
          heap[p]       = t;
          i             = p;
        }
      }
    }
  }
  free(heap);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * One float32 pull SpMV sweep  y = init + alpha * sum x[src] (*w)  over a CSC — the unit the
 * CPU baseline times (same arithmetic the GPU kernel does per iteration, a5 in SURVEY §8a:
 * per_v_transform_reduce_incoming_e with PageRank's e_op, pagerank_impl.cuh:262-287).
 * ------------------------------------------------------------------------------------------ */
void oracle_spmv_f32(const int64_t* offsets,
                     const int32_t* indices,
                     const float* weights /* or NULL */,
                     int32_t num_vertices,
                     const float* x,
                     float alpha,
                     float init,
                     float* y)
{
#pragma omp parallel for schedule(dynamic, 4096)
  for (int32_t i = 0; i < num_vertices; ++i) {
    double acc = 0.0;
    if (weights) {
      for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j)
        acc += (double)x[indices[j]] * (double)weights[j];
    } else {
      for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j)
        acc += (double)x[indices[j]];
    }
    y[i] = (float)(acc * (double)alpha + (double)init);
  }
}
