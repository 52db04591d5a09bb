// RMAT edge-list generator on the device (the role of cpp/src/generators/generate_rmat_edgelist.cuh:28-112 and
// scramble.cuh:44-67), behind the C ABI as cugraph_b200_generate_rmat_edgelist.  Sampling rule of the reference: for every edge
// and every bit from scale-1 down to 0 two uniforms r0, r1;  src_bit = r0 > a + b;  dst_bit = r1 > (src_bit ? c / (1 - (a + b))
// : a / (a + b));  clip-and-flip moves an edge that is about to leave the diagonal into the upper triangle back below it;
// the Graph500 scramble permutes the ids.  The reference draws its uniforms from raft's device RNG (not vendored): the
// STREAM here is a counter-based one — 24-bit uniforms from a 64-bit mix of (seed, edge, bit) — restated in numpy by
// oracle/rmat.py:rmat_edgelist_counter, against which the output is checked bit for bit (tests/test_generators_*.py).
#include "common.cuh"

namespace b200 {
namespace {

__host__ __device__ __forceinline__ unsigned long long rmat_mix64(unsigned long long z)
{
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__host__ __device__ __forceinline__ uint32_t bitreverse32(uint32_t v)
{
  v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
  v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
  v = ((v >> 4) & 0x0F0F0F0Fu) | ((v & 0x0F0F0F0Fu) << 4);
  v = ((v >> 8) & 0x00FF00FFu) | ((v & 0x00FF00FFu) << 8);
  return (v >> 16) | (v << 16);
}

// 32-bit variant of detail::scramble (scramble.cuh:44-67)
__host__ __device__ __forceinline__ uint32_t scramble32(uint32_t v, int lgn)
{
  const uint32_t s0 = 282475248u, s1 = 2617694917u;
  v += s0 + s1;
  v *= (s0 | 0x11493211u);  // low 32 bits of 0x4519840211493211
  v = bitreverse32(v) >> (32 - lgn);
  v *= (s1 | 0x02C843A5u);  // low 32 bits of 0x3050852102C843A5
  v = bitreverse32(v) >> (32 - lgn);
  return v;
}

// edges [first, first + n) of the stream: edge first + e lands at src[e], dst[e]
__global__ void k_rmat_edges(int scale, unsigned long long first, long long n, unsigned long long seed, float a_plus_b,
                             float a_norm, float c_norm, int clip_and_flip, int scramble, int32_t* __restrict__ src,
                             int32_t* __restrict__ dst)
{
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long ge = first + (unsigned long long)e;
    uint32_t s = 0, d = 0;
    for (int bit = scale - 1; bit >= 0; --bit) {
      const unsigned long long r = rmat_mix64(seed ^ (ge * 64ull + (unsigned)bit));
      const float r0 = (float)(r >> 40) * (1.0f / 16777216.0f);
      const float r1 = (float)((r >> 8) & 0xffffffull) * (1.0f / 16777216.0f);
      int sb = r0 > a_plus_b;
      int db = r1 > (sb ? c_norm : a_norm);
      if (clip_and_flip && s == d && !sb && db) {
        sb = 1;
        db = 0;
      }
      s |= (uint32_t)sb << bit;
      d |= (uint32_t)db << bit;
    }
    if (scramble) {
      s = scramble32(s, scale);
      d = scramble32(d, scale);
    }
    src[e] = (int32_t)s;
    dst[e] = (int32_t)d;
  }
}

// counter-based uniforms for edge weights / edge types: value i = lo + u_i * (hi - lo) with u_i = the top 24 (float) or 53
// (double) bits of mix64(seed ^ i) as a fraction; integers: lo + mix64(seed ^ i) % (hi - lo).  Values [first, first + n) of
// the stream: value first + i lands at out[i]
template <typename T>
__global__ void k_uniform_real(T* __restrict__ out, unsigned long long first, long long n, unsigned long long seed, double lo,
                               double hi)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long r = rmat_mix64(seed ^ (first + (unsigned long long)i));
    const double u = sizeof(T) == 4 ? (double)(r >> 40) * (1.0 / 16777216.0) : (double)(r >> 11) * (1.0 / 9007199254740992.0);
    out[i]         = (T)(lo + u * (hi - lo));
  }
}
__global__ void k_uniform_int(int32_t* __restrict__ out, unsigned long long first, long long n, unsigned long long seed,
                              long long lo, long long hi)
{
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = (int32_t)(lo + (long long)(rmat_mix64(seed ^ (first + (unsigned long long)i)) % (unsigned long long)(hi - lo)));
}

void generate_uniform(handle_impl const& h, uint64_t seed, uint64_t first, double lo, double hi,
                      cugraph_type_erased_device_array_view_t* out)
{
  B200_EXPECTS(out != nullptr, CUGRAPH_INVALID_INPUT, "NULL argument");
  auto const* ov = V(out);
  B200_EXPECTS(ov->type == FLOAT32 || ov->type == FLOAT64 || ov->type == INT32, CUGRAPH_INVALID_INPUT,
               "generate_uniform writes FLOAT32, FLOAT64 or INT32 arrays");
  B200_EXPECTS(hi > lo, CUGRAPH_INVALID_INPUT, "Invalid input argument: the range [lo, hi) is empty");
  if (ov->size == 0) return;
  const int grid = grid_for((int64_t)ov->size, 1, h.sm_count * 16);
  const auto f   = (unsigned long long)first;
  if (ov->type == FLOAT32)
    B200_LAUNCH(h, (k_uniform_real<float>), grid, kBlock, 0, (float*)ov->data, f, (long long)ov->size, (unsigned long long)seed, lo, hi);
  else if (ov->type == FLOAT64)
    B200_LAUNCH(h, (k_uniform_real<double>), grid, kBlock, 0, (double*)ov->data, f, (long long)ov->size, (unsigned long long)seed, lo,
                hi);
  else
    B200_LAUNCH(h, k_uniform_int, grid, kBlock, 0, (int32_t*)ov->data, f, (long long)ov->size, (unsigned long long)seed, (long long)lo,
                (long long)hi);
  check_last("generate_uniform");
}

void generate_rmat(handle_impl const& h, size_t scale, uint64_t first, size_t num_edges, double a, double b, double c, uint64_t seed,
                   bool_t clip_and_flip, bool_t scramble_vertex_ids, cugraph_type_erased_device_array_view_t* src,
                   cugraph_type_erased_device_array_view_t* dst)
{
  B200_EXPECTS(src && dst, CUGRAPH_INVALID_INPUT, "NULL argument");
  auto const* sv = V(src);
  auto const* dv = V(dst);
  B200_EXPECTS(scale >= 1 && scale <= 31, CUGRAPH_INVALID_INPUT, "scale must be in [1, 31] (32-bit vertex ids)");
  B200_EXPECTS(sv->type == INT32 && dv->type == INT32, CUGRAPH_INVALID_INPUT, "src / dst must be INT32 arrays");
  B200_EXPECTS(sv->size >= num_edges && dv->size >= num_edges, CUGRAPH_INVALID_INPUT, "src / dst shorter than num_edges");
  // the reference's checks (generate_rmat_edgelist.cuh:41-47)
  B200_EXPECTS(a >= 0.0 && b >= 0.0 && c >= 0.0 && a + b + c <= 1.0, CUGRAPH_INVALID_INPUT,
               "Invalid input argument: a, b, c should be non-negative and a + b + c should not exceed 1.0.");
  if (num_edges == 0) return;
  const double ab = a + b;
  const float a_norm = (float)(ab > 0.0 ? a / ab : 0.0), c_norm = (float)((1.0 - ab) > 0.0 ? c / (1.0 - ab) : 0.0);
  const int grid = grid_for((int64_t)num_edges, 1, h.sm_count * 16);
  B200_LAUNCH(h, k_rmat_edges, grid, kBlock, 0, (int)scale, (unsigned long long)first, (long long)num_edges, (unsigned long long)seed,
              (float)ab, a_norm, c_norm, clip_and_flip == TRUE ? 1 : 0, scramble_vertex_ids == TRUE ? 1 : 0, (int32_t*)sv->data,
              (int32_t*)dv->data);
  check_last("generate_rmat_edgelist");
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" cugraph_error_code_t cugraph_b200_generate_uniform(const cugraph_resource_handle_t* handle, uint64_t seed, double lo,
                                                              double hi, cugraph_type_erased_device_array_view_t* out,
                                                              cugraph_error_t** error)
{
  return guarded(error, [&] { generate_uniform(H(handle), seed, 0, lo, hi, out); });
}

extern "C" cugraph_error_code_t cugraph_b200_generate_uniform_at(const cugraph_resource_handle_t* handle, uint64_t seed,
                                                                 uint64_t first, double lo, double hi,
                                                                 cugraph_type_erased_device_array_view_t* out,
                                                                 cugraph_error_t** error)
{
  return guarded(error, [&] { generate_uniform(H(handle), seed, first, lo, hi, out); });
}

extern "C" cugraph_error_code_t cugraph_b200_generate_rmat_edgelist(const cugraph_resource_handle_t* handle, size_t scale,
                                                                    size_t num_edges, double a, double b, double c,
                                                                    uint64_t seed, bool_t clip_and_flip,
                                                                    bool_t scramble_vertex_ids,
                                                                    cugraph_type_erased_device_array_view_t* src,
                                                                    cugraph_type_erased_device_array_view_t* dst,
                                                                    cugraph_error_t** error)
{
  return guarded(error, [&] {
    generate_rmat(H(handle), scale, 0, num_edges, a, b, c, seed, clip_and_flip, scramble_vertex_ids, src, dst);
  });
}

extern "C" cugraph_error_code_t cugraph_b200_generate_rmat_edgelist_at(const cugraph_resource_handle_t* handle, size_t scale,
                                                                       uint64_t first_edge, size_t num_edges, double a, double b,
                                                                       double c, uint64_t seed, bool_t clip_and_flip,
                                                                       bool_t scramble_vertex_ids,
                                                                       cugraph_type_erased_device_array_view_t* src,
                                                                       cugraph_type_erased_device_array_view_t* dst,
                                                                       cugraph_error_t** error)
{
  return guarded(error, [&] {
    generate_rmat(H(handle), scale, first_edge, num_edges, a, b, c, seed, clip_and_flip, scramble_vertex_ids, src, dst);
  });
}
