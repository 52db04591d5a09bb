// The vector passes of the sweep-based centralities (Katz, eigenvector, HITS): sums, maxima, scaling and differences over
// a vertex array, with fp64 partials added into a caller's device scalars.  Shared by the single-GPU drivers
// (centrality.cu) and the multi-GPU owner steps (mg.cu), so that both round and sum the same way: a value is scaled as
// (T)((double)v * inv), and differences and norms are taken in fp64.
#pragma once
#include "common.cuh"

namespace b200 {
namespace {

// *out = max(*out, the warp's largest m); m >= 0, so the bits compare like unsigned integers
__device__ __forceinline__ void warp_max_into(double m, double* out)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double t = __shfl_xor_sync(0xffffffffu, m, o);
    m              = t > m ? t : m;
  }
  if ((threadIdx.x & 31) == 0 && m > 0.0)
    atomicMax(reinterpret_cast<unsigned long long*>(out), (unsigned long long)__double_as_longlong(m));
}

template <typename T>
__device__ __forceinline__ T scaled(T v, double inv)
{
  return (T)((double)v * inv);
}

// out[0] += sum |a - b| ; optionally b <- a (the next sweep's input)
template <typename T>
__global__ void __launch_bounds__(kBlock) k_abs_diff(T const* __restrict__ a, T* __restrict__ b, int32_t n, int copy, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  double d = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    d += fabs((double)a[i] - (double)b[i]);
    if (copy) b[i] = a[i];
  }
  d = block_sum(d, smem);
  if (threadIdx.x == 0 && d != 0.0) atomicAdd(out, d);
}

template <typename T>
__global__ void __launch_bounds__(kBlock) k_add_vec(T* __restrict__ y, T const* __restrict__ add, int32_t n)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] += add[i];
}

// out[0] += sum v^2 (mode 0) | sum v (mode 1) ; out[1] = max v (mode 2, values are non-negative: integer compare of the bits)
template <typename T>
__global__ void __launch_bounds__(kBlock) k_norm(T const* __restrict__ v, int32_t n, int mode, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  double s = 0.0, m = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = (double)v[i];
    s += mode == 0 ? x * x : x;
    m = x > m ? x : m;
  }
  if (mode == 2) {
    warp_max_into(m, out + 1);
    return;
  }
  s = block_sum(s, smem);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(out, s);
}

template <typename T>
__global__ void __launch_bounds__(kBlock) k_scale(T* __restrict__ v, int32_t n, double inv)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v[i] = scaled(v[i], inv);
}

}  // namespace
}  // namespace b200
