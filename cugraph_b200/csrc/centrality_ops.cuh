// The vertex passes of the sweep-based centralities (Katz, eigenvector, HITS): the per-iteration steps that follow the
// sweep, plus a sum and a scaling for the normalisations outside the loop.  One set of kernels, run by the single-GPU
// drivers (centrality.cu) over all vertices and by the multi-GPU owner steps (mg.cu) over a rank's owned slice.  Each adds
// its fp64 partials into a caller's device scalars (the multi-GPU launcher all-reduces them); a value is scaled as
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

// out[0] += sum v^2 (mode 0) | sum v (mode 1)
template <typename T>
__global__ void __launch_bounds__(kBlock) k_norm(T const* __restrict__ v, int32_t n, int mode, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  double s = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = (double)v[i];
    s += mode == 0 ? x * x : x;
  }
  s = block_sum(s, smem);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(out, s);
}

template <typename T>
__global__ void __launch_bounds__(kBlock) k_scale(T* __restrict__ v, int32_t n, double inv)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v[i] = scaled(v[i], inv);
}

// Katz: x_new = y + beta (y carries alpha from the sweep) ; out[0] += sum |x_new - x| ; out[1] += sum x_new^2 ; x = x_new
template <typename T>
__global__ void __launch_bounds__(kBlock)
k_katz_step(T const* __restrict__ y, T* __restrict__ x, int32_t n, double beta, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  double d = 0.0, s = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T nv = (T)((double)y[i] + beta);
    d += fabs((double)nv - (double)x[i]);
    s += (double)nv * (double)nv;
    x[i] = nv;
  }
  d = block_sum(d, smem);
  s = block_sum(s, smem);
  if (threadIdx.x == 0) {
    if (d != 0.0) atomicAdd(out, d);
    if (s != 0.0) atomicAdd(out + 1, s);
  }
}

// eigenvector, first half: y += x ; out[0] += sum y^2
template <typename T>
__global__ void __launch_bounds__(kBlock) k_eig_add(T* __restrict__ y, T const* __restrict__ x, int32_t n, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  double s = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T v = y[i] + x[i];
    y[i]      = v;
    s += (double)v * (double)v;
  }
  s = block_sum(s, smem);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(out, s);
}

// eigenvector, second half: y *= 1 / sqrt(sumsq[0]) ; out[0] += sum |y - x| ; x = y
template <typename T>
__global__ void __launch_bounds__(kBlock)
k_eig_scale(T* __restrict__ y, T* __restrict__ x, int32_t n, double const* __restrict__ sumsq, double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  const double inv = 1.0 / sqrt(sumsq[0]);
  double d         = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T v = scaled(y[i], inv);
    d += fabs((double)v - (double)x[i]);
    y[i] = v;
    x[i] = v;
  }
  d = block_sum(d, smem);
  if (threadIdx.x == 0 && d != 0.0) atomicAdd(out, d);
}

// HITS: out[0] = max(out[0], max hubs), out[1] = max(out[1], max auth)
template <typename T>
__global__ void __launch_bounds__(kBlock) k_hits_max(T const* __restrict__ hubs, T const* __restrict__ auth, int32_t n, double* __restrict__ out)
{
  double mh = 0.0, ma = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double h = (double)hubs[i], a = (double)auth[i];
    mh = h > mh ? h : mh;
    ma = a > ma ? a : ma;
  }
  warp_max_into(mh, out);
  warp_max_into(ma, out + 1);
}

// HITS: hubs *= 1 / mx[0] ; auth *= 1 / mx[1] ; out[0] += sum |hubs - prev|
template <typename T>
__global__ void __launch_bounds__(kBlock)
k_hits_scale(T* __restrict__ hubs, T* __restrict__ auth, T const* __restrict__ prev, int32_t n, double const* __restrict__ mx,
             double* __restrict__ out)
{
  __shared__ double smem[kBlock / 32];
  const double inv_h = 1.0 / mx[0], inv_a = 1.0 / mx[1];
  double d = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const T h = scaled(hubs[i], inv_h);
    hubs[i]   = h;
    auth[i]   = scaled(auth[i], inv_a);
    d += fabs((double)h - (double)prev[i]);
  }
  d = block_sum(d, smem);
  if (threadIdx.x == 0 && d != 0.0) atomicAdd(out, d);
}

}  // namespace
}  // namespace b200
