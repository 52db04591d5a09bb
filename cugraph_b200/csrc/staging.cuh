// Launch grids and CUB wrappers of the one-time staging passes, shared by graph_build.cu and sweep_layout.cu.  Everything
// lives in an anonymous namespace, as in advance.cuh: every translation unit gets its own instantiations.
#pragma once
#include "common.cuh"

#include <cub/cub.cuh>
#include <type_traits>

namespace b200 {
namespace {

constexpr int kBlock = 256;

inline int grid_for(int64_t n, int per_thread = 1)
{
  int64_t b = (n + (int64_t)kBlock * per_thread - 1) / ((int64_t)kBlock * per_thread);
  return (int)std::min<int64_t>(std::max<int64_t>(b, 1), 1 << 20);
}

__global__ void k_iota64(int64_t n, uint32_t* v)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    v[i] = (uint32_t)i;
}

template <typename K, typename Val>
void sort_pairs(handle_impl const& h, K const* kin, K* kout, Val const* vin, Val* vout, int64_t n, int begin_bit, int end_bit)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, n, begin_bit, end_bit, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.data(), bytes, kin, kout, vin, vout, n, begin_bit, end_bit, h.stream));
  h.launches += 4;
}

inline void exclusive_scan_i32(handle_impl const& h, int32_t const* in, int32_t* out, int64_t n)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, in, out, n, h.stream));
  h.launches += 2;
}

// out = the elements of in[0, n) whose flag is set, in order; returns how many.  `in` is a T const* unless the caller names
// another input iterator as In (In is not deduced from the argument).
template <typename T, typename In = T const*>
int64_t select_flagged(handle_impl const& h, std::common_type_t<In> in, uint8_t const* flags, T* out, int64_t n)
{
  dbuf d_count(sizeof(int64_t), h.stream);
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, bytes, in, flags, out, d_count.as<int64_t>(), n, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.data(), bytes, in, flags, out, d_count.as<int64_t>(), n, h.stream));
  h.launches += 2;
  int64_t cnt = 0;
  CUDA_TRY(cudaMemcpyAsync(&cnt, d_count.data(), sizeof(int64_t), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  return cnt;
}

inline int bits_for(int64_t n)
{
  int b = 1;
  while ((1ll << b) < n) ++b;
  return b;
}

}  // namespace
}  // namespace b200
