// CUB wrappers of the one-time staging passes, shared by graph_build.cu and sweep_layout.cu (and PageRank's expensive input
// check, pagerank.cu).  Everything
// lives in an anonymous namespace, as in advance.cuh: every translation unit gets its own instantiations.
#pragma once
#include "common.cuh"

#include <cub/cub.cuh>
#include <type_traits>

namespace b200 {
namespace {

template <typename K>
void sort_keys(handle_impl const& h, K const* in, K* out, int64_t n, int begin_bit, int end_bit)
{
  size_t bytes = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, bytes, in, out, n, begin_bit, end_bit, h.stream));
  dbuf tmp(bytes, h.stream);
  CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp.data(), bytes, in, out, n, begin_bit, end_bit, h.stream));
  h.launches += 4;
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
  return read_back(h, d_count.as<int64_t>());
}

inline int bits_for(int64_t n)
{
  int b = 1;
  while ((1ll << b) < n) ++b;
  return b;
}

}  // namespace
}  // namespace b200
