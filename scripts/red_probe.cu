// Development probe (not part of the library): what does one warp-wide accumulation into an fp64 array cost the SM,
// by access shape and by the array's footprint against the L2 (50 MB on the H100)?  The piece-stream sweep issues one
// scattered RED.64 per piece; this measures the alternatives a row-aligned layout would use.  One 512-thread CTA per SM, every warp runs ITER operations
// on pseudo-random 32-row groups.  Output: ns per warp operation per SM (= time / (ITER * 16)), one JSON line per variant.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a scripts/red_probe.cu -o cugraph_b200/lib/red_probe
//   red_probe [MB [VARIANT]]   MB: accumulator footprint in MB (default 64); VARIANT: run only the variant of that name
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cuda_runtime.h>

constexpr int kThreads = 512;
constexpr int kWarps   = kThreads / 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned lcg(unsigned& s)
{
  s = s * 1664525u + 1013904223u;
  return s;
}
__device__ __forceinline__ unsigned mix(unsigned x)
{
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

template <int V>
__global__ void __launch_bounds__(kThreads, 1) k_probe(double* __restrict__ acc, unsigned rows, int iters, unsigned seed)
{
  __shared__ __align__(128) double stage[kWarps][2][128];  // 2 x 1 KiB per warp
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned s = seed + (blockIdx.x * kWarps + warp) * 7919u;  // warp-uniform stream
  float* accf = reinterpret_cast<float*>(acc);
  for (int it = 0; it < iters; ++it) {
    const unsigned r    = mix(lcg(s));
    const unsigned base = (r % (rows / 128)) * 128;  // 128-row aligned group start
    const double v      = (double)(r & 255) * 1e-9 + lane;
    if (V == 0) {  // scattered RED.64
      const unsigned row = mix(r + lane * 0x9e3779b9u) % rows;
      atomicAdd(acc + row, v);
    } else if (V == 1) {  // coalesced RED.64: 32 consecutive rows
      atomicAdd(acc + base + lane, v);
    } else if (V == 2) {  // coalesced, ~50 % of the lanes
      if ((r >> (lane & 15)) & 1) atomicAdd(acc + base + lane, v);
    } else if (V == 3) {  // coalesced, ~25 %
      if (((r >> (lane & 15)) & 1) && ((r >> (16 + (lane >> 1))) & 1)) atomicAdd(acc + base + lane, v);
    } else if (V == 4) {  // coalesced plain store
      acc[base + lane] = v;
    } else if (V == 5) {  // red.v2.f32 coalesced: 64 fp32 rows per warp
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(accf + base + 2 * lane), "f"((float)v), "f"((float)v + 1.f) : "memory");
    } else if (V == 6) {  // red.v4.f32 coalesced: 128 fp32 rows per warp
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(accf + base + 4 * lane), "f"((float)v), "f"((float)v + 1.f),
                   "f"((float)v + 2.f), "f"((float)v + 3.f)
                   : "memory");
    } else if (V == 7) {  // staged: STS.64 + one 256-byte bulk reduce per warp
      double* buf = stage[warp][it & 1];
      if (it >= 2) {
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        __syncwarp();
      }
      buf[lane] = v;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) {
        asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], 256;" ::"l"(acc + base), "r"(smem_u32(buf))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    } else if (V == 8) {  // staged: 4 x STS.64 + one 1 KiB bulk reduce per 4 operations (128 consecutive rows)
      double* buf = stage[warp][(it >> 2) & 1];
      if ((it & 3) == 0 && it >= 8) {
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        __syncwarp();
      }
      buf[(it & 3) * 32 + lane] = v;
      if ((it & 3) == 3) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
          asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], 1024;" ::"l"(acc + base),
                       "r"(smem_u32(buf))
                       : "memory");
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
      }
    } else if (V == 9) {  // scattered RED.32 (fp32)
      const unsigned row = mix(r + lane * 0x9e3779b9u) % rows;
      atomicAdd(accf + row, (float)v);
    } else if (V == 10) {  // coalesced RED.64, 64 rows per warp as two instructions
      atomicAdd(acc + base + lane, v);
      atomicAdd(acc + base + 32 + lane, v + 1.0);
    } else if (V == 11) {  // scattered RED.64, ~50 % of the lanes
      const unsigned row = mix(r + lane * 0x9e3779b9u) % rows;
      if ((r >> (lane & 15)) & 1) atomicAdd(acc + row, v);
    } else if (V == 12) {  // coalesced fp32 RED.32: 32 consecutive fp32 rows
      atomicAdd(accf + base + lane, (float)v);
    } else if (V == 13) {  // rows ascending but sparse inside a 256-row window (8 sectors x 4 lanes)
      const unsigned row = base + ((lane * 8 + (mix(r + lane) & 7)) & 127);
      atomicAdd(acc + row, v);
    }
  }
  if (V == 7 || V == 8) {
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

static const char* g_only = nullptr;  // run only this variant

template <int V>
void run(const char* name, double* acc, unsigned rows, int n_sm, int iters, double rows_per_op)
{
  if (g_only && std::strcmp(g_only, name)) return;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(e0);
    k_probe<V><<<n_sm, kThreads>>>(acc, rows, iters, 12345u + rep);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaError_t err = cudaGetLastError();
  const double ns_per_op = best * 1e6 / ((double)iters * kWarps);
  printf("{\"variant\": \"%s\", \"footprint_mb\": %.1f, \"ms\": %.4f, \"ns_per_warp_op_per_sm\": %.3f, \"cycles_at_1965\": %.2f, \"G_rows_per_s\": %.2f, \"err\": \"%s\"}\n", name,
         rows * 8.0 / (1 << 20), best, ns_per_op, ns_per_op * 1.965, rows_per_op * iters * kWarps * n_sm / (best * 1e6), cudaGetErrorString(err));
  fflush(stdout);
}

int main(int argc, char** argv)
{
  const double mb     = argc > 1 ? std::atof(argv[1]) : 64.0;
  const unsigned rows = (unsigned)(mb * (1 << 20) / 8) / 128 * 128;  // whole 128-row groups
  if (argc > 2) g_only = argv[2];
  int n_sm = 132;
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
  double* acc;
  cudaMalloc(&acc, (size_t)rows * sizeof(double));
  cudaMemset(acc, 0, (size_t)rows * sizeof(double));
  const int iters = 20000;
  run<0>("scattered_red64", acc, rows, n_sm, iters, 32);
  run<11>("scattered_red64_half_lanes", acc, rows, n_sm, iters, 16);
  run<9>("scattered_red32", acc, rows, n_sm, iters, 32);
  run<1>("coalesced_red64", acc, rows, n_sm, iters, 32);
  run<2>("coalesced_red64_half_lanes", acc, rows, n_sm, iters, 16);
  run<3>("coalesced_red64_quarter_lanes", acc, rows, n_sm, iters, 8);
  run<10>("coalesced_red64_x2", acc, rows, n_sm, iters, 64);
  run<13>("windowed_red64_4_per_sector", acc, rows, n_sm, iters, 32);
  run<12>("coalesced_red32", acc, rows, n_sm, iters, 32);
  run<4>("coalesced_st64", acc, rows, n_sm, iters, 32);
  run<5>("coalesced_red_v2_f32", acc, rows, n_sm, iters, 64);
  run<6>("coalesced_red_v4_f32", acc, rows, n_sm, iters, 128);
  run<7>("sts_bulk_reduce_256B", acc, rows, n_sm, iters, 32);
  run<8>("sts_bulk_reduce_1KiB", acc, rows, n_sm, iters, 32);
  return 0;
}
