// The shared-memory pull sweep: y[v] = init + alpha * sum_{(u->v)} x[u] * w(u,v) for EVERY row, gathers served from
// shared memory — per_v_transform_reduce_incoming_e specialised to reduce_op::plus and PageRank's e_op (reference
// cpp/include/cugraph/prims/detail/per_v_transform_reduce_e.cuh:389-885, cpp/src/link_analysis/pagerank_impl.cuh:262-287).
//
// Why: the plain sweep (spmv.cuh) is bound by the L2 -> SM path: every gather of x[src] costs a 32-byte L2 sector for
// 4 useful bytes.  Here the source space is cut into blocks of W
// vertices whose x slice (192 KiB) a persistent CTA keeps in shared memory (TMA bulk copies + mbarrier), and the
// adjacency is re-laid as a stream of PIECES with 16-bit local column ids (sweep_layout_t, sweep_layout.cuh).
//
// Execution structure (a kernel with one batch of id / row loads in flight per warp, nothing while it processed them,
// spent most of its stall samples waiting on those loads, and some at CTA barriers):
//   * one 512-thread CTA per SM, 128 registers per thread.  A warp works on CHUNKS (a few step-rows of one kind, ~1-3 KiB of
//     ids + rows) and is double-buffered in REGISTERS: the 128-bit loads of chunk i+1 are issued before chunk i is
//     processed, its header before that, the draw of its index before that — no global-memory latency sits on the
//     critical path of a warp, and 16 warps x ~3 KiB are in flight per SM at all times (Little: 32 KiB needed).
//   * warps draw chunks from a per-phase cursor (one atomic per chunk, two draws ahead); there is no CTA barrier inside a
//     PHASE (= the chunks of one block in this CTA's range): barriers only where the slice changes.
//   * a CTA that finishes its own phases joins the phase with the most chunks left (same cursor: work stealing).
//   * a lane sums the 8 gathers of a slot as an fp32 tree and converts ONCE (the round-1 kernel issued one F2F + one DADD per
//     gather: 20 % of its instructions); slots, pieces and rows accumulate in fp64.
//   * one fp64 RED per piece into acc[row] (L2); the pieces of a hub row that fill a whole warp are summed by shuffles
//     first.  k_sweep_finish turns acc into y, clears it and resets the cursors.
//   * the rows are split into bands whose accumulators fit in the L2 (sweep_layout.cuh); the sweep runs band by band, k_sweep over
//     the band's phases, then k_sweep_finish over its rows while their accumulators are still in the L2.
//   * on large graphs the rows of small in-degree (the tail, sweep_layout.cuh) are not in the stream: one k_sweep_tail launch
//     gathers their few edges directly from a layout of their own (runs of equal in-degree, lane-interleaved: no RED, and
//     fewer stream rows need fewer bands), the hubs' x from a shared-memory copy of the first column block.  It runs on a
//     share of the SMs beside the bands, from the handle's side stream (launch_sweep), or after them on every SM.
#pragma once
#include "spmv.cuh"
#include "sweep_layout.cuh"

namespace b200 {

constexpr int kSweepThreads = 512;  // 16 warps x 128 registers, two chunk buffers per warp (384 threads x 3 buffers: no faster)
constexpr int kSweepWarps   = kSweepThreads / 32;
constexpr int kSweepDynSmem = kHotSliceBytes;
constexpr int kTmaPiece     = 16 * 1024;  // bytes per bulk copy of the slice
constexpr int kStealMin     = 12;         // chunks a phase must have left for another CTA to load its slice and join

#ifndef B200_HOST_EMU
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity)
{
  asm volatile(
    "{\n"
    ".reg .pred p;\n"
    "WAIT_LOOP:\n"
    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
    "@p bra DONE;\n"
    "bra WAIT_LOOP;\n"
    "DONE:\n"
    "}\n" ::"r"(smem_u32(bar)),
    "r"(parity)
    : "memory");
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                 smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ uint4 ld_stream_v4(const void* p)
{
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
// L2 eviction policies (createpolicy).  The 0.8 GB id / row stream is read once: marked evict-FIRST it leaves the L2 to the
// accumulators (fp64, 8 bytes per row), whose REDs carry an evict-LAST policy (without it most RED sectors missed the L2
// and fetched their line from DRAM first).  A run-time choice per RED cost as much as the policy gains, so both are
// unconditional.
__device__ __forceinline__ unsigned long long make_l2_policy_evict_first()
{
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint4 ld_stream_v4(const void* p, unsigned long long pol)
{
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint2 ld_stream_v2(const void* p, unsigned long long pol)
{
  uint2 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0, %1}, [%2], %3;" : "=r"(v.x), "=r"(v.y) : "l"(p), "l"(pol));
  return v;
}
// fp64 accumulation with an L2 eviction policy on the accumulator line
__device__ __forceinline__ void red_acc(double* p, double v, unsigned long long acc_pol)
{
  asm volatile("red.global.add.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(acc_pol) : "memory");
}
__device__ __forceinline__ unsigned long long make_l2_policy_evict_last()
{
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ int ld_stream_i32(const int* p, unsigned long long pol)
{
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint2 ld_stream_v2(const void* p)
{
  uint2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ int ld_volatile(const int* p)
{
  int v;
  asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
#define B200_DYN_SMEM(name) extern __shared__ __align__(128) unsigned char name[]
#else  // host emulation (emu/cuda_runtime.h): a bulk copy is a memcpy by the issuing thread, waiting on the mbarrier is a
       // CTA barrier (every thread of the CTA waits on it in this kernel)
inline void mbar_init(uint64_t*, unsigned) {}
inline void mbar_expect_tx(uint64_t*, unsigned) {}
inline void mbar_wait(uint64_t*, unsigned) { __syncthreads(); }
inline void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, uint64_t*) { std::memcpy(dst_smem, src_gmem, bytes); }
inline uint4 ld_stream_v4(const void* p)
{
  uint4 v;
  std::memcpy(&v, p, sizeof(v));
  return v;
}
inline uint2 ld_stream_v2(const void* p)
{
  uint2 v;
  std::memcpy(&v, p, sizeof(v));
  return v;
}
inline int ld_volatile(const int* p) { return *p; }
inline unsigned long long make_l2_policy_evict_first() { return 0ull; }
inline uint4 ld_stream_v4(const void* p, unsigned long long) { return ld_stream_v4(p); }
inline uint2 ld_stream_v2(const void* p, unsigned long long) { return ld_stream_v2(p); }
inline int ld_stream_i32(const int* p, unsigned long long) { return *p; }
inline void red_acc(double* p, double v, unsigned long long) { *p += v; }
inline unsigned long long make_l2_policy_evict_last() { return 0ull; }
#define B200_DYN_SMEM(name) extern unsigned char name[] /* one CTA at a time: emu/emu_debug.cpp defines b200::smem_raw */
#endif

// the slice of column block `block`, x[block * W, (block + 1) * W), into shared memory at `dst` by TMA bulk copies of
// kTmaPiece bytes, completion signalled on `bar`; one thread issues it
template <typename T>
__device__ __forceinline__ void load_slice(unsigned char* dst, T const* x, int block, int W, uint64_t* bar)
{
  const unsigned bytes = (unsigned)(W * sizeof(T));
  mbar_expect_tx(bar, bytes);
  const unsigned char* src = reinterpret_cast<const unsigned char*>(x + (size_t)block * W);
  for (unsigned o = 0; o < bytes; o += kTmaPiece)
    tma_bulk_g2s(dst + o, src + o, (bytes - o) < (unsigned)kTmaPiece ? (bytes - o) : (unsigned)kTmaPiece, bar);
}

// ------------------------------------------------------------------------------------------
// per-lane arithmetic
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned lo16(unsigned v) { return v & 0xffffu; }
__device__ __forceinline__ unsigned hi16(unsigned v) { return v >> 16; }
__device__ __forceinline__ unsigned comp(uint4 const& v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w)); }

// the two entries packed in one 32-bit word of ids (weights wp[0], wp[1])
template <typename T, bool WEIGHTED>
__device__ __forceinline__ T pair_sum(unsigned ids, T const* __restrict__ sx, T const* wp)
{
  T a = sx[lo16(ids)], b = sx[hi16(ids)];
  if (WEIGHTED) {
    a *= wp[0];
    b *= wp[1];
  }
  return a + b;
}
// the 8 entries of a lane slot: summed as a tree in T (float: fp32 adds, ONE conversion), returned in fp64
template <typename T, bool WEIGHTED>
__device__ __forceinline__ double slot_sum(uint4 const& ids, T const* __restrict__ sx, T const* wp)
{
  const T a = pair_sum<T, WEIGHTED>(ids.x, sx, wp), b = pair_sum<T, WEIGHTED>(ids.y, sx, wp + 2);
  const T c = pair_sum<T, WEIGHTED>(ids.z, sx, wp + 4), d = pair_sum<T, WEIGHTED>(ids.w, sx, wp + 6);
  return (double)((a + b) + (c + d));
}

template <typename T>
__device__ __forceinline__ void load_w8(T (&wv)[8], T const* __restrict__ w, size_t slot)
{
#pragma unroll
  for (int k = 0; k < 8; ++k) wv[k] = ld_stream(w + slot * 8 + k);
}

// end of an F8 group (full 64-entry pieces): consecutive lanes may hold pieces of the same (hub) row — suffix-sum inside
// the runs first, run heads emit
__device__ __forceinline__ void emit_runs(double acc, int row, double* __restrict__ acc_out, int lane, unsigned long long acc_pol)
{
  const int r0 = __shfl_sync(0xffffffffu, row, 0);
  if (__all_sync(0xffffffffu, row == r0)) {  // 32 pieces of one hub row
    acc = warp_sum(acc);
    if (lane == 0 && r0 >= 0) red_acc(acc_out + r0, acc, acc_pol);
    return;
  }
  const int left = __shfl_up_sync(0xffffffffu, row, 1);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, acc, o);
    const int rn    = __shfl_down_sync(0xffffffffu, row, o);
    if (lane + o < 32 && rn == row) acc += nb;
  }
  if (lane > 0 && left == row) row = -1;  // not the head of its run
  if (row >= 0) red_acc(acc_out + row, acc, acc_pol);
}

// ------------------------------------------------------------------------------------------
// a chunk in registers: up to 8 x 128 bits of ids / rows + 2 row words; what sits where depends on the kind
//   S  x 2 groups : q[3g] ids, q[3g+1], q[3g+2] the 8 rows
//   Q  x 4 groups : q[2g] ids, q[2g+1] the 4 rows
//   H  x 4 groups : q[g] ids, rows of groups (0,1) in q[4], of (2,3) in q[5]
//   F1 x 6 groups : q[g] ids, rows in q[6], q[7]
//   F2 x 3, F3 x 2: q[g*C+j] ids, rows in q[6]
//   F4 x 2        : q[g*4+j] ids, rows r0, r1
//   F5..F8 x 1    : q[j] ids, row r0
// ------------------------------------------------------------------------------------------
struct chunk_regs_t {
  uint4 q[8];
  int r0, r1;
};

struct sweep_ptrs_t {
  uint4 const* __restrict__ ids;
  int32_t const* __restrict__ rows;
  void const* __restrict__ w;
  double* __restrict__ acc;
  unsigned long long pol;      // L2 eviction policy of the stream loads
  unsigned long long acc_pol;  // of the accumulator REDs
};

template <int C, int G>
__device__ __forceinline__ void load_F(chunk_regs_t& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p, int lane)
{
  uint4 const* ip   = p.ids + ((size_t)(unsigned)ch.sr_begin << 5) + lane;
  int32_t const* rp = p.rows + (size_t)(unsigned)ch.row_begin + lane;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (g < ch.n_groups) {
#pragma unroll
      for (int j = 0; j < C; ++j) b.q[g * C + j] = ld_stream_v4(ip + ((g * C + j) << 5), p.pol);
      const int r = ld_stream_i32(rp + (g << 5), p.pol);
      if (C >= 4) {
        if (g == 0) b.r0 = r; else b.r1 = r;
      } else if (C == 1) {
        if (g == 0) b.q[6].x = r; else if (g == 1) b.q[6].y = r; else if (g == 2) b.q[6].z = r; else if (g == 3) b.q[6].w = r;
        else if (g == 4) b.q[7].x = r; else b.q[7].y = r;
      } else {
        if (g == 0) b.q[6].x = r; else if (g == 1) b.q[6].y = r; else b.q[6].z = r;
      }
    }
  }
}

template <typename T, bool WEIGHTED, int C, int G>
__device__ __forceinline__ void process_F(chunk_regs_t const& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p,
                                          T const* __restrict__ sx, int lane)
{
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (g < ch.n_groups) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < C; ++j) {
        T wv[8];
        if (WEIGHTED) load_w8<T>(wv, (T const*)p.w, ((size_t)(unsigned)(ch.sr_begin + g * C + j) << 5) + lane);
        s += slot_sum<T, WEIGHTED>(b.q[g * C + j], sx, wv);
      }
      int row;
      if (C >= 4) row = g == 0 ? b.r0 : b.r1;
      else if (C == 1) row = (int)(g < 4 ? comp(b.q[6], g) : comp(b.q[7], g - 4));
      else row = (int)comp(b.q[6], g);
      if (C == 8) emit_runs(s, row, p.acc, lane, p.acc_pol);
      else if (row >= 0) red_acc(p.acc + row, s, p.acc_pol);
    }
  }
}

// narrow kinds: ROWS rows per lane and step-row (S: 8, Q: 4, H: 2), G groups (= step-rows) per chunk
template <int ROWS, int G>
__device__ __forceinline__ void load_N(chunk_regs_t& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p, int lane)
{
  uint4 const* ip   = p.ids + ((size_t)(unsigned)ch.sr_begin << 5) + lane;
  int32_t const* rp = p.rows + (size_t)(unsigned)ch.row_begin + (size_t)lane * ROWS;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (g < ch.n_groups) {
      const uint4 ids = ld_stream_v4(ip + (g << 5), p.pol);
      if (ROWS == 8) {
        b.q[3 * g]     = ids;
        b.q[3 * g + 1] = ld_stream_v4(rp + g * 256, p.pol);
        b.q[3 * g + 2] = ld_stream_v4(rp + g * 256 + 4, p.pol);
      } else if (ROWS == 4) {
        b.q[2 * g]     = ids;
        b.q[2 * g + 1] = ld_stream_v4(rp + g * 128, p.pol);
      } else {
        b.q[g]        = ids;
        const uint2 r = ld_stream_v2(rp + g * 64, p.pol);
        uint4& dst    = b.q[4 + (g >> 1)];
        if (g & 1) {
          dst.z = r.x;
          dst.w = r.y;
        } else {
          dst.x = r.x;
          dst.y = r.y;
        }
      }
    }
  }
}

template <typename T, bool WEIGHTED, int ROWS, int G>
__device__ __forceinline__ void process_N(chunk_regs_t const& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p,
                                          T const* __restrict__ sx, int lane)
{
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (g < ch.n_groups) {
      T wv[8];
      if (WEIGHTED) load_w8<T>(wv, (T const*)p.w, ((size_t)(unsigned)(ch.sr_begin + g) << 5) + lane);
      if (ROWS == 8) {
        const uint4 ids = b.q[3 * g];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const unsigned word = comp(ids, k >> 1);
          T v                 = sx[(k & 1) ? hi16(word) : lo16(word)];
          if (WEIGHTED) v *= wv[k];
          const int row = (int)comp(b.q[3 * g + 1 + (k >> 2)], k & 3);
          if (row >= 0) red_acc(p.acc + row, (double)v, p.acc_pol);
        }
      } else if (ROWS == 4) {
        const uint4 ids = b.q[2 * g];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const T v     = pair_sum<T, WEIGHTED>(comp(ids, k), sx, wv + 2 * k);
          const int row = (int)comp(b.q[2 * g + 1], k);
          if (row >= 0) red_acc(p.acc + row, (double)v, p.acc_pol);
        }
      } else {
        const uint4 ids = b.q[g];
        const uint4 rr  = b.q[4 + (g >> 1)];
        const T v0      = pair_sum<T, WEIGHTED>(ids.x, sx, wv) + pair_sum<T, WEIGHTED>(ids.y, sx, wv + 2);
        const T v1      = pair_sum<T, WEIGHTED>(ids.z, sx, wv + 4) + pair_sum<T, WEIGHTED>(ids.w, sx, wv + 6);
        const int row0 = (int)((g & 1) ? rr.z : rr.x), row1 = (int)((g & 1) ? rr.w : rr.y);
        if (row0 >= 0) red_acc(p.acc + row0, (double)v0, p.acc_pol);
        if (row1 >= 0) red_acc(p.acc + row1, (double)v1, p.acc_pol);
      }
    }
  }
}

// issue every load of the chunk (nothing is waited for); kind < 0: nothing to load
__device__ __forceinline__ void chunk_load(chunk_regs_t& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p, int lane)
{
  switch (ch.kind) {
    case kKindS: load_N<8, 2>(b, ch, p, lane); break;
    case kKindQ: load_N<4, 4>(b, ch, p, lane); break;
    case kKindH: load_N<2, 4>(b, ch, p, lane); break;
    case kKindF1: load_F<1, 6>(b, ch, p, lane); break;
    case kKindF1 + 1: load_F<2, 3>(b, ch, p, lane); break;
    case kKindF1 + 2: load_F<3, 2>(b, ch, p, lane); break;
    case kKindF1 + 3: load_F<4, 2>(b, ch, p, lane); break;
    case kKindF1 + 4: load_F<5, 1>(b, ch, p, lane); break;
    case kKindF1 + 5: load_F<6, 1>(b, ch, p, lane); break;
    case kKindF1 + 6: load_F<7, 1>(b, ch, p, lane); break;
    case kKindF1 + 7: load_F<8, 1>(b, ch, p, lane); break;
    default: break;
  }
}

template <typename T, bool WEIGHTED>
__device__ __forceinline__ void chunk_process(chunk_regs_t const& b, sweep_chunk_t const& ch, sweep_ptrs_t const& p,
                                              T const* __restrict__ sx, int lane)
{
  switch (ch.kind) {
    case kKindS: process_N<T, WEIGHTED, 8, 2>(b, ch, p, sx, lane); break;
    case kKindQ: process_N<T, WEIGHTED, 4, 4>(b, ch, p, sx, lane); break;
    case kKindH: process_N<T, WEIGHTED, 2, 4>(b, ch, p, sx, lane); break;
    case kKindF1: process_F<T, WEIGHTED, 1, 6>(b, ch, p, sx, lane); break;
    case kKindF1 + 1: process_F<T, WEIGHTED, 2, 3>(b, ch, p, sx, lane); break;
    case kKindF1 + 2: process_F<T, WEIGHTED, 3, 2>(b, ch, p, sx, lane); break;
    case kKindF1 + 3: process_F<T, WEIGHTED, 4, 2>(b, ch, p, sx, lane); break;
    case kKindF1 + 4: process_F<T, WEIGHTED, 5, 1>(b, ch, p, sx, lane); break;
    case kKindF1 + 5: process_F<T, WEIGHTED, 6, 1>(b, ch, p, sx, lane); break;
    case kKindF1 + 6: process_F<T, WEIGHTED, 7, 1>(b, ch, p, sx, lane); break;
    case kKindF1 + 7: process_F<T, WEIGHTED, 8, 1>(b, ch, p, sx, lane); break;
    default: break;
  }
}

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
template <typename T>
struct sweep_args_t {
  sweep_ptrs_t p;
  sweep_chunk_t const* __restrict__ chunks;
  sweep_phase_t const* __restrict__ phases;
  int32_t const* __restrict__ cta_phase;
  int* __restrict__ cursor;
  T const* __restrict__ x;
  pr_state_t const* __restrict__ st;
  int ph_lo, ph_hi;  // the band's phases; a CTA only steals inside them (a later band's accumulators would enter the L2 early)
  int W;
};

// ---- chunk supply of a warp.  Chunks are drawn from the phase's cursor in BATCHES of consecutive chunks (lane j holds
// the header of chunk base + j, one coalesced load), sized by what is left (remaining / 64, 1..8: long streams first,
// single chunks at the end of a phase so that the warps finish together).  The chain draw -> headers -> ids is three
// dependent round trips through L2 / HBM (~3 us); the draw of batch b+2 and the headers of batch b+1 are in flight while
// batch b is processed, the ids of chunk i+1 while chunk i is (with one chunk per stage a warp spent most of its stall
// samples on these three waits).
constexpr int kDrawMax = 8;

__device__ __forceinline__ int draw_want(int n, int seen)
{
  const int w = (n - seen) >> 6;
  return w < 1 ? 1 : (w > kDrawMax ? kDrawMax : w);
}
// lane 0 draws; the value is broadcast (draw_get) only when it is needed, a batch later
__device__ __forceinline__ int draw_issue(int* cursor, int want, int lane, bool more)
{
  int k = 0x3fffffff;
  if (more && lane == 0) k = atomicAdd(cursor, want);
  return k;
}
__device__ __forceinline__ int draw_get(int raw) { return __shfl_sync(0xffffffffu, raw, 0); }

__device__ __forceinline__ uint4 batch_headers(sweep_chunk_t const* __restrict__ chunks, int first, int cnt, int lane)
{
  uint4 v = make_uint4(0u, 0u, 0u, 0xffffffffu);  // kind = -1
  if (lane < cnt) v = ld_stream_v4(chunks + first + lane);
  return v;
}

// The headers of the current batch sit in a per-warp shared-memory ring (read back with one broadcast LDS per chunk);
// the headers of the next batch are a load in flight into `pend`, which is only touched at the next batch switch (kept in
// registers and copied with moves, ptxas hoisted the moves above the switch branch and every chunk waited for the load).
struct chunk_supply_t {
  sweep_chunk_t const* __restrict__ chunks;  // of the phase
  int* cursor;
  uint4* ring;  // [2][kDrawMax] of this warp
  int n;        // chunks in the phase
  uint4 pend;
  int cnt_cur, cnt_nxt, j, slot;
  int raw_nn, want_nn;  // draw in flight for the batch after `pend`

  __device__ __forceinline__ void start(sweep_chunk_t const* __restrict__ c, int* cur, uint4* warp_ring, int n_chunks, int lane)
  {
    chunks = c;
    cursor = cur;
    ring   = warp_ring;
    n      = n_chunks;
    const int w0 = draw_want(n, 0);
    const int r0 = draw_issue(cursor, w0, lane, true), r1 = draw_issue(cursor, w0, lane, true);
    const int b0 = draw_get(r0);
    cnt_cur      = b0 < n ? (n - b0 < w0 ? n - b0 : w0) : 0;
    const uint4 v0 = batch_headers(chunks, b0, cnt_cur, lane);
    const int b1 = draw_get(r1);
    cnt_nxt      = b1 < n ? (n - b1 < w0 ? n - b1 : w0) : 0;
    pend         = batch_headers(chunks, b1, cnt_nxt, lane);
    want_nn      = draw_want(n, b1 < n ? b1 + w0 : n);
    raw_nn       = draw_issue(cursor, want_nn, lane, b1 + w0 < n);
    j            = 0;
    slot         = 0;
    __syncwarp();  // the previous phase's readers of the ring are done
    if (lane < kDrawMax) ring[lane] = v0;
    __syncwarp();
  }
  __device__ __forceinline__ sweep_chunk_t next(int lane)
  {
    if (j == cnt_cur && cnt_cur > 0) {  // warp-uniform: the batch is used up
      slot ^= 1;
      if (lane < kDrawMax) ring[slot * kDrawMax + lane] = pend;  // its load was issued a batch ago
      __syncwarp();
      cnt_cur = cnt_nxt;
      j       = 0;
      const int b2 = draw_get(raw_nn);
      cnt_nxt      = b2 < n ? (n - b2 < want_nn ? n - b2 : want_nn) : 0;
      pend         = batch_headers(chunks, b2, cnt_nxt, lane);
      const int w3 = draw_want(n, b2 < n ? b2 + want_nn : n);
      raw_nn       = draw_issue(cursor, w3, lane, b2 + want_nn < n);
      want_nn      = w3;
    }
    sweep_chunk_t ch;
    ch.kind = -1;
    ch.n_groups = ch.sr_begin = ch.row_begin = 0;
    if (cnt_cur > 0) {
      const uint4 h = ring[slot * kDrawMax + j];
      ++j;
      ch.sr_begin  = (int)h.x;
      ch.row_begin = (int)h.y;
      ch.n_groups  = (int)h.z;
      ch.kind      = (int)h.w;
    }
    return ch;
  }
};

template <typename T, bool WEIGHTED>
__global__ void __launch_bounds__(kSweepThreads, 1) k_sweep(sweep_args_t<T> a)
{
  B200_DYN_SMEM(smem_raw);
  T* sx = reinterpret_cast<T*>(smem_raw);
  __shared__ uint64_t bar;
  __shared__ int s_best;
  __shared__ uint4 s_ring[kSweepWarps][2 * kDrawMax];
  if (a.st->done) return;
  a.p.pol        = make_l2_policy_evict_first();
  a.p.acc_pol    = make_l2_policy_evict_last();
  const int lane = threadIdx.x & 31;
  const int me   = (int)blockIdx.x;
  if (threadIdx.x == 0) mbar_init(&bar, 1);
  if (threadIdx.x < kHotZeroPad) sx[a.W + threadIdx.x] = (T)0;  // the zero columns every slice ends with
  const int own_lo = a.cta_phase[me], own_hi = a.cta_phase[me + 1];  // cta_phase: this band's entries
  int next_own    = own_lo;
  unsigned parity = 0;
  int cur_block   = -1;
  while (true) {
    // ---- which phase next: the own ones in order, then the phase of another CTA with the most chunks left
    int p = -1;
    if (next_own < own_hi) {
      p = next_own++;
    } else {
      if (threadIdx.x == 0) s_best = 0;
      __syncthreads();
      int best = 0;
      for (int q = a.ph_lo + (int)threadIdx.x; q < a.ph_hi; q += kSweepThreads) {
        if (q >= own_lo && q < own_hi) continue;
        const sweep_phase_t ph = a.phases[q];
        const int left         = (ph.chunk_end - ph.chunk_begin) - ld_volatile(a.cursor + q);
        if (left >= kStealMin && left > best) best = left;
      }
      if (best > 0) atomicMax(&s_best, best);
      __syncthreads();
      const int win = s_best;
      __syncthreads();
      if (win > 0) {
        if (threadIdx.x == 0) s_best = a.ph_hi;
        __syncthreads();
        for (int q = a.ph_lo + (int)threadIdx.x; q < a.ph_hi; q += kSweepThreads) {
          if (q >= own_lo && q < own_hi) continue;
          const sweep_phase_t ph = a.phases[q];
          const int left         = (ph.chunk_end - ph.chunk_begin) - ld_volatile(a.cursor + q);
          if (left >= kStealMin && left * 2 >= win) atomicMin(&s_best, q);
        }
        __syncthreads();
        p = s_best < a.ph_hi ? s_best : -1;
      }
    }
    __syncthreads();  // every warp is done with the previous phase's slice (and has read s_best)
    if (p < 0) break;
    const sweep_phase_t ph = a.phases[p];
    const int n            = ph.chunk_end - ph.chunk_begin;
    const bool fresh       = ph.block != cur_block;
    if (fresh) {
      if (threadIdx.x == 0) load_slice(smem_raw, a.x, ph.block, a.W, &bar);
      cur_block = ph.block;
    }
    // ---- the phase: chunk i is processed while the loads of i+1, the header of i+2 and the draw of i+3 are in flight
    chunk_supply_t sup;
    sup.start(a.chunks + ph.chunk_begin, a.cursor + p, s_ring[threadIdx.x >> 5], n, lane);
    sweep_chunk_t hA = sup.next(lane);
    sweep_chunk_t hB = sup.next(lane);
    chunk_regs_t A, B;
    chunk_load(A, hA, a.p, lane);
    if (fresh) {
      mbar_wait(&bar, parity);
      parity ^= 1;
    }
    while (hA.kind >= 0) {
      chunk_load(B, hB, a.p, lane);  // loads of chunk i+1
      const sweep_chunk_t hC = sup.next(lane);
      chunk_process<T, WEIGHTED>(A, hA, a.p, sx, lane);
      if (hB.kind < 0) break;
      chunk_load(A, hC, a.p, lane);
      const sweep_chunk_t hD = sup.next(lane);
      chunk_process<T, WEIGHTED>(B, hB, a.p, sx, lane);
      hA = hC;
      hB = hD;
    }
  }
}

// the epilogue of rows r, r + 1 of a float sweep without row_vertex, their out_w given: y_old read, x_next written as float2
__device__ __forceinline__ void epi_row_pair(row_epi_t<float> const& e, int r, float v0, float v1, float2 ow, epi_sums_t& s)
{
  *reinterpret_cast<float2*>(e.x_next + r) = make_float2(ow.x == 0.f ? v0 : v0 / ow.x, ow.y == 0.f ? v1 : v1 / ow.y);
  if (ow.x == 0.f) s.dangling += (double)v0;
  if (ow.y == 0.f) s.dangling += (double)v1;
  if (e.y_old) {
    const float2 o = *reinterpret_cast<float2 const*>(e.y_old + r);
    s.diff += fabs((double)v0 - (double)o.x) + fabs((double)v1 - (double)o.y);
  }
}

// y[row] = acc * alpha + init for the rows [row_lo, n_rows): acc for the stream rows (< n_cov, the caller passes n_str), init
// for the empty rows behind them (and the row epilogue of each, if any); clears their accumulators and the n_phases
// cursors.  row_lo is a multiple of kBandRowAlign.  A warp handles 64 kFinishSteps consecutive rows in steps of 64: every
// step is one 512-byte load + one 512-byte store of accumulators and one 256-byte store of y per warp (lane = two rows),
// all loads issued before the first use, the epilogue's out_w among them.  (Eight CONSECUTIVE rows per thread looked the
// same on paper and ran at 2.3 TB/s: every warp-wide 128-bit access then touched sixteen 128-byte lines for a quarter of
// their bytes.)
template <typename T, int kFinishSteps>
__global__ void __launch_bounds__(256)
k_sweep_finish(double* __restrict__ acc, int row_lo, int n_cov, int n_rows, T* __restrict__ y, int32_t const* __restrict__ row_vertex,
               double alpha, int* __restrict__ cursor, int n_phases, pr_state_t const* __restrict__ st, row_epi_t<T> epi)
{
  static_assert(kBandRowAlign % (64 * kFinishSteps) == 0, "a warp's rows must not straddle a band bound");
  if (st->done) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_phases) cursor[t] = 0;
  const int lane = threadIdx.x & 31;
  const int base = row_lo + (t >> 5) * (64 * kFinishSteps) + 2 * lane;  // first of this lane's two rows in step 0
  if (base - 2 * lane >= n_rows) return;
  const double init = st->init;
  epi_sums_t sums;
  double2 q[kFinishSteps];
  T ow[kFinishSteps][2];  // the epilogue's out_w of the lane's two rows
#pragma unroll
  for (int k = 0; k < kFinishSteps; ++k) {
    const int r = base + 64 * k;
    q[k]        = make_double2(0.0, 0.0);
    if (r + 1 < n_cov) q[k] = *reinterpret_cast<double2*>(acc + r);
    else if (r < n_cov) q[k].x = acc[r];
    ow[k][0] = ow[k][1] = (T)0;
    if (epi.x_next) {
      if (sizeof(T) == 4 && !row_vertex && r + 1 < n_rows) {
        const float2 o = *reinterpret_cast<float2 const*>(epi.out_w + r);
        ow[k][0]       = (T)o.x;
        ow[k][1]       = (T)o.y;
      } else {
        if (r < n_rows) ow[k][0] = epi.out_w[row_vertex ? row_vertex[r] : r];
        if (r + 1 < n_rows) ow[k][1] = epi.out_w[row_vertex ? row_vertex[r + 1] : r + 1];
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kFinishSteps; ++k) {
    const int r = base + 64 * k;
    if (r + 1 < n_cov) *reinterpret_cast<double2*>(acc + r) = make_double2(0.0, 0.0);
    else if (r < n_cov) acc[r] = 0.0;
    const T v0 = (T)(q[k].x * alpha + init), v1 = (T)(q[k].y * alpha + init);
    bool paired = false;
    if constexpr (sizeof(T) == 4) {
      if (!row_vertex && r + 1 < n_rows) {
        if (y) *reinterpret_cast<float2*>(y + r) = make_float2(v0, v1);
        if (epi.x_next) epi_row_pair(epi, r, v0, v1, make_float2((float)ow[k][0], (float)ow[k][1]), sums);
        paired = true;
      }
    }
    if (!paired) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (r + j < n_rows) {
          const int v = row_vertex ? row_vertex[r + j] : r + j;
          store_row(y, epi, v, j ? v1 : v0, epi_in_t<T>{ow[k][j], epi.y_old ? epi.y_old[v] : (T)0}, sums);
        }
      }
    }
  }
  epi_flush(epi, sums);  // the early return above is the whole warp's
}

// The tail rows [n_str, n_cov) from the tail layout (sweep_layout.cuh), then y = init for the empty rows [n_cov, empty_hi).  Its
// sources are mostly hubs (RMAT-24: 47 % of them in the first column block), and a plain row kernel pays a 32-byte L2 sector
// for each of those 4-byte gathers: persistent CTAs (one per SM) keep x[0, W) in shared memory, loaded once by TMA bulk
// copies as in k_sweep, and gather the other sources from global memory with an evict-LAST hint (x is reused across the
// tail, the ids are read once and marked evict-first).  Warps draw WORK UNITS (a few tiles of one run, ~24 entries per lane)
// from one cursor, so every SM works until the tail is done; a unit's ids are one contiguous lane-interleaved span, loaded by
// one fully used 128-byte line per warp-wide load, and the next unit's ids are in flight while a unit is processed.  The
// entries of a lane are its row's: the row sum is made in registers (products in T, batches of 8 summed in fp64 as a tree,
// rounded once) and stored, no RED and no accumulator.  The processing is instantiated per in-degree d (registers are
// indexed statically).
constexpr int kTailThreads = 512;  // 16 warps, up to 128 registers: two units of ids and one unit of gathers per lane
constexpr int kTailBatch   = 8;

#ifndef B200_HOST_EMU
__device__ __forceinline__ float ld_keep(float const* p, unsigned long long pol)
{
  float v;
  asm("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ double ld_keep(double const* p, unsigned long long pol)
{
  double v;
  asm("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  return v;
}
#else
inline float ld_keep(float const* p, unsigned long long) { return *p; }
inline double ld_keep(double const* p, unsigned long long) { return *p; }
#endif

template <typename T>
struct tail_args_t {
  tail_run_t const* __restrict__ runs;  // n_runs + 1
  int32_t const* __restrict__ ids;
  T const* __restrict__ w;  // or nullptr
  T const* __restrict__ x;
  T* __restrict__ y;
  int32_t const* __restrict__ row_vertex;
  int* __restrict__ cursor;  // this launch's slot of the tail cursor
  int* __restrict__ spent;   // the other slot, left behind by the launch before: cleared for the next one
  pr_state_t const* __restrict__ st;
  int n_runs, empty_hi, W;
  double alpha;
  row_epi_t<T> epi;
};

struct tail_unit_t {  // warp-uniform; d = 0: no unit
  int d, n_tiles, row0, row_end;
  long long base;  // first entry in tail_ids
};

__device__ __forceinline__ tail_unit_t tail_unit(tail_run_t const* runs, int n_runs, int u)
{
  tail_unit_t t{0, 0, 0, 0, 0};
  if (u >= runs[n_runs].first_unit) return t;
  int r = 0;
  while (u >= runs[r + 1].first_unit) ++r;
  const tail_run_t R = runs[r];
  const int per      = tail_unit_tiles(R.degree);
  const int tile     = (u - R.first_unit) * per;  // inside the run
  t.d                = R.degree;
  const int left     = runs[r + 1].first_tile - R.first_tile - tile;
  t.n_tiles          = left < per ? left : per;
  t.row0             = R.first_row + tile * kTailTile;
  t.row_end          = runs[r + 1].first_row;
  t.base             = R.id_off + (long long)tile * kTailTile * R.degree;
  return t;
}

// the ids of a unit: entry j of this lane at base + 32 j (j < n_tiles * d <= kTailUnitEntries)
__device__ __forceinline__ void tail_load(int (&q)[kTailUnitEntries], tail_unit_t const& u, int32_t const* __restrict__ ids,
                                          unsigned long long pol, int lane)
{
  const int n         = u.n_tiles * u.d;  // the first kTailUnitEntries of them
  int32_t const* base = ids + u.base + lane;
#pragma unroll
  for (int j = 0; j < kTailUnitEntries; ++j)
    if (j < n) q[j] = ld_stream_i32(base + j * kTailTile, pol);
}

// the unit's rows, in-degree D: a row's entries in batches of 8, gathered, then summed as an fp64 tree (the order of
// k_spmv_low), the batches added in order; EPI: with the row epilogue (a.epi)
template <typename T, bool WEIGHTED, int D, bool EPI>
__device__ __forceinline__ void tail_rows(int const (&q)[kTailUnitEntries], tail_unit_t const& u, tail_args_t<T> const& a,
                                          T const* __restrict__ sx, double init, unsigned long long pol, unsigned long long keep,
                                          int lane, epi_sums_t& sums)
{
  constexpr int U = tail_unit_tiles(D);
  T const* wp       = WEIGHTED ? a.w + u.base + lane : nullptr;  // entry j: wp[32 j]
#pragma unroll
  for (int t = 0; t < U; ++t) {
    if (t < u.n_tiles) {
      const int row = u.row0 + t * kTailTile + lane;
      const int v   = row < u.row_end ? (a.row_vertex ? a.row_vertex[row] : row) : -1;
      // the epilogue's loads are issued with the gathers: after the sum they would be one more round trip per tile
      const epi_in_t<T> p = EPI && v >= 0 ? epi_load(a.epi, v) : epi_in_t<T>{(T)0, (T)0};
      double s = 0.0;
#pragma unroll
      for (int k0 = 0; k0 < D; k0 += kTailBatch) {
        double b[kTailBatch];
#pragma unroll
        for (int i = 0; i < kTailBatch; ++i) {
          b[i] = 0.0;
          if (k0 + i < D) {
            const int j = t * D + k0 + i;  // a tile holds more entries than a unit's registers only at D > kTailUnitEntries
            const int c = j < kTailUnitEntries ? q[j] : ld_stream_i32(a.ids + u.base + j * kTailTile + lane, pol);
            T v         = c < a.W ? sx[c] : ld_keep(a.x + c, keep);
            if (WEIGHTED) v *= ld_stream(wp + j * kTailTile);
            b[i] = (double)v;
          }
        }
        s += ((b[0] + b[1]) + (b[2] + b[3])) + ((b[4] + b[5]) + (b[6] + b[7]));
      }
      if (v >= 0) {
        if constexpr (EPI) store_row(a.y, a.epi, v, (T)(s * a.alpha + init), p, sums);
        else a.y[v] = (T)(s * a.alpha + init);
      }
    }
  }
}

template <typename T, bool WEIGHTED, bool EPI, int D = 1>
__device__ __forceinline__ void tail_process(int const (&q)[kTailUnitEntries], tail_unit_t const& u, tail_args_t<T> const& a,
                                             T const* __restrict__ sx, double init, unsigned long long pol,
                                             unsigned long long keep, int lane, epi_sums_t& sums)
{
  if (u.d == D) tail_rows<T, WEIGHTED, D, EPI>(q, u, a, sx, init, pol, keep, lane, sums);
  else if constexpr (D < kTailMaxDegree) tail_process<T, WEIGHTED, EPI, D + 1>(q, u, a, sx, init, pol, keep, lane, sums);
}

// EPI: with the row epilogue (a.epi.x_next set).  A template argument, not a run-time test: the kernel runs at the register
// limit, and sweeps without an epilogue (Katz, HITS, ...) keep the code they had.
template <typename T, bool WEIGHTED, bool EPI>
__global__ void __launch_bounds__(kTailThreads, 1) k_sweep_tail(tail_args_t<T> a)
{
  B200_DYN_SMEM(smem_raw);
  T const* sx = reinterpret_cast<T const*>(smem_raw);
  __shared__ uint64_t bar;
  __shared__ tail_run_t s_run[kTailMaxDegree + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.spent = 0;  // also once the loop is done: a later sweep may start a new one
  if (a.st->done) return;
  const unsigned long long pol = make_l2_policy_evict_first(), keep = make_l2_policy_evict_last();
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    load_slice(smem_raw, a.x, 0, a.W, &bar);
  }
  if ((int)threadIdx.x <= a.n_runs) s_run[threadIdx.x] = a.runs[threadIdx.x];
  const double init = a.st->init;
  // the lane's epilogue sums over all its units and empty rows, flushed once per warp at the end.  In registers: 8 KiB of
  // them in shared memory took the kernel past the 196 KiB shared-memory carve-out, and the L1 that serves its gathers shrank
  // from 60 to 28 KiB (the whole sweep 8 % slower, epilogue or not)
  epi_sums_t sums;
  __syncthreads();  // the barrier is initialised before anybody waits on it, the run table is in place
  // unit i is processed while the ids of unit i+1 and the draw of unit i+2 are in flight
  const int ra = draw_issue(a.cursor, 1, lane, true), rb = draw_issue(a.cursor, 1, lane, true);
  tail_unit_t A = tail_unit(s_run, a.n_runs, draw_get(ra));
  int qa[kTailUnitEntries], qb[kTailUnitEntries];
  tail_load(qa, A, a.ids, pol, lane);
  tail_unit_t B = tail_unit(s_run, a.n_runs, draw_get(rb));
  mbar_wait(&bar, 0);
  while (A.d > 0) {
    tail_load(qb, B, a.ids, pol, lane);
    const int rc = draw_issue(a.cursor, 1, lane, B.d > 0);
    tail_process<T, WEIGHTED, EPI>(qa, A, a, sx, init, pol, keep, lane, sums);
    if (B.d == 0) break;
    const tail_unit_t C = tail_unit(s_run, a.n_runs, draw_get(rc));
    tail_load(qa, C, a.ids, pol, lane);
    const int rd = draw_issue(a.cursor, 1, lane, C.d > 0);
    tail_process<T, WEIGHTED, EPI>(qb, B, a, sx, init, pol, keep, lane, sums);
    A = C;
    B = tail_unit(s_run, a.n_runs, draw_get(rd));
  }
  // the empty rows: y = init, and with an epilogue x_next = init / out_w (about half of RMAT's vertices).  Without
  // row_vertex in 16-byte vectors, kEmptyBatch of them in flight per thread (a row at a time measured ~1 % slower)
  const int stride = gridDim.x * blockDim.x;
  const int tid    = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  const int lo     = a.runs[a.n_runs].first_row;
  if constexpr (!EPI) {
    for (int r = lo + tid; r < a.empty_hi; r += stride) a.y[a.row_vertex ? a.row_vertex[r] : r] = (T)init;
  } else if (a.row_vertex) {
    for (int r = lo + tid; r < a.empty_hi; r += stride) store_row(a.y, a.epi, a.row_vertex[r], (T)init, sums);
  } else {
    constexpr int kV = 16 / sizeof(T), kEmptyBatch = 4;
    const int v_lo = (lo + kV - 1) / kV, v_hi = a.empty_hi / kV;  // whole vectors [v_lo, v_hi)
    const int s_hi = v_lo < v_hi ? v_lo * kV : a.empty_hi;         // rows before them; the rest from v_hi * kV on
    for (int r = lo + tid; r < s_hi; r += stride) store_row(a.y, a.epi, r, (T)init, sums);
    for (int r = (v_lo < v_hi ? v_hi * kV : a.empty_hi) + tid; r < a.empty_hi; r += stride) store_row(a.y, a.epi, r, (T)init, sums);
    const T fill = (T)init;
    for (int i0 = v_lo + tid; i0 < v_hi; i0 += kEmptyBatch * stride) {
      uint4 ow[kEmptyBatch], old[kEmptyBatch];
#pragma unroll
      for (int j = 0; j < kEmptyBatch; ++j) {
        const int i = i0 + j * stride;
        if (i < v_hi) {
          ow[j] = reinterpret_cast<uint4 const*>(a.epi.out_w)[i];
          if (a.epi.y_old) old[j] = reinterpret_cast<uint4 const*>(a.epi.y_old)[i];
        }
      }
#pragma unroll
      for (int j = 0; j < kEmptyBatch; ++j) {
        const int i = i0 + j * stride;
        if (i < v_hi) {
          T w[kV], o[kV], yv[kV], xv[kV];
          std::memcpy(w, &ow[j], 16);
          if (a.epi.y_old) std::memcpy(o, &old[j], 16);
#pragma unroll
          for (int k = 0; k < kV; ++k) {
            yv[k] = fill;
            xv[k] = w[k] == (T)0 ? fill : fill / w[k];
            if (w[k] == (T)0) sums.dangling += (double)fill;
            if (a.epi.y_old) sums.diff += fabs((double)fill - (double)o[k]);
          }
          uint4 qy, qx;
          std::memcpy(&qy, yv, 16);
          std::memcpy(&qx, xv, 16);
          if (a.y) reinterpret_cast<uint4*>(a.y)[i] = qy;
          reinterpret_cast<uint4*>(a.epi.x_next)[i] = qx;
        }
      }
    }
  }
  if constexpr (EPI) epi_flush(a.epi, sums);
}

// x must hold padded_x_elems() elements, zero behind n_vertices (slices are copied whole).
// With a tail and L.tail_sms > 0 the tail runs on the handle's side stream, forked from h.stream before the bands and
// joined back into it after them: k_sweep_tail on tail_sms SMs beside the bands' k_sweep on the other L.n_cta.  They share
// nothing but x (read by both), the fp64 sums of the row epilogue in *st (atomics) and the tail's cursor, which the tail
// launches alternate (sweep_layout_t::cursor).  Whatever the caller enqueues on h.stream afterwards runs after both.
template <typename T>
void launch_sweep(handle_impl const& h, csx_t const& c, sweep_layout_t const& L, T const* x, T* y, double* acc, double alpha,
                  pr_state_t const* st, bool use_weights, bool covered_rows_only, row_epi_t<T> const& epi)
{
  const bool weighted = use_weights && L.w.data() != nullptr;
  auto* const sweep_kernel = weighted ? k_sweep<T, true> : k_sweep<T, false>;
  auto* const tail_kernel  = epi.x_next ? (weighted ? k_sweep_tail<T, true, true> : k_sweep_tail<T, false, true>)
                                        : (weighted ? k_sweep_tail<T, true, false> : k_sweep_tail<T, false, false>);
  // the attribute is per device and cheap to set: no process-wide "done" flag (a second device would miss it)
  CUDA_TRY(cudaFuncSetAttribute(sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSweepDynSmem));
  // covered_rows_only: y of the rows without edges already holds their (unvarying) value — multi-GPU blocks, where more than
  // half of the row slots are empty and the unvarying term is 0 (mg.cu)
  const int32_t finish_rows = covered_rows_only ? L.n_cov : c.n_rows;
  const bool tail           = L.n_str < L.n_cov;  // rows of small in-degree left the stream (sweep_layout.cuh)
  const bool split          = tail && L.tail_sms > 0;
  // the rows [n_str, n_cov) and (unless covered_rows_only) the empty rows, by k_sweep_tail
  auto launch_tail = [&](cudaStream_t s, int sms) {
    tail_args_t<T> t;
    const unsigned slot = L.tail_sweeps++ & 1u;
    t.runs       = L.tail_run.as<tail_run_t>();
    t.ids        = L.tail_ids.as<int32_t>();
    t.w          = weighted ? L.tail_w.as<T>() : nullptr;
    t.x          = x;
    t.y          = y;
    t.row_vertex = c.row_vertex.as<int32_t>();
    t.cursor     = L.cursor.as<int>() + L.n_phases + slot;
    t.spent      = L.cursor.as<int>() + L.n_phases + (slot ^ 1u);
    t.st         = st;
    t.n_runs     = L.n_tail_runs;
    t.empty_hi   = finish_rows;
    t.W          = L.W;
    t.alpha      = alpha;
    t.epi        = epi;
    const int units  = L.tail_runs.back().first_unit;
    const int blocks = std::max(1, std::min(sms, (units + kTailThreads / 32 - 1) / (kTailThreads / 32)));
    CUDA_TRY(cudaFuncSetAttribute(tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSweepDynSmem));
    B200_LAUNCH_ON(h, s, tail_kernel, blocks, kTailThreads, kSweepDynSmem, t);
  };
  if (split) {
    CUDA_TRY(cudaEventRecord(h.fork, h.stream));
    CUDA_TRY(cudaStreamWaitEvent(h.side, h.fork, 0));
    launch_tail(h.side, L.tail_sms);
  }
  sweep_args_t<T> a;
  a.p.ids     = L.ids.as<uint4>();
  a.p.rows    = L.rows.as<int32_t>();
  a.p.w       = L.w.data();
  a.p.acc     = acc;
  a.chunks    = L.chunks.as<sweep_chunk_t>();
  a.phases    = L.phases.as<sweep_phase_t>();
  a.cursor    = L.cursor.as<int>();
  a.x         = x;
  a.st        = st;
  a.W         = L.W;
  a.p.pol     = 0;
  a.p.acc_pol = 0;
  // 8 steps of 64 rows per warp: faster than 4 or 2 steps
  constexpr int kFinishSteps = 8;
  // band by band: the band's rows are finished while its accumulators are in the L2, before the next band's REDs evict them.
  // y (and the epilogue's x_next) must not overlap x: a band's finish writes y while later bands (and the tail) still read x.
  for (int band = 0; band < L.n_bands; ++band) {
    // the last band also writes the empty rows, unless the tail launch does
    const int row_hi = band < L.n_bands - 1 ? L.band_row[band + 1] : (tail ? L.n_str : finish_rows);
    const int row_lo = L.band_row[band];
    a.cta_phase      = L.cta_phase.as<int32_t>() + (size_t)band * L.n_cta;
    a.ph_lo          = L.band_phase[band];
    a.ph_hi          = L.band_phase[band + 1];
    B200_LAUNCH(h, sweep_kernel, L.n_cta, kSweepThreads, kSweepDynSmem, a);
    const int n_ph = a.ph_hi - a.ph_lo;  // the cursors to reset: the band's phases'
    const int n    = std::max((row_hi - row_lo + 2 * kFinishSteps - 1) / (2 * kFinishSteps), n_ph);  // threads: 16 rows each
    B200_LAUNCH(h, (k_sweep_finish<T, kFinishSteps>), (std::max(n, 1) + 255) / 256, 256, 0, acc, row_lo, L.n_str, row_hi, y,
                c.row_vertex.as<int32_t>(), alpha, L.cursor.as<int>() + a.ph_lo, n_ph, st, epi);
  }
  if (split) {
    CUDA_TRY(cudaEventRecord(h.join, h.side));
    CUDA_TRY(cudaStreamWaitEvent(h.stream, h.join, 0));
  } else if (tail) {
    launch_tail(h.stream, h.sm_count);
  }
}

}  // namespace b200
