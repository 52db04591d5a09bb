// Builder of the pull sweep's layout (sweep_layout.cuh), staged on the GPU on first use and cached in the csx, and the
// host-side planner of the sweep's chunks, phases and CTA ranges with its debug entries in the C ABI.
#include "sweep_layout.cuh"
#include "staging.cuh"

#include <thrust/iterator/counting_iterator.h>

namespace b200 {

namespace {

// ---- staging of the piece stream.  All passes are O(nnz + #segments):
//   1. head flags: an edge starts a (row, block) segment if it starts its row or its source lies in another
//      block than its predecessor's (neighbours are sorted by source id)
//   2. segments = compacted head positions; each is cut into pieces of <= 64 entries, a piece gets its kind
//      (S / Q / H = 1 / 2 / <= 4 entries, F1..F8 = that many lane slots of 8 entries)
//   3. pieces are ordered (stable radix sort) by (band, block, kind); a run of one (band, block, kind) is cut into groups
//      of 256 / 128 / 64 / 32 pieces and chunks of a few groups; band by band, chunks are dealt to the persistent CTAs as
//      contiguous, cost-balanced ranges, the part of one block inside a range is a phase
//   4. one warp per group writes its step-rows (32 lanes x 16 bytes of ids) and row slots

__global__ void k_hot_row_starts(int32_t const* __restrict__ off, int32_t n_cov, uint8_t* __restrict__ flag)
{
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_cov; r += (int64_t)gridDim.x * blockDim.x) flag[(size_t)off[r]] = 1;  // covered rows are never empty
}

__global__ void k_hot_heads(int32_t const* __restrict__ idx, long long nnz, int W, uint8_t* __restrict__ flag)
{
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nnz; e += (long long)gridDim.x * blockDim.x) {
    if (e > 0 && !flag[e] && idx[e] / W != idx[e - 1] / W) flag[e] = 1;
  }
}

constexpr int kHotPieceSlots   = 8;                          // slots per piece (= steps per group) at most
constexpr int kHotPieceEntries = kHotPieceSlots * kHotSlot;  // 64

// per segment: its row (binary search in the offsets) and how many pieces it yields
__global__ void k_hot_segment_info(int32_t const* __restrict__ head_pos, int32_t n_segs, long long nnz,
                                   int32_t const* __restrict__ off, int32_t n_cov, int32_t* __restrict__ seg_row,
                                   int32_t* __restrict__ seg_pieces)
{
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k <= n_segs; k += (int64_t)gridDim.x * blockDim.x) {
    if (k == n_segs) {
      seg_pieces[k] = 0;
      continue;
    }
    const long long start = head_pos[k];
    const long long end   = (k + 1 < n_segs) ? (long long)head_pos[k + 1] : nnz;
    int lo = 0, hi = n_cov;  // last row r with off[r] <= start
    while (hi - lo > 1) {
      const int mid = lo + ((hi - lo) >> 1);
      if ((long long)off[mid] <= start) lo = mid; else hi = mid;
    }
    seg_row[k]    = lo;
    seg_pieces[k] = (int)((end - start + kHotPieceEntries - 1) / kHotPieceEntries);
  }
}

__host__ __device__ __forceinline__ int piece_kind(int len)
{
  return len == 1 ? kKindS : (len == 2 ? kKindQ : (len <= 4 ? kKindH : kKindF1 + (len + kHotSlot - 1) / kHotSlot - 1));
}

// per segment: write its pieces (start edge, entries, row) and their key = (band * B + block) * kNumKinds + kind
__global__ void k_hot_emit_pieces(int32_t const* __restrict__ head_pos, int32_t n_segs, long long nnz,
                                  int32_t const* __restrict__ idx, int W, int B, int32_t band_rows,
                                  int32_t const* __restrict__ seg_row,
                                  int32_t const* __restrict__ piece_off, uint32_t* __restrict__ piece_key,
                                  int32_t* __restrict__ piece_start, int32_t* __restrict__ piece_len,
                                  int32_t* __restrict__ piece_row)
{
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n_segs; k += (int64_t)gridDim.x * blockDim.x) {
    const long long start = head_pos[k];
    const long long end   = (k + 1 < n_segs) ? (long long)head_pos[k + 1] : nnz;
    const int row         = seg_row[k];
    const int bb          = (row / band_rows) * B + idx[start] / W;  // (band, block)
    int p                 = piece_off[k];
    for (long long s = start; s < end; s += kHotPieceEntries, ++p) {
      const int len  = (int)((end - s < kHotPieceEntries) ? end - s : kHotPieceEntries);
      piece_key[p]   = (uint32_t)(bb * kNumKinds + piece_kind(len));
      piece_start[p] = (int32_t)s;
      piece_len[p]   = len;
      piece_row[p]   = row;
    }
  }
}

__global__ void k_hot_class_starts(uint32_t const* __restrict__ sorted_key, int32_t n_pieces, int n_keys,
                                   int32_t* __restrict__ class_start)
{
  for (int64_t key = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; key <= n_keys; key += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_pieces;  // first piece with sorted_key >= key
    while (lo < hi) {
      const int mid = lo + ((hi - lo) >> 1);
      if (sorted_key[mid] < (uint32_t)key) lo = mid + 1; else hi = mid;
    }
    class_start[key] = lo;
  }
}

struct sweep_fill_t {  // build-time companion of a chunk: its pieces start at piece_begin, its (band, block, kind) run ends at piece_end
  int32_t piece_begin, piece_end, block, pad;
};

// Host-side plan of the sweep's work structure, from the piece counts per (band, block, kind) alone (class_start[key] =
// first piece of key = (band * B + block) * kNumKinds + kind, pieces ordered by key):
//   group = 256 / 128 / 64 / 32 pieces of one kind (S / Q / H / F), 1 or (F kinds) 1..8 step-rows
//   chunk = consecutive groups of one kind in one block of one band, at most kind_chunk_groups(kind)
//   range = contiguous chunks of one band per persistent CTA, balanced by an estimate of their load/store-unit time (the
//           sweep is bound by it: one cycle per 128-byte line of ids, per conflict-free 32 gathers, per sector of atomics);
//           every band is dealt to the same n_cta CTAs on its own (one sweep launch per band)
//   phase = the chunks of one block inside one range (a CTA loads the block's slice once per phase)
// Pure host code: exercised on CPU through cugraph_b200_debug_plan_sweep[_bands] (tests/test_sweep_plan*_cpu.py).
struct sweep_plan_t {
  std::vector<sweep_chunk_t> chunks;
  std::vector<sweep_fill_t> fills;
  std::vector<sweep_phase_t> phases;
  std::vector<int32_t> cta_phase;   // n_bands * n_cta + 1
  std::vector<int32_t> band_phase;  // n_bands + 1
  int64_t n_steprows{0}, n_rowslots{0};
  int n_cta{1};
};

inline double sweep_group_cost(int kind)
{
  // Load/store-unit cycles.  The atomics dominate: a scattered 64-bit RED costs about one cycle PER LANE whatever its
  // sectors (measured: plain stores or one sector per warp instead of scattered atomics made no difference), i.e.
  // ~1.2 cycles per piece; a step-row costs 4 lines of ids + 8 gathers at ~1.5 wavefronts.  The F8 pieces of hub rows are
  // summed by shuffles first (one RED per 32 pieces).
  return kind_steps(kind) * 14.0 + kind_pieces(kind) * (kind == kNumKinds - 1 ? 0.1 : 1.2) + 4.0;
}
constexpr double kPhaseCost = 2500.0;  // barrier + 192 KiB slice fill, in the same unit

bool plan_sweep(std::vector<int32_t> const& cstart, int n_bands, int B, int sm_count, sweep_plan_t& P)
{
  std::vector<double> cost;          // per chunk, the phase overhead on the first chunk of every block
  std::vector<size_t> band_chunk(1);  // chunks of band k: [band_chunk[k], band_chunk[k+1])
  for (int band = 0; band < n_bands; ++band) {
    for (int b = 0; b < B; ++b) {
      bool first = true;
      for (int kind = 0; kind < kNumKinds; ++kind) {
        const int key    = (band * B + b) * kNumKinds + kind;
        int32_t p        = cstart[key];
        const int32_t pe = cstart[key + 1];
        const int ppg = kind_pieces(kind), steps = kind_steps(kind), gmax = kind_chunk_groups(kind);
        while (p < pe) {
          const int groups = (int)std::min<int64_t>(gmax, ((int64_t)(pe - p) + ppg - 1) / ppg);
          if (P.n_steprows + (int64_t)groups * steps >= (1ll << 31) - 64 || P.n_rowslots + (int64_t)groups * ppg >= (1ll << 31) - 64)
            return false;  // 32-bit step-row / row-slot numbers
          P.chunks.push_back({(int32_t)P.n_steprows, (int32_t)P.n_rowslots, groups, kind});
          P.fills.push_back({p, pe, b, 0});
          cost.push_back(groups * sweep_group_cost(kind) + (first ? kPhaseCost : 0.0));
          first = false;
          P.n_steprows += (int64_t)groups * steps;
          P.n_rowslots += (int64_t)groups * ppg;
          p += groups * ppg;  // may pass pe inside the last group: the fill pads
        }
      }
    }
    band_chunk.push_back(P.chunks.size());
  }
  size_t most = 0;
  for (int band = 0; band < n_bands; ++band) most = std::max(most, band_chunk[band + 1] - band_chunk[band]);
  P.n_cta = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm_count, most));
  P.cta_phase.assign((size_t)n_bands * P.n_cta + 1, 0);
  P.band_phase.assign(n_bands + 1, 0);
  for (int band = 0; band < n_bands; ++band) {
    const size_t c_lo = band_chunk[band], n = band_chunk[band + 1] - c_lo;
    std::vector<double> pre(n + 1, 0.0);
    for (size_t c = 0; c < n; ++c) pre[c + 1] = pre[c] + cost[c_lo + c];
    P.band_phase[band] = (int32_t)P.phases.size();
    size_t c = 0;
    for (int cta = 0; cta < P.n_cta; ++cta) {
      const double target = pre[n] * (cta + 1) / P.n_cta;
      const size_t c0     = c;
      if (cta == P.n_cta - 1) c = n;
      else while (c < n && pre[c + 1] <= target) ++c;
      P.cta_phase[(size_t)band * P.n_cta + cta] = (int32_t)P.phases.size();
      for (size_t k = c_lo + c0; k < c_lo + c;) {  // split the range by block
        size_t e = k;
        while (e < c_lo + c && P.fills[e].block == P.fills[k].block) ++e;
        P.phases.push_back({P.fills[k].block, (int32_t)k, (int32_t)e, 0});
        k = e;
      }
    }
  }
  P.band_phase[n_bands]                  = (int32_t)P.phases.size();
  P.cta_phase[(size_t)n_bands * P.n_cta] = (int32_t)P.phases.size();
  return true;
}

// Bank-aware entry order inside the lane slots of the F kinds (4-byte values): order the entries of the 32 pieces of a group
// so that the k-th shared-memory gathers of the 32 lanes in every step (one LDS of the sweep kernel) fall into different
// banks.  Any assignment of a piece's entries to its (step, position) places is a valid layout (the sweep adds all of them
// into one sum per piece); padding may point at any of the kHotZeroPad zero columns, i.e. at any bank.  Greedy, place by
// place (bank_order_place below); a lane without a free bank waits for a later place while it has spare places left; all
// padding of a place shares one zero column on a free bank.  Sweep on RMAT-24: 0.373 ms without, 0.331 ms with this order.
// State per lane: bank_bits[b] = the piece's entries (bit e = entry e, <= 64 per piece) on bank b, `rem` = not placed yet,
// `have` = banks with an entry left.
struct bank_piece_t {
  unsigned long long bank_bits[32];
  unsigned long long rem;
  unsigned have;
  unsigned have2;  // banks with at least two entries left: used first, which keeps the number of distinct banks up
};

// one place of all 32 lanes: returns this lane's entry index (>= 0) or -1 - pad_bank for padding.
// PARALLEL greedy: every lane that still holds entries proposes a bank nobody has taken at this place (preferring banks of
// which its piece still holds several entries, search start rotated by lane and place); of the lanes proposing the same
// bank the one that comes first in an order rotating with the place wins, the others propose again — three rounds, then
// lanes that must place an entry now (no spare places left) take any bank.  (A version in which the 32 lanes took turns
// one after the other reached 1.5 wavefronts per load on RMAT-20 but cost 42 ms of staging at RMAT-24.)
constexpr int kBankRounds = 8;
__device__ __forceinline__ int bank_order_place(bank_piece_t& P, int places_left, int lane)
{
  unsigned taken = 0, taken2 = 0;  // banks used once / twice at this place (the same in every lane)
  int mine       = -1;
  const int spare = places_left - __popcll(P.rem);  // places beyond the ones the remaining entries need
  const int prio  = (lane + 11 * places_left) & 31;  // who wins a contested bank changes from place to place
  const int r0    = (lane + 5 * places_left) & 31;
#pragma unroll 1
  for (int round = 0; round < kBankRounds; ++round) {
    int want = -1;
    if (mine < 0 && P.rem != 0ull) {
      unsigned pick = P.have2 & ~taken;
      if (!pick) pick = P.have & ~taken;
      if (!pick && round >= kBankRounds - 2 && spare <= 0) {  // must place now: accept a conflict, on a bank used once if any
        pick = P.have & ~taken2;
        if (!pick && round == kBankRounds - 1) pick = P.have;
      }
      if (pick) {
        const unsigned rot = r0 ? ((pick >> r0) | (pick << (32 - r0))) : pick;
        want               = (__ffs(rot) - 1 + r0) & 31;
      }
    }
    // lanes with the same proposal: the smallest rotated priority wins (in the last round everybody proposing wins)
    const unsigned same = __match_any_sync(0xffffffffu, want);
    bool win            = want >= 0;
    if (win && round < kBankRounds - 1) {
      // winner = the lane of `same` whose prio is smallest: compare by scanning the (few) competitors
      unsigned others = same & ~(1u << lane);
      while (others) {
        const int o = __ffs(others) - 1;
        others &= others - 1;
        const int po = (o + 11 * places_left) & 31;
        if (po < prio) win = false;
      }
    }
    if (win) {
      mine = __ffsll((long long)(P.bank_bits[want] & P.rem)) - 1;
      P.rem &= ~(1ull << mine);
      const int left = __popcll(P.bank_bits[want] & P.rem);
      if (left < 2) P.have2 &= ~(1u << want);
      if (left < 1) P.have &= ~(1u << want);
    }
    const unsigned won = __reduce_or_sync(0xffffffffu, win ? (1u << want) : 0u);
    taken2 |= taken & won;
    taken |= won;
    if (!__any_sync(0xffffffffu, mine < 0 && P.rem != 0ull)) break;
  }
  if (mine >= 0) return mine;
  const int pad_bank = (~taken) ? __ffs(~taken) - 1 : 0;
  return -1 - pad_bank;
}

constexpr int kFillWarps = 6;  // = the largest kind_chunk_groups()

// one CTA per chunk, one warp per group
template <typename T, bool BANK>
__global__ void __launch_bounds__(kFillWarps * 32)
k_sweep_fill(sweep_chunk_t const* __restrict__ chunks, sweep_fill_t const* __restrict__ fills, int32_t const* __restrict__ perm,
             int32_t const* __restrict__ piece_start, int32_t const* __restrict__ piece_len,
             int32_t const* __restrict__ piece_row, int32_t const* __restrict__ idx, T const* __restrict__ w, int W,
             uint4* __restrict__ ids_out, T* __restrict__ w_out, int32_t* __restrict__ rows_out)
{
  const sweep_chunk_t ch = chunks[blockIdx.x];
  const sweep_fill_t fl  = fills[blockIdx.x];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  if (g >= ch.n_groups) return;
  const int col0 = fl.block * W;
  if (ch.kind < kKindF1) {  // S / Q / H: R pieces of E entries per lane; piece k of lane l is piece k * 32 + l of the group
    const int R = ch.kind == kKindS ? 8 : (ch.kind == kKindQ ? 4 : 2), E = 8 / R;
    const size_t slot = ((size_t)(unsigned)(ch.sr_begin + g) << 5) + lane;
    unsigned v[8];
    for (int k = 0; k < R; ++k) {
      const long long pi = (long long)fl.piece_begin + ((long long)g * 32 * R) + k * 32 + lane;
      int st = 0, ln = 0, row = -1;
      if (pi < fl.piece_end) {
        const int p = perm[pi];
        st          = piece_start[p];
        ln          = piece_len[p];
        row         = piece_row[p];
      }
      for (int e = 0; e < E; ++e) {
        v[k * E + e] = e < ln ? (unsigned)(idx[st + e] - col0) : (unsigned)W;
        if (w_out) w_out[slot * 8 + k * E + e] = e < ln ? w[st + e] : (T)0;
      }
      rows_out[(size_t)(unsigned)ch.row_begin + ((size_t)g * 32 + lane) * R + k] = row;
    }
    ids_out[slot] = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
    return;
  }
  const int C        = ch.kind - kKindF1 + 1;
  const long long pi = (long long)fl.piece_begin + (long long)g * 32 + lane;
  int st = 0, ln = 0, row = -1;
  if (pi < fl.piece_end) {
    const int p = perm[pi];
    st          = piece_start[p];
    ln          = piece_len[p];
    row         = piece_row[p];
  }
  rows_out[(size_t)(unsigned)ch.row_begin + (size_t)g * 32 + lane] = row;
  bank_piece_t bp;  // only used by the BANK instantiation
  if (BANK) {       // the whole warp takes part (lanes without a piece hold padding only)
    for (int b = 0; b < 32; ++b) bp.bank_bits[b] = 0ull;
    bp.have = bp.have2 = 0u;
    for (int e = 0; e < ln; ++e) {
      const int b = (idx[st + e] - col0) & 31;
      if (bp.bank_bits[b]) bp.have2 |= 1u << b;
      bp.bank_bits[b] |= 1ull << e;
      bp.have |= 1u << b;
    }
    bp.rem = ln >= 64 ? ~0ull : ((1ull << ln) - 1ull);
  }
  for (int j = 0; j < C; ++j) {
    const size_t slot = ((size_t)(unsigned)(ch.sr_begin + g * C + j) << 5) + lane;
    unsigned v[kHotSlot];
    if (BANK) {
#pragma unroll 1
      for (int k = 0; k < kHotSlot; ++k) {
        const int e = bank_order_place(bp, (C - j) * kHotSlot - k, lane);
        v[k]        = e >= 0 ? (unsigned)(idx[st + e] - col0) : (unsigned)(W + ((-1 - e - (W & 31)) & 31));
        if (w_out) w_out[slot * kHotSlot + k] = e >= 0 ? w[st + e] : (T)0;
      }
    } else {
#pragma unroll
      for (int k = 0; k < kHotSlot; ++k) {
        const int e   = j * kHotSlot + k;
        const bool in = e < ln;
        v[k]          = in ? (unsigned)(idx[st + e] - col0) : (unsigned)W;
        if (w_out) w_out[slot * kHotSlot + k] = in ? w[st + e] : (T)0;
      }
    }
    ids_out[slot] = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
  }
}

// ---- the tail layout (sweep_layout.cuh): runs of equal in-degree, tiles of 32 rows, lane-interleaved ids
// below[d] = first row of [row_lo, row_hi) whose in-degree is < d (rows are degree-descending), d = 0 .. kTailMaxDegree + 1
__global__ void k_tail_run_bounds(int32_t const* __restrict__ off, int32_t row_lo, int32_t row_hi, int32_t* __restrict__ below)
{
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d > kTailMaxDegree + 1) return;
  int lo = row_lo, hi = row_hi;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if ((long long)(off[mid + 1] - off[mid]) >= d) lo = mid + 1; else hi = mid;
  }
  below[d] = lo;
}

// one thread per lane of a tile, striding over the grid
template <typename T>
__global__ void k_tail_fill(tail_run_t const* __restrict__ runs, int n_runs, int32_t const* __restrict__ off,
                            int32_t const* __restrict__ idx, T const* __restrict__ w, int32_t pad_col,
                            int32_t* __restrict__ ids_out, T* __restrict__ w_out)
{
  const long long n_lanes = (long long)runs[n_runs].first_tile * kTailTile;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n_lanes; t += (int64_t)gridDim.x * blockDim.x) {
    const int tile = (int)(t / kTailTile), lane = (int)(t % kTailTile);
    int r = 0;
    while (tile >= runs[r + 1].first_tile) ++r;
    const tail_run_t R = runs[r];
    const int d        = R.degree;
    const int row      = R.first_row + (tile - R.first_tile) * kTailTile + lane;
    const bool live    = row < runs[r + 1].first_row;
    const long long e0 = live ? (long long)off[row] : 0;
    const long long o  = R.id_off + (long long)(tile - R.first_tile) * kTailTile * d + lane;
    for (int k = 0; k < d; ++k) {
      ids_out[o + (long long)k * kTailTile] = live ? idx[e0 + k] : pad_col;
      if (w_out) w_out[o + (long long)k * kTailTile] = live ? w[e0 + k] : (T)0;
    }
  }
}

void build_tail_layout(handle_impl const& h, csx_t const& c, int32_t nv, size_t es, sweep_layout_t& L)
{
  dbuf d_below = make_dbuf<int32_t>(kTailMaxDegree + 2, h.stream);
  B200_LAUNCH(h, k_tail_run_bounds, 1, 64, 0, c.offsets.as<int32_t>(), L.n_str, L.n_cov, d_below.as<int32_t>());
  int32_t below[kTailMaxDegree + 2];
  CUDA_TRY(cudaMemcpyAsync(below, d_below.data(), sizeof(below), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  tail_run_t at{0, L.n_str, 0, 0, 0};  // the next run starts here
  for (int d = kTailMaxDegree; d >= 1; --d) {
    const int32_t lo = below[d + 1], hi = below[d];  // the rows of in-degree d
    if (hi <= lo) continue;
    B200_EXPECTS(lo == at.first_row, CUGRAPH_UNKNOWN_ERROR, "tail rows are not degree-descending");
    at.degree = d;
    L.tail_runs.push_back(at);
    const int32_t tiles = (hi - lo + kTailTile - 1) / kTailTile;
    at.first_row = hi;
    at.first_tile += tiles;
    at.first_unit += (tiles + tail_unit_tiles(d) - 1) / tail_unit_tiles(d);
    at.id_off += (int64_t)tiles * kTailTile * d;
  }
  B200_EXPECTS(at.first_row == L.n_cov, CUGRAPH_UNKNOWN_ERROR, "tail rows of in-degree >= the bound or 0");
  at.degree     = 0;
  L.n_tail_runs = (int)L.tail_runs.size();
  L.tail_runs.push_back(at);
  L.tail_run = make_dbuf<tail_run_t>(L.tail_runs.size(), h.stream);
  CUDA_TRY(cudaMemcpyAsync(L.tail_run.data(), L.tail_runs.data(), sizeof(tail_run_t) * L.tail_runs.size(), cudaMemcpyHostToDevice,
                           h.stream));
  L.tail_ids = make_dbuf<int32_t>((size_t)std::max<int64_t>(at.id_off, 1), h.stream);
  const bool weighted = c.weights.data() != nullptr;
  if (weighted) L.tail_w = dbuf((size_t)std::max<int64_t>(at.id_off, 1) * es, h.stream);
  const int64_t threads = (int64_t)at.first_tile * kTailTile;
  if (es == 4)
    B200_LAUNCH(h, (k_tail_fill<float>), grid_for(threads), kBlock, 0, L.tail_run.as<tail_run_t>(), L.n_tail_runs,
                c.offsets.as<int32_t>(), c.indices.as<int32_t>(), c.weights.as<float>(), nv, L.tail_ids.as<int32_t>(), L.tail_w.as<float>());
  else
    B200_LAUNCH(h, (k_tail_fill<double>), grid_for(threads), kBlock, 0, L.tail_run.as<tail_run_t>(), L.n_tail_runs,
                c.offsets.as<int32_t>(), c.indices.as<int32_t>(), c.weights.as<double>(), nv, L.tail_ids.as<int32_t>(), L.tail_w.as<double>());
  check_last("sweep tail layout");
  sync(h);  // the host run table is pageable
}

// Row bands: the sweep's fp64 REDs into acc[row] hit the L2 only while the rows they scatter over fit in it (measured on an
// H100 80GB HBM3 at 700 W, 50 MB of L2: a scattered RED.64 costs the same up to 24 MB of accumulators, 1.3x at 48 MB and
// 3.7x at 64 MB), so the stream rows are split into bands whose accumulators take at most kBandL2Share of the L2.  Half
// gave the fastest RMAT-24 sweep without a tail (3 bands, DESIGN.md §3.2); more bands add launch tails and slice loads.
// CUGRAPH_B200_SWEEP_BANDS forces a count (tests, A/B runs).
constexpr double kBandL2Share = 0.5;

int sweep_bands(handle_impl const& h, int32_t n_str)
{
  const int most = std::max(1, (int)(((int64_t)n_str + kBandRowAlign - 1) / kBandRowAlign));
  int P          = h.tune.sweep_bands;
  if (P <= 0) P = h.l2_bytes ? (int)std::ceil(8.0 * n_str / (kBandL2Share * (double)h.l2_bytes)) : 1;
  return std::min(std::max(P, 1), most);
}

// The tail's share of the SMs.  k_sweep_tail runs on k SMs from the handle's side stream while the bands' k_sweep runs on the
// other sm_count - k (k_sweep is bound by the L2's sector rate more than by its SMs, the tail by the latency of its gathers:
// side by side the two take less than one after the other, DESIGN.md §3.2).  By default k splits the SMs in proportion to
// the two kernels' work: the stream's in the planner's cost unit (sweep_group_cost, summed over the chunks plan_sweep will
// cut), the tail's in entries (an empty row counts a quarter of an entry, a tail row one more), converted by
// kTailEntryCost.  CUGRAPH_B200_SWEEP_TAIL_SMS forces k (tests, A/B runs); 0 = no split: the tail after the bands on every SM.
// Measured on an H100 80GB HBM3 at 700 W, RMAT-24 PageRank (DESIGN.md §8.1): k_sweep takes 0.45-0.50 ms per sweep on 132,
// 116, 100 or 84 CTAs when it runs alone, so it is not bound by its SMs; side by side with the tail the iteration took 0.644
// / 0.730 / 0.647 / 0.611 / 0.658 ms at k = 0 / 40 / 48 / 56 / 64.  The ratio puts RMAT-24 at k = 56.
constexpr double kTailEntryCost = 1.4;  // sweep_group_cost units per tail entry
constexpr double kTailRowEntries = 1.0, kTailEmptyEntries = 0.25;

int sweep_tail_sms(handle_impl const& h, std::vector<int32_t> const& cstart, int n_bands, int B, int64_t tail_entries,
                   int64_t tail_rows, int64_t empty_rows, double* stream_cost, double* tail_cost)
{
  double stream = 0.0;
  for (int key = 0; key < n_bands * B * kNumKinds; ++key) {
    const int kind = key % kNumKinds, ppg = kind_pieces(kind);
    stream += (double)(((int64_t)cstart[key + 1] - cstart[key] + ppg - 1) / ppg) * sweep_group_cost(kind);
  }
  const double tail = kTailEntryCost * ((double)tail_entries + kTailRowEntries * (double)tail_rows + kTailEmptyEntries * (double)empty_rows);
  *stream_cost = stream;
  *tail_cost   = tail;
  if (tail_rows <= 0 || h.sm_count < 2) return 0;
  int k = h.tune.sweep_tail_sms;
  if (k < 0) k = (int)std::lround(h.sm_count * tail / std::max(stream + tail, 1.0));
  return std::min(std::max(k, 0), h.sm_count - 1);
}

// The piece stream holds the rows [0, seg[k]) for the bin k this returns: rows of in-degree >= kSegThreshold[k].
// By default the rows of in-degree < kSweepTailDegree leave it on graphs of at least kSweepTailMinEdges edges, and it holds
// every non-empty row on smaller ones.  CUGRAPH_B200_SWEEP_TAIL_DEGREE forces a bound on any graph (tests, A/B runs):
// 1 = no tail, other values are rounded down to a bin threshold.
int sweep_stream_bin(handle_impl const& h, csx_t const& c)
{
  int bound = h.tune.sweep_tail_degree;
  if (bound <= 0) bound = c.nnz >= kSweepTailMinEdges ? kSweepTailDegree : 1;
  int k = 0;
  while (kSegThreshold[k] > bound) ++k;  // kSegThreshold[kNumSeg - 2] = 1
  return k;
}

std::unique_ptr<sweep_layout_t> build_sweep_layout(handle_impl const& h, csx_t const& c, int32_t nv, size_t es)
{
  phase_trace tr(h);
  const int W         = (int)(kHotSliceBytes / es) - kHotZeroPad;  // columns per block; the pad holds zeros
  const int32_t n_cov = c.seg[kNumSeg - 2];                         // rows of degree >= 1
  const int32_t n_str = c.seg[sweep_stream_bin(h, c)];              // rows of the stream; the tail is swept by k_sweep_tail
  if (n_str <= 0) return nullptr;                                   // no row reaches the bound: the plain sweep fits better
  const int B         = (int)(((int64_t)nv + W - 1) / W);
  const int64_t nnz   = read_back(h, c.offsets.as<int32_t>() + n_str);  // edges of the stream rows: a prefix of indices (rows are degree-descending)
  auto L              = std::make_unique<sweep_layout_t>();
  L->W = W; L->B = B; L->n_cov = n_cov; L->n_str = n_str; L->nnz = c.nnz;
  int32_t const* idx = c.indices.as<int32_t>();
  // equal bands of whole kBandRowAlign spans; rounding may leave fewer than asked for
  const int asked         = sweep_bands(h, n_str);
  const int32_t band_rows = (int32_t)((((int64_t)n_str + asked - 1) / asked + kBandRowAlign - 1) / kBandRowAlign * kBandRowAlign);
  const int n_bands       = (int)(((int64_t)n_str + band_rows - 1) / band_rows);
  L->n_bands              = n_bands;
  for (int b = 0; b <= n_bands; ++b) L->band_row.push_back((int32_t)std::min<int64_t>((int64_t)b * band_rows, n_str));

  // 1. segment heads
  dbuf flag = make_dbuf<uint8_t>(nnz, h.stream);
  CUDA_TRY(cudaMemsetAsync(flag.data(), 0, nnz, h.stream));
  B200_LAUNCH(h, k_hot_row_starts, grid_for(n_str), kBlock, 0, c.offsets.as<int32_t>(), n_str, flag.as<uint8_t>());
  B200_LAUNCH(h, k_hot_heads, grid_for(nnz, 4, h.sm_count * 32), kBlock, 0, idx, (long long)nnz, W, flag.as<uint8_t>());
  dbuf head_pos = make_dbuf<int32_t>(nnz, h.stream);
  const int64_t n_segs64 = select_flagged<int32_t, thrust::counting_iterator<int32_t>>(
    h, thrust::counting_iterator<int32_t>(0), flag.as<uint8_t>(), head_pos.as<int32_t>(), nnz);
  flag.release();
  const int32_t n_segs = (int32_t)n_segs64;
  tr.mark("sweep layout: segment heads");

  // 2. pieces
  dbuf seg_row = make_dbuf<int32_t>(n_segs, h.stream), seg_pieces = make_dbuf<int32_t>((size_t)n_segs + 1, h.stream);
  dbuf piece_off = make_dbuf<int32_t>((size_t)n_segs + 1, h.stream);
  B200_LAUNCH(h, k_hot_segment_info, grid_for((int64_t)n_segs + 1), kBlock, 0, head_pos.as<int32_t>(), n_segs,
              (long long)nnz, c.offsets.as<int32_t>(), n_str, seg_row.as<int32_t>(), seg_pieces.as<int32_t>());
  exclusive_scan_i32(h, seg_pieces.as<int32_t>(), piece_off.as<int32_t>(), (int64_t)n_segs + 1);
  const int32_t n_pieces = read_back(h, piece_off.as<int32_t>() + n_segs);
  seg_pieces.release();
  L->n_pieces = n_pieces;
  dbuf piece_key = make_dbuf<uint32_t>(n_pieces, h.stream), piece_key2 = make_dbuf<uint32_t>(n_pieces, h.stream);
  dbuf piece_start = make_dbuf<int32_t>(n_pieces, h.stream), piece_len = make_dbuf<int32_t>(n_pieces, h.stream);
  dbuf piece_row = make_dbuf<int32_t>(n_pieces, h.stream);
  B200_LAUNCH(h, k_hot_emit_pieces, grid_for(n_segs), kBlock, 0, head_pos.as<int32_t>(), n_segs, (long long)nnz, idx, W, B,
              band_rows, seg_row.as<int32_t>(), piece_off.as<int32_t>(), piece_key.as<uint32_t>(), piece_start.as<int32_t>(),
              piece_len.as<int32_t>(), piece_row.as<int32_t>());
  head_pos.release();
  seg_row.release();
  piece_off.release();
  tr.mark("sweep layout: pieces");

  // 3. order pieces by (band, block, kind)
  const int n_keys = n_bands * B * kNumKinds;
  dbuf perm = make_dbuf<uint32_t>(n_pieces, h.stream), perm2 = make_dbuf<uint32_t>(n_pieces, h.stream);
  B200_LAUNCH(h, k_iota<uint32_t>, grid_for(n_pieces, 4), kBlock, 0, perm.as<uint32_t>(), (int64_t)n_pieces);
  sort_pairs<uint32_t, uint32_t>(h, piece_key.as<uint32_t>(), piece_key2.as<uint32_t>(), perm.as<uint32_t>(),
                                 perm2.as<uint32_t>(), n_pieces, 0, bits_for(n_keys + 1));
  dbuf class_start = make_dbuf<int32_t>((size_t)n_keys + 1, h.stream);
  B200_LAUNCH(h, k_hot_class_starts, grid_for(n_keys + 1), kBlock, 0, piece_key2.as<uint32_t>(), n_pieces, n_keys,
              class_start.as<int32_t>());
  std::vector<int32_t> cstart((size_t)n_keys + 1);
  CUDA_TRY(cudaMemcpyAsync(cstart.data(), class_start.data(), sizeof(int32_t) * cstart.size(), cudaMemcpyDeviceToHost, h.stream));
  sync(h);
  piece_key.release();
  piece_key2.release();
  perm.release();
  tr.mark("sweep layout: kind sort");
  if (tr.on) {  // layout statistics: pieces by kind, per range of blocks
    int edges[] = {0, 1, 4, 16, 64, 160, B};
    std::fprintf(stderr, "[sweep] B=%d W=%d rows=%d (tail %d rows, %lld edges) nnz=%lld segments=%d pieces=%d bands=%d of %d rows\n",
                 B, W, n_str, n_cov - n_str, (long long)(c.nnz - nnz), (long long)nnz, n_segs, n_pieces, n_bands, band_rows);
    for (int k = 0; k + 1 < 7; ++k) {
      const int b0 = std::min(edges[k], B), b1 = std::min(edges[k + 1], B);
      if (b1 <= b0) continue;
      std::fprintf(stderr, "[sweep] blocks [%d,%d) pieces by kind S Q H F1..F8:", b0, b1);
      for (int kind = 0; kind < kNumKinds; ++kind) {
        long long np = 0;
        for (int band = 0; band < n_bands; ++band)
          for (int b = b0; b < b1; ++b) np += cstart[(band * B + b) * kNumKinds + kind + 1] - cstart[(band * B + b) * kNumKinds + kind];
        std::fprintf(stderr, " %lld", np);
      }
      std::fprintf(stderr, "\n");
    }
  }

  // 4. chunks, CTA ranges, phases, on the SMs the tail leaves to the stream
  double stream_cost = 0.0, tail_cost = 0.0;
  L->tail_sms = sweep_tail_sms(h, cstart, n_bands, B, c.nnz - nnz, n_cov - n_str, c.n_rows - n_cov, &stream_cost, &tail_cost);
  sweep_plan_t plan;
  if (!plan_sweep(cstart, n_bands, B, h.sm_count - L->tail_sms, plan)) return nullptr;  // step-row numbers overflow 31 bits
  L->band_phase = plan.band_phase;
  L->n_steprows = plan.n_steprows;
  L->n_rowslots = plan.n_rowslots;
  L->n_chunks   = (int32_t)plan.chunks.size();
  L->n_phases   = (int32_t)plan.phases.size();
  L->n_cta      = plan.n_cta;
  L->chunks     = make_dbuf<sweep_chunk_t>(std::max<size_t>(plan.chunks.size(), 1), h.stream);
  L->phases     = make_dbuf<sweep_phase_t>(std::max<size_t>(plan.phases.size(), 1), h.stream);
  L->cta_phase  = make_dbuf<int32_t>(plan.cta_phase.size(), h.stream);
  dbuf d_fills  = make_dbuf<sweep_fill_t>(std::max<size_t>(plan.fills.size(), 1), h.stream);
  if (!plan.chunks.empty()) {
    CUDA_TRY(cudaMemcpyAsync(L->chunks.data(), plan.chunks.data(), sizeof(sweep_chunk_t) * plan.chunks.size(), cudaMemcpyHostToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(L->phases.data(), plan.phases.data(), sizeof(sweep_phase_t) * plan.phases.size(), cudaMemcpyHostToDevice, h.stream));
    CUDA_TRY(cudaMemcpyAsync(d_fills.data(), plan.fills.data(), sizeof(sweep_fill_t) * plan.fills.size(), cudaMemcpyHostToDevice, h.stream));
  }
  CUDA_TRY(cudaMemcpyAsync(L->cta_phase.data(), plan.cta_phase.data(), sizeof(int32_t) * plan.cta_phase.size(), cudaMemcpyHostToDevice, h.stream));
  sync(h);  // the host vectors are pageable
  L->cursor = make_dbuf<int>(L->n_phases + 2, h.stream);  // the last two: the tail's
  CUDA_TRY(cudaMemsetAsync(L->cursor.data(), 0, sizeof(int) * (L->n_phases + 2), h.stream));

  // 5. step-rows and row slots
  L->ids  = make_dbuf<uint4>((size_t)std::max<int64_t>(L->n_steprows, 1) * 32, h.stream);
  L->rows = make_dbuf<int32_t>(std::max<int64_t>(L->n_rowslots, 1), h.stream);
  const bool weighted = c.weights.data() != nullptr;
  if (weighted) L->w = dbuf((size_t)std::max<int64_t>(L->n_steprows, 1) * 32 * kHotSlot * es, h.stream);
  L->bank_order = h.tune.sweep_bank_order && es == 4;  // a double spans two banks
  if (!plan.chunks.empty()) {
    const int grid = (int)plan.chunks.size();
    if (es == 4 && L->bank_order)
      B200_LAUNCH(h, (k_sweep_fill<float, true>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<float>(), W, L->ids.as<uint4>(), L->w.as<float>(), L->rows.as<int32_t>());
    else if (es == 4)
      B200_LAUNCH(h, (k_sweep_fill<float, false>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<float>(), W, L->ids.as<uint4>(), L->w.as<float>(), L->rows.as<int32_t>());
    else
      B200_LAUNCH(h, (k_sweep_fill<double, false>), grid, kFillWarps * 32, 0, L->chunks.as<sweep_chunk_t>(), d_fills.as<sweep_fill_t>(),
                  perm2.as<int32_t>(), piece_start.as<int32_t>(), piece_len.as<int32_t>(), piece_row.as<int32_t>(), idx,
                  c.weights.as<double>(), W, L->ids.as<uint4>(), L->w.as<double>(), L->rows.as<int32_t>());
  }
  check_last("sweep layout");
  sync(h);
  tr.mark("sweep layout: fill");
  if (n_str < n_cov) {
    build_tail_layout(h, c, nv, es, *L);
    tr.mark("sweep layout: tail");
    if (tr.on) {
      std::fprintf(stderr, "[sweep] tail: %d runs, %d tiles, %d units, %.1f MB of ids\n", L->n_tail_runs,
                   L->tail_runs.back().first_tile, L->tail_runs.back().first_unit, (double)L->tail_runs.back().id_off * 4 / 1e6);
    }
  }
  if (tr.on) {
    std::fprintf(stderr, "[sweep] %lld step-rows = %.1f MB of ids, %lld row slots = %.1f MB, %d chunks, %d phases, %d CTAs\n",
                 (long long)L->n_steprows, (double)L->n_steprows * 512 / 1e6, (long long)L->n_rowslots,
                 (double)L->n_rowslots * 4 / 1e6, L->n_chunks, L->n_phases, L->n_cta);
    std::fprintf(stderr, "[sweep] split: tail on %d of %d SMs%s (cost: stream %.4g, tail %.4g = %.1f %%)\n", L->tail_sms,
                 h.sm_count, h.tune.sweep_tail_sms >= 0 ? ", forced" : "", stream_cost, tail_cost,
                 100.0 * tail_cost / std::max(stream_cost + tail_cost, 1.0));
    for (int band = 0; band < n_bands; ++band) {  // slice loads: a CTA loads a block's slice once per phase
      const int p0 = plan.band_phase[band], p1 = plan.band_phase[band + 1];
      const int c0 = p1 > p0 ? plan.phases[p0].chunk_begin : 0, c1 = p1 > p0 ? plan.phases[p1 - 1].chunk_end : 0;
      std::fprintf(stderr, "[sweep] band %d rows [%d,%d): %d pieces, %d chunks, %d phases = slice loads\n", band,
                   L->band_row[band], L->band_row[band + 1], cstart[(band + 1) * B * kNumKinds] - cstart[band * B * kNumKinds],
                   c1 - c0, p1 - p0);
    }
  }
  return L;
}

}  // namespace

// flat copy of plan_sweep's result for the debug C entries (CPU tests)
bool debug_plan_sweep(std::vector<int32_t> const& cstart, int n_bands, int B, int sm_count, int64_t totals[3],
                      std::vector<int32_t>& chunks4, std::vector<int32_t>& fills4, std::vector<int32_t>& phases4,
                      std::vector<int32_t>& cta_phase, std::vector<int32_t>& band_phase)
{
  sweep_plan_t P;
  if (!plan_sweep(cstart, n_bands, B, sm_count, P)) return false;
  totals[0] = P.n_steprows; totals[1] = P.n_rowslots; totals[2] = P.n_cta;
  for (auto const& x : P.chunks) chunks4.insert(chunks4.end(), {x.sr_begin, x.row_begin, x.n_groups, x.kind});
  for (auto const& x : P.fills) fills4.insert(fills4.end(), {x.piece_begin, x.piece_end, x.block, x.pad});
  for (auto const& x : P.phases) phases4.insert(phases4.end(), {x.block, x.chunk_begin, x.chunk_end, x.pad});
  cta_phase  = P.cta_phase;
  band_phase = P.band_phase;
  return true;
}

sweep_layout_t const* sweep_layout(handle_impl const& h, csx_t const& c, int32_t n_vertices, size_t elem_size)
{
  if (!c.sweep) c.sweep = std::make_unique<sweep_cache_t>();
  auto& slot = c.sweep->of(elem_size);
  if (slot.tried) return slot.layout.get();
  slot.tried = true;
  // 32-bit edge positions / step-row numbers; build_sweep_layout itself gives up (nullptr) if the step-rows overflow
  if (!c.degree_sorted || c.seg[kNumSeg - 2] <= 0 || c.nnz < h.tune.sweep_min_edges || c.offs64 || c.nnz >= (1ll << 31) - 4096)
    return nullptr;
  slot.layout = build_sweep_layout(h, c, n_vertices, elem_size);
  return slot.layout.get();
}

csx_t::csx_t()  = default;
csx_t::~csx_t() = default;

}  // namespace b200

extern "C" cugraph_error_code_t cugraph_b200_debug_plan_sweep_bands(const int32_t* class_start, int n_bands, int n_blocks,
                                                                    int sm_count, int64_t* totals, int32_t* chunks,
                                                                    int32_t* fills, size_t chunks_capacity, size_t* n_chunks,
                                                                    int32_t* phases, size_t phases_capacity, size_t* n_phases,
                                                                    int32_t* cta_phase, size_t cta_capacity,
                                                                    int32_t* band_phase, cugraph_error_t** error)
{
  using namespace b200;
  return guarded(error, [&] {
    B200_EXPECTS(class_start && totals && chunks && fills && phases && cta_phase && band_phase && n_chunks && n_phases,
                 CUGRAPH_INVALID_INPUT, "null argument");
    B200_EXPECTS(n_bands >= 1 && n_blocks >= 0 && sm_count >= 1, CUGRAPH_INVALID_INPUT, "bad parameter");
    std::vector<int32_t> cstart(class_start, class_start + (size_t)n_bands * n_blocks * kNumKinds + 1);
    std::vector<int32_t> c4, f4, p4, r, bp;
    int64_t t[3];
    B200_EXPECTS(debug_plan_sweep(cstart, n_bands, n_blocks, sm_count, t, c4, f4, p4, r, bp), CUGRAPH_INVALID_INPUT,
                 "step-row numbers overflow 31 bits");
    B200_EXPECTS(c4.size() / 4 <= chunks_capacity && p4.size() / 4 <= phases_capacity && r.size() <= cta_capacity,
                 CUGRAPH_INVALID_INPUT, "output capacity too small");
    std::copy(t, t + 3, totals);
    std::copy(c4.begin(), c4.end(), chunks);
    std::copy(f4.begin(), f4.end(), fills);
    std::copy(p4.begin(), p4.end(), phases);
    std::copy(r.begin(), r.end(), cta_phase);
    std::copy(bp.begin(), bp.end(), band_phase);
    *n_chunks = c4.size() / 4;
    *n_phases = p4.size() / 4;
  });
}

extern "C" cugraph_error_code_t cugraph_b200_debug_plan_sweep(const int32_t* class_start, int n_blocks, int sm_count,
                                                              int64_t* totals, int32_t* chunks, int32_t* fills,
                                                              size_t chunks_capacity, size_t* n_chunks, int32_t* phases,
                                                              size_t phases_capacity, size_t* n_phases, int32_t* cta_phase,
                                                              size_t cta_capacity, cugraph_error_t** error)
{
  int32_t band_phase[2];
  return cugraph_b200_debug_plan_sweep_bands(class_start, 1, n_blocks, sm_count, totals, chunks, fills, chunks_capacity, n_chunks,
                                             phases, phases_capacity, n_phases, cta_phase, cta_capacity, band_phase, error);
}
