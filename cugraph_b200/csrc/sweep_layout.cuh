// The layout the shared-memory pull sweep (sweep.cuh) reads, built by sweep_layout.cu.  Private to the sweep: the rest of the
// library reaches it through pull_sweep / prepare_pull_sweep (graph.cuh).
#pragma once
#include "graph.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// Column-blocked "piece stream" of the rows [0, n_str) for the shared-memory pull sweep (sweep.cuh).  n_str is a degree-bin
// bound: on large graphs the rows of in-degree < kSweepTailDegree (the TAIL) leave the stream and are swept by a row
// kernel instead (k_sweep_tail); on smaller graphs the stream covers every non-empty row.
// The source (column) space is cut into B blocks of W vertices (W * sizeof(T) = 192 KiB minus 64 zero columns: the slice of
// x a persistent CTA keeps in shared memory).  Rows keep their neighbours sorted by source id, so a row's adjacency is
// already partitioned by block; every (row, block) SEGMENT is cut into PIECES of <= 64 entries.  A piece is stored with
// 16-bit local column ids in one of 11 KINDS: S / Q / H = 1 / 2 / <= 4 entries (2 / 4 / 8 bytes of ids), F1..F8 = 1..8 lane
// slots of 8 entries (16 bytes each; short pieces are padded with a column that reads 0).  The stream rows are split into
// BANDS of consecutive rows (a multiple of kBandRowAlign each, sized so that a band's fp64 accumulators stay in the L2) and
// pieces are ordered by (band, block, kind): the sweep runs band after band.  The unit every kernel step works on is a
// STEP-ROW = 32 lanes x 16 bytes of ids (one 128-bit load per lane, 512 contiguous bytes per warp): it holds 256 S pieces, 128 Q pieces, 64 H pieces, or one of the c slots of 32 Fc
// pieces (a GROUP of kind Fc is c consecutive step-rows, lane = piece).  Row ids (int32, -1 = unused piece) are stored per
// group so that a lane's rows are contiguous: 8 / 4 / 2 / 1 per lane.
// ---------------------------------------------------------------------------------------------
constexpr int kHotSliceBytes = 192 * 1024;  // x slice a CTA keeps in shared memory
constexpr int kHotZeroPad    = 64;          // trailing elements of the slice that hold zeros (padding target)
constexpr int kHotSlot       = 8;           // entries per lane slot

constexpr int kBandRowAlign = 512;  // band bounds: a multiple of the finish kernel's rows per warp (k_sweep_finish)

// Tail of the piece stream: a row of small in-degree has its few edges in different column blocks, so the stream pays one
// fp64 RED per edge for it, and such rows are most of the rows (their accumulators decide how many bands are needed).
// Rows of in-degree < kSweepTailDegree are gathered by k_sweep_tail instead, on graphs of at least kSweepTailMinEdges edges.
// A kSegThreshold value.  Measured on an H100 80GB HBM3 at 700 W, RMAT-24 PageRank step, with the row-per-thread tail kernel
// of before: 86.3 ms without a tail, 78.8 / 73.4 / 72.7 / 74.5 ms with bounds 4 / 8 / 16 / 32 (DESIGN.md §3.2); from 8 on the
// stream needs one band.  With the tail layout below, at 400 W: 73.1 / 68.3-70.6 / 69.1 ms with bounds 8 / 16 / 32 (sweep
// 0.660 / 0.635-0.642 / 0.612 ms): 32 is not yet separated from 16 by more than the run-to-run spread.
constexpr int kSweepTailDegree         = 16;
constexpr long long kSweepTailMinEdges = 1ll << 24;

constexpr int kNumKinds = 11;  // S, Q, H, F1..F8
constexpr int kKindS = 0, kKindQ = 1, kKindH = 2, kKindF1 = 3;
__host__ __device__ __forceinline__ int kind_steps(int kind) { return kind < kKindF1 ? 1 : kind - 2; }  // step-rows per group
__host__ __device__ __forceinline__ int kind_pieces(int kind) { return kind == kKindS ? 256 : (kind == kKindQ ? 128 : (kind == kKindH ? 64 : 32)); }
// groups per chunk (a chunk = consecutive groups of one kind in one block = what a warp loads into its registers at once:
// at most 8 x 128 bits of ids / rows + 2 row words, chunk_regs_t in sweep.cuh)
__host__ __device__ __forceinline__ int kind_chunk_groups(int kind)
{
  return kind == kKindS ? 2 : (kind == kKindQ ? 4 : (kind == kKindH ? 4 : (kind == kKindF1 ? 6 : (kind == kKindF1 + 1 ? 3 : (kind <= kKindF1 + 3 ? 2 : 1)))));
}

struct sweep_chunk_t {  // 16 bytes
  int32_t sr_begin;   // first step-row
  int32_t row_begin;  // first row slot
  int32_t n_groups;   // 1 .. kind_chunk_groups(kind)
  int32_t kind;
};
struct sweep_phase_t {  // consecutive chunks of one block inside one CTA's range; its cursor is phase-indexed
  int32_t block;
  int32_t chunk_begin;
  int32_t chunk_end;
  int32_t pad;
};

// ---------------------------------------------------------------------------------------------
// Tail layout of the rows [n_str, n_cov) for k_sweep_tail (sweep.cuh).  Rows are degree-descending, so the tail is made of
// RUNS of rows of one in-degree d (< kSweepTailDegree <= 32).  A run is cut into TILES of 32 consecutive rows, lane l = row
// first_row + 32 * t + l; entry k of lane l of tile t of a run sits at tail_ids[id_off + t * 32 * d + k * 32 + l] (int32 source
// id, a row's entries in ascending source order: hubs first).  No offsets and no padding inside a run: every warp-wide load
// of ids is one 128-byte line; only the last tile of a run has lanes without a row, whose entries read column n_vertices (x
// is zero there).  A WORK UNIT is tail_unit_tiles(d) consecutive tiles of one run (the last one of a run may be shorter):
// about kTailUnitEntries entries per lane whatever d, consecutive in tail_ids.
// ---------------------------------------------------------------------------------------------
constexpr int kTailTile        = 32;  // rows per tile (= lanes)
constexpr int kTailUnitEntries = 24;  // entries per lane in a work unit, at least one tile (ids held in registers, twice)
constexpr int kTailMaxDegree   = 31;  // kSegThreshold[0] - 1: the largest bound leaves rows of in-degree <= 31 in the tail
__host__ __device__ constexpr int tail_unit_tiles(int d) { return d >= kTailUnitEntries ? 1 : kTailUnitEntries / d; }

struct tail_run_t {   // 24 bytes; a run table ends with a sentinel that holds the totals (first_row = n_cov)
  int32_t degree;
  int32_t first_row;
  int32_t first_tile;
  int32_t first_unit;
  int64_t id_off;     // first entry in tail_ids
};

struct sweep_layout_t {
  int W{0};               // source columns per block (= slice elements - kHotZeroPad)
  int B{0};               // blocks
  int32_t n_cov{0};       // rows [0, n_cov) are covered = every non-empty row (rows are degree-descending)
  int32_t n_str{0};       // rows [0, n_str) are in the piece stream (a degree-bin bound <= n_cov); [n_str, n_cov) is the tail
  int64_t nnz{0};         // edges of the graph (the stream holds the first offsets[n_str] of them)
  bool bank_order{false};  // entries inside the F slots ordered by shared-memory bank (4-byte values)
  int64_t n_steprows{0};
  int64_t n_rowslots{0};
  int64_t n_pieces{0};
  dbuf ids;        // n_steprows x 32 x uint4 (8 x uint16: column - block * W; padding -> one of the zero columns)
  dbuf w;          // n_steprows x 32 x 8 x T, padding 0; or empty
  dbuf rows;       // n_rowslots x int32
  dbuf chunks;     // n_chunks x sweep_chunk_t
  dbuf phases;     // n_phases x sweep_phase_t
  dbuf cta_phase;  // (n_bands * n_cta + 1) x int32: in band b, CTA c owns phases [cta_phase[b * n_cta + c], the next entry)
                   // (cost-balanced, contiguous chunks)
  dbuf cursor;     // n_phases + 2 x int: next chunk of the phase (relative), reset by the band's finish kernel; then the tail's
                   // next work unit, in two slots that alternate from sweep to sweep (tail_sweeps): each tail launch uses
                   // one and clears the other, which the tail launch before it used and left behind
  int32_t n_chunks{0};
  int32_t n_phases{0};
  int n_cta{0};     // persistent CTAs of the stream: the SMs the tail does not take
  int tail_sms{0};  // SMs the tail sweeps on beside the stream, from a side stream; 0: after the bands, on every SM
  mutable unsigned tail_sweeps{0};  // tail launches so far: the cursor slot of the next one is tail_sweeps & 1
  int n_bands{1};
  std::vector<int32_t> band_row;    // n_bands + 1: band b holds rows [band_row[b], band_row[b+1]); band_row[n_bands] = n_str
  std::vector<int32_t> band_phase;  // n_bands + 1: the phases of band b are [band_phase[b], band_phase[b+1])
  // the tail (rows [n_str, n_cov)), when there is one
  int n_tail_runs{0};
  std::vector<tail_run_t> tail_runs;  // n_tail_runs + 1 (sentinel), on the host
  dbuf tail_run;                      // the same on the device
  dbuf tail_ids;                      // tail_runs[n_tail_runs].id_off x int32
  dbuf tail_w;                        // the same x T, padding 0; or empty
};

// what a csx_t caches for the sweep: per element size (4 or 8 bytes), whether a layout was tried and what it built (or nullptr)
struct sweep_cache_t {
  struct slot_t { bool tried{false}; std::unique_ptr<sweep_layout_t> layout; } slot[2];
  slot_t& of(size_t elem_size) { return slot[elem_size == 4 ? 0 : 1]; }
};

// piece stream for elements of `elem_size` bytes, or nullptr when the graph is too small for it or has 64-bit offsets
sweep_layout_t const* sweep_layout(handle_impl const& h, csx_t const& c, int32_t n_vertices, size_t elem_size);

}  // namespace b200
