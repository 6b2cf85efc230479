// pr_plan.cuh — the JACOBI PageRank layout (PrPlan) and what its build (pr_layout.cu) and its sweep
// (pagerank.cu) both need: the layout constants, the cyclic deal of rows over ranks, and the launch-shape
// stage that ends the build.
#pragma once
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "csr_split.h"

namespace gb {

constexpr int PR_WARPS = 32;        // warps per CTA of the sweep kernels: one persistent CTA per SM
constexpr int PR_THREADS = PR_WARPS * 32;
constexpr int PR_SELL_THREADS = 512; // SELL kernel: two 16-warp CTAs per SM and no shared memory (L1 keeps it all)
constexpr int PR_FIN_THREADS = 256;
constexpr uint32_t PR_MAX_PROFILE_EVENTS = 256;  // sweeps bracketed by CUDA events when profiling is on
constexpr uint32_t CB_G = 4;                 // block-local ids per group (one 64-bit load per lane)
constexpr uint32_t CB_BLOCK_DEFAULT = 49152; // source-vector entries per block (192 KB of shared memory)
constexpr uint32_t CB_BLOCK_MAX = 56 * 1024;
constexpr double CB_TAU_DEFAULT = 1.5;       // a (row, block) pair gets a segment if it expects >= tau edges
constexpr uint32_t CB_MAX_BLOCKS = 8192;     // hot blocks kept (the staircase rarely needs more than ~1000)
constexpr uint32_t CB_TASK_CHUNKS = 32;      // chunks per task (one per warp)
constexpr uint32_t CB_WIDE_MIN = 128;        // chunks of at least this many groups take k_pr_cb's 128-group step
// groups per lane in k_pr_cb's steps over chunk [g0, g1); k_cb_bank_order orders the ids for those steps
__host__ __device__ __forceinline__ uint32_t cb_step_groups(uint32_t g0, uint32_t g1) {
  return g1 - g0 >= CB_WIDE_MIN ? 4u : 2u;
}
constexpr uint32_t SELL_FEW = 4;             // rows with segments in at most this many blocks are finished by k_pr_sell itself
constexpr uint32_t FIN_CTA_BLOCKS = 64;      // finish: 32-row groups with segments in more blocks get a CTA each
constexpr uint32_t CB_NONE = 0xFFFFFFFFu;
constexpr uint32_t CB_MEGA_DEG = 32768;      // layout build: rows with more in-edges go through one stable radix sort
constexpr uint32_t CB_MEGA_JBITS = 14;       // key = row << 14 | block rank (0x3FFF = not in a segment)
constexpr uint32_t CB_ILP = 4;               // 32-edge batches in flight per warp in the layout build
// chunk flags (bits 24.. of PrChunk.w)
constexpr uint32_t CB_HEAD_CONT = 1u, CB_TAIL_CONT = 2u, CB_INTERIOR = 4u;

// ---- the cyclic deal of 32-row slices over the ranks of the 1-D edge-cut ---------------------------
struct PrDeal {
  uint32_t P = 1, p = 0;
};
__host__ __device__ __forceinline__ uint32_t deal_global(uint32_t l, uint32_t P, uint32_t p) {
  return (((l >> 5) * P + p) << 5) | (l & 31u);
}
// number of local rows whose global index is below R
static inline uint32_t deal_count(uint32_t R, uint32_t P, uint32_t p) {
  const uint32_t F = R >> 5, rem = R & 31u;
  const uint32_t full = F > p ? (F - p + P - 1) / P : 0;
  uint32_t c = full * 32;
  if (rem && (F % P) == p) c += rem;
  return c;
}

struct PrPlan {
  uint32_t n = 0;
  uint32_t n_active = 0;  // global rows with in-degree > 0 (renumbered to [0, n_active))
  uint64_t m = 0;
  PrDeal deal;
  uint32_t n_loc = 0;     // local active rows
  uint32_t n_cb = 0;      // local rows [0, n_cb) own at least one column-block segment
  uint64_t loc_edges = 0; // in-edges of the local rows
  uint64_t cb_edges = 0;  // of which served from column blocks
  DevBuf<uint32_t> new_id;    // old id -> internal id
  DevBuf<uint32_t> outdeg;    // out-degree by internal id [n]
  // column blocks
  uint32_t B = 0, KB = 0;       // block entries, hot blocks
  uint64_t S = 0;               // staircase size = sum of nrows[j]
  uint64_t NG = 0;              // groups in all block streams
  uint32_t chunk_groups = 0, n_chunks = 0, n_tasks = 0, n_fix = 0;
  uint32_t fix_max_row = 0;     // largest local row that owns a segment cut by a chunk boundary
  uint32_t n_mega = 0;          // local rows [0, n_mega) went through the sort path of the layout build
  uint32_t last_hot_block = CB_NONE;  // largest source block index among the hot blocks
  DevBuf<uint32_t> blk;         // [KB] source block of hot rank j
  DevBuf<uint32_t> nrows;       // [KB] local rows [0, nrows[j]) have a segment in block j (non-increasing)
  DevBuf<uint32_t> poff;        // [KB+1] staircase offsets
  DevBuf<uint2> cb_ids;         // [NG] groups of 4 block-local 16-bit ids (pad id = B)
  DevBuf<uint32_t> cb_bits;     // [NG/32 + 8] bit g set <=> group g starts a segment
  DevBuf<float> partial;        // [S] one partial sum per (block, row) pair
  DevBuf<uint4> chunks;         // [n_chunks] (g_begin, g_end, row_before, j | flags << 24)
  DevBuf<uint32_t> tail_slot;   // [n_chunks] staircase slot of the segment cut by the chunk end
  DevBuf<double> side;          // [2 n_chunks] head / tail parts of segments cut by chunk boundaries
  DevBuf<uint32_t> fix_list;    // [n_fix] chunks whose tail segment continues in later chunks
  DevBuf<uint2> tasks;          // [n_tasks] (first chunk, chunk count | block rank << 8), fattest blocks first
  DevBuf<uint32_t> task_ctr;    // [grid_cb] per-range task cursors (reset by the finish kernel)
  DevBuf<float> rem;            // [n_cb] SELL remainder sums of the rows that also have segments
  DevBuf<uint32_t> fin_kb;      // [ceil(n_cb / 32)] blocks of the first row of each 32-row group (finish kernel)
  // SELL-32 (all local active rows; rows < n_cb hold only the edges outside their segments)
  uint32_t num_slices = 0;
  DevBuf<uint4> sell;         // slice-major, then 4-edge group, then lane
  DevBuf<uint2> slice_meta;   // per slice: (first uint4 index, uint4 groups per lane)
  // state (single-GPU path; the shard API brings its own vectors)
  DevBuf<float> x[2];
  DevBuf<float> scores;
  unsigned grid_cb = 0, grid_sell = 0, grid_fin = 1;
  uint32_t n_fin_warp = 0;   // rows [0, n_fin_warp) own segments in more than FIN_CTA_BLOCKS blocks
  uint32_t fin_u = 4;        // finish: row groups per warp iteration (template argument of k_pr_finish)
  uint32_t fin_hub_ctas = 0; // finish CTAs that take the hub groups (the others take rows [n_fin_warp, n_fin))
  uint32_t n_fin = 0;        // rows [0, n_fin) are completed by k_pr_finish, [n_fin, n_cb) by k_pr_sell
  uint32_t few_nrows[SELL_FEW] = {}, few_poff[SELL_FEW] = {};
  DevBuf<double> block_err;  // per CTA error partials (SELL CTAs, then finish CTAs)
  DevBuf<double> err_hist;   // error of each sweep of the current batch
  DevBuf<uint32_t> ctrl;     // [0] = done flag (sweep number at which tolerance was met), [1] = ticket
  size_t smem_cb = 0;
  std::vector<cudaEvent_t> prof_events;
  // GB_PR_TRACE=1 (diagnostics): CUDA events between the kernels of every sweep; averages are printed
  // to stderr when the layout is released
  bool trace = false;
  mutable std::vector<cudaEvent_t> trace_events;  // 5 per traced sweep
  uint64_t bytes() const {
    return new_id.bytes() + outdeg.bytes() + blk.bytes() + nrows.bytes() + poff.bytes() + cb_ids.bytes() +
           cb_bits.bytes() + partial.bytes() + chunks.bytes() + tail_slot.bytes() + side.bytes() +
           fix_list.bytes() + tasks.bytes() + rem.bytes() + fin_kb.bytes() + sell.bytes() + slice_meta.bytes() + x[0].bytes() +
           x[1].bytes() + scores.bytes() + block_err.bytes() + err_hist.bytes();
  }
};

// blocks in which local row l owns a segment: the first j with nrows[j] <= l (nrows is non-increasing)
__host__ __device__ __forceinline__ uint32_t fin_blocks_of(const uint32_t* __restrict__ nrows, uint32_t KB, uint32_t l) {
  uint32_t lo = 0, hi = KB;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (nrows[mid] > l) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Where a layout build (pr_layout.cu) finds the degrees: the internal order, the active rows and the hot
// blocks come from the full in- and out-offsets (n + 1 each, device memory of `device`), and the build runs
// on `stream`.  m is the graph's edge count (the hot-block threshold tau m / e_b).  The rows themselves come
// from a separate row source (layout_end), which need not be the in-CSR: it only has to hold the rows of the
// rank being built, in CSR order.
struct PrSource {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint32_t n = 0;
  uint64_t m = 0;
  const uint32_t* in_off = nullptr;
  const uint32_t* out_off = nullptr;
  // a feed of the whole in-CSR whose targets are still landing, in the chunks `chunks`: the row source is its
  // in-CSR, and the build checks and classifies each chunk as soon as its landed event fires
  const CsrFeed* feed = nullptr;
  const CsrChunks* chunks = nullptr;
};
struct LayoutBuild;
// The order stage of rank deal.p's layout; afterwards layout_new_id(*out) (old id -> internal id, n entries on
// src.device) is valid.
gb_status layout_begin(const PrSource& src, PrDeal deal, LayoutBuild** out);
const uint32_t* layout_new_id(const LayoutBuild* b);
// The other stages, ending with plan_sweep_shape.  Row v's in-edges are row_tgt[row_off[v] .. row_off[v + 1])
// (row_off indexed by original id, row_entries entries in all); only the rows of rank deal.p are read.  Frees
// b whatever it returns.
gb_status layout_end(LayoutBuild* b, const uint32_t* row_off, const uint32_t* row_tgt, uint64_t row_entries,
                     PrPlan** out_plan);
void layout_free(LayoutBuild* b);
gb_status build_pr_plan(const PrSource& src, PrDeal deal, const uint32_t* row_off, const uint32_t* row_tgt,
                        uint64_t row_entries, PrPlan** out_plan);
// the layout of rank deal.p's rows of g: its in-CSR is both the degree and the row source
gb_status build_pr_plan(const gb_graph* g, PrDeal deal, PrPlan** out_plan);
// a shard of the sweep API that owns `plan` and no graph (gb_pr_shards_csr_u32; pagerank.cu)
gb_status shard_from_plan(int device, PrPlan* plan, gb_pr_shard** out);

// The O(1) host checks of a host PageRank CSR (n + 1 in- and out-offsets, the in-targets), in the order and
// with the messages of every entry point that takes one (multi.cu)
gb_status check_pr_host_csr(uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt, const uint32_t* out_off);
// The layouts of ranks 0 .. U-1 (U = devs.size() * V, rank r on devs[r / V]) of a host CSR that passed
// check_pr_host_csr (multi.cu).  Part u of the split (pr_split, targets in chunks of about chunk_edges >= 1
// edges) is uploaded by the device of rank u; the offsets are checked on the device.  A lone rank builds its
// layout from its part as the chunks land; with several, every rank gathers the rows it owns from all parts into
// a local in-CSR first.  On success plans holds U plans, the caller's to free; on failure nothing is left.
gb_status pr_csr_plans(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                       const uint32_t* in_tgt, const uint32_t* out_off, uint64_t chunk_edges,
                       std::vector<PrPlan*>* plans);
// launch shapes of the sweep kernels, their error buffers and k_pr_cb's shared-memory size (pagerank.cu).
// h_nrows / h_poff: the staircase (nrows[], poff[]) as the layout build holds it on the host.
gb_status plan_sweep_shape(PrPlan* p, const std::vector<uint32_t>& h_nrows, const std::vector<uint32_t>& h_poff,
                           int dev_sms, cudaStream_t s);

}  // namespace gb
