// pr_plan.cuh — the JACOBI PageRank layout (PrPlan) and what its build (pr_layout.cu), its sweep (pagerank.cu),
// the host-CSR part pipeline (pr_csr.cu) and the communicator (multi.cu) share: the layout constants, the cyclic
// deal of rows over ranks, the launch-shape stage that ends the build, and the rules every PageRank call keeps.
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

constexpr uint32_t VB_ALIGN = 32;            // virtual blocks start at multiples of 32 slots of V (128-byte lines)
constexpr uint32_t VB_RUN_ALIGN = 8;         // runs of V start at multiples of 8 slots (32-byte sectors) and fill them
constexpr uint16_t BIN_PAD = 0xFFFFu;        // pass A: a position that holds no pair (B < 2^16 - 1)
constexpr uint32_t BIN_STEP = 256;           // pass A: positions per warp step (8 groups of 32, 8 per lane)
constexpr uint32_t BIN_CHUNK = 8;            // pass A: steps per chunk (2048 positions, one warp)
// pass A: where the id of position pos is stored.  Inside a step, position 32 k + L sits at 8 L + k, so that lane L
// reads its positions L, L + 32, .., L + 224 with one 128-bit load
__host__ __device__ __forceinline__ uint32_t bin_id_index(uint32_t pos) {
  return (pos & ~(BIN_STEP - 1)) | (pos & 31u) << 3 | (pos >> 5 & 7u);
}

// ---- the cyclic deal of 32-row slices over the ranks of the 1-D edge-cut ---------------------------
struct PrDeal {
  uint32_t P = 1, p = 0;  // rank p of P
  PrDeal() = default;
  PrDeal(uint32_t world, uint32_t rank) : P(world), p(rank) {}
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

// One id stream of k_pr_cb's walker and what its consumers read: KB blocks; block j's local rows [0, nrows[j])
// own one segment each, row by row, and the segments' partials start at poff[j].  The hot blocks (PrPlan::hot,
// k_pr_cb<CB_MAIN>) are blocks of the source vector: blk[j] is the source block of hot rank j.  Pass B of the
// virtual blocks (PrVBlocks::virt, k_pr_cb<CB_VIRT>) walks the slots of V: blk[j] .. blk[j + 1] are virtual
// block j's slot bounds, poff[j] is partition j's first local row and nrows[j] its row count, so that every
// local row's partial lands at its own index.
struct CbStream {
  uint32_t KB = 0;              // blocks
  uint64_t S = 0;               // segments = partials = sum of nrows[j]
  uint64_t NG = 0;              // groups in all blocks
  DevBuf<uint32_t> blk;         // [KB] hot rank j's source block (pass B: [KB + 1] V slot bounds, multiples of VB_ALIGN)
  DevBuf<uint32_t> nrows;       // [KB] rows with a segment in block j (non-increasing for the hot blocks)
  DevBuf<uint32_t> poff;        // [KB + 1] first partial of block j
  DevBuf<uint2> ids;            // [NG] groups of 4 block-local 16-bit ids (pad id = B; pass B: its window)
  DevBuf<uint32_t> bits;        // [NG/32 + 8] bit g set <=> group g starts a segment
  DevBuf<float> partial;        // [S] one partial sum per segment
  // the chunks and tasks (k_pr_cb's unit of work), as cb_chunk_table cuts them
  uint32_t chunk_groups = 0, n_chunks = 0, n_tasks = 0, n_fix = 0;
  uint32_t fix_max_row = 0;     // largest row that owns a segment cut by a chunk boundary
  DevBuf<uint4> chunks;         // [n_chunks + 1] (g_begin, g_end, row_before, j | flags << 24); a zero sentinel
  DevBuf<uint32_t> tail_slot;   // [n_chunks] partial of the segment cut by the chunk end
  DevBuf<double> side;          // [2 n_chunks] head / tail parts of segments cut by chunk boundaries
  DevBuf<uint32_t> fix_list;    // [n_fix] chunks whose tail segment continues in later chunks
  DevBuf<uint2> tasks;          // [n_tasks] (first chunk, chunk count | block rank << 8), fattest blocks first
  uint64_t bytes() const {
    return blk.bytes() + nrows.bytes() + poff.bytes() + ids.bytes() + bits.bytes() + partial.bytes() + chunks.bytes() +
           tail_slot.bytes() + side.bytes() + fix_list.bytes() + tasks.bytes();
  }
};

// Virtual blocks: the edges that no column-block segment takes (COLD edges) on graphs whose source vector does
// not fit in L2.  The rows are cut into contiguous PARTITIONS of at most B cold edges; each distinct (source,
// partition) PAIR owns one slot of the value buffer V (partition-major, by source inside a partition: a
// partition's slots are one virtual block).  The pairs of one source block inside one partition are a RUN of
// consecutive slots.  With `sectors`, every run starts at a multiple of VB_RUN_ALIGN slots and is followed by pad
// slots up to the next one, which pass A zeroes in the step that stores the run's last value: every 32-byte
// sector of V is then written whole by one warp, and none is left half-written in L2 to be read back from HBM
// when it is evicted.  A padded virtual block may then hold more than B slots; pass B's window (its shared-memory
// block, pad id and zero slot) is the largest that fits.  Without `sectors` (some padded partition would not fit
// in that window) the runs are packed and pass B's window is B.  Pass A writes the values of each source block's
// pairs to V, run by run, from the block in shared memory; it runs inside k_pr_cb<CB_FUSED>, whose tasks carry a
// source block's hot chunks and its pass-A chunks side by side, so that the block is loaded once for both.  Pass
// B (k_pr_cb<CB_VIRT>) walks a column-block stream over the virtual blocks, with V in place of the source
// vector, and leaves one partial per local row.  k_pr_finish then completes every local row, and k_pr_sell does
// not run.
struct PrVBlocks {
  uint64_t pairs = 0, edges = 0;  // (source, partition) pairs and the cold edges they serve
  uint32_t bin_blocks = 0, n_runs = 0;
  uint32_t wide_steps = 0;      // pass A steps whose positions touch more than 32 runs (the run-window loop)
  bool sectors = false;         // runs start on 32-byte sectors and pass A zeroes their pad slots
  uint32_t window = 0;          // pass B's block: V slots of its shared-memory block, and its pad id
  uint64_t slots = 0;           // V's length
  DevBuf<float> val;            // V
  // pass A: the pairs in (source block, partition, source) order, each block's share starting at a multiple of
  // BIN_STEP positions (BIN_PAD in between); a RUN is the pairs of one (block, partition), consecutive slots of V
  DevBuf<uint16_t> bin_ids;     // block-local source id of every position, at bin_id_index(position)
  DevBuf<uint32_t> bin_bits;    // per 32 positions: bit i set <=> position 32 g + i starts a run; then one step
                                // whose first position starts a run (the end of the last one)
  DevBuf<uint32_t> bin_grun;    // per 32 positions: the last run that starts at or before position 32 g
  DevBuf<uint32_t> bin_runs;    // [n_runs + 32] first V slot - first position of each run (mod 2^32); 32 spare
  DevBuf<uint2> bin_chunks;     // [steps s0, s1) of one block: a warp's unit of pass A
  // k_pr_cb<CB_FUSED>'s tasks over the union of the hot blocks and pass A's source blocks, fattest blocks first
  // (bytes of ids and values), a block's tasks consecutive: (first hot chunk, first pass-A chunk, hot chunks |
  // pass-A chunks << 8, source block).  Task i of a block holds the block's i-th run of up to CB_TASK_CHUNKS hot
  // chunks (hot.tasks cuts them) and its i-th run of up to CB_TASK_CHUNKS pass-A chunks; either may be empty.
  DevBuf<uint4> tasks;
  uint32_t n_tasks = 0;
  // pass B: one block per partition (KB = partitions), one segment per local row (a padding group when the row
  // has no cold edge); its partials are the cold sums of the local rows
  CbStream virt;
  uint64_t bytes() const {
    return val.bytes() + bin_ids.bytes() + bin_bits.bytes() + bin_grun.bytes() + bin_runs.bytes() +
           bin_chunks.bytes() + tasks.bytes() + virt.bytes();
  }
};

// Which kernel adds the parts of the hot blocks' segments cut by chunk boundaries: one that runs after k_pr_cb
// and before the kernel that completes their rows (plan_sweep_shape decides)
enum class PrFix : uint32_t {
  NONE,    // no segment is cut
  FIXUP,   // a k_pr_fixup launch before k_pr_sell: some cut row is completed by its k_pr_sell lane (few hot blocks)
  SELL,    // k_pr_sell's first warps: every cut row is completed later, by k_pr_finish (rows below n_fin)
  PASS_B,  // pass B's first warps (virtual blocks): k_pr_finish completes every row
};

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
  // column blocks: B entries per block, the hot blocks' stream (the staircase: one partial per (block, row) pair)
  uint32_t B = 0;
  CbStream hot;
  uint32_t n_mega = 0;          // local rows [0, n_mega) went through the sort path of the layout build
  uint32_t last_hot_block = CB_NONE;  // largest source block index among the hot blocks
  DevBuf<uint32_t> task_ctr;    // [task_ranges()] per-range task cursors (reset by the finish kernel)
  DevBuf<float> rem;            // [n_cb] SELL remainder sums of the rows that also have segments
  DevBuf<uint32_t> fin_kb;      // [ceil(n_cb / 32)] blocks of the first row of each 32-row group (finish kernel)
  // SELL-32 (all local active rows; rows < n_cb hold only the edges outside their segments)
  uint32_t num_slices = 0;
  DevBuf<uint4> sell;         // slice-major, then 4-edge group, then lane
  DevBuf<uint2> slice_meta;   // per slice: (first uint4 index, uint4 groups per lane)
  // virtual blocks (vb: they take the cold edges, the SELL slices above are empty and k_pr_sell does not run)
  bool vb = false;
  PrVBlocks v;
  unsigned grid_vb = 0;      // persistent CTAs of pass B
  // state (single-GPU path; the shard API brings its own vectors)
  DevBuf<float> x[2];
  DevBuf<float> scores;
  unsigned grid_cb = 0, grid_sell = 0, grid_fin = 1;  // grid_cb: k_pr_cb<CB_MAIN>, or <CB_FUSED> (vb)
  uint32_t n_fin_warp = 0;   // rows [0, n_fin_warp) own segments in more than FIN_CTA_BLOCKS blocks
  uint32_t fin_u = 4;        // finish: row groups per warp iteration (template argument of k_pr_finish)
  uint32_t fin_hub_ctas = 0; // finish CTAs that take the hub groups (the others take rows [n_fin_warp, n_fin))
  uint32_t n_fin = 0;        // rows [0, n_fin) are completed by k_pr_finish, [n_fin, n_cb) by k_pr_sell
  uint32_t few_nrows[SELL_FEW] = {}, few_poff[SELL_FEW] = {};
  PrFix fix_at = PrFix::NONE;  // the kernel that adds the parts of the hot blocks' cut segments
  DevBuf<double> block_err;  // per CTA error partials (SELL CTAs, then finish CTAs)
  DevBuf<double> err_hist;   // error of each sweep of the current batch
  DevBuf<uint32_t> ctrl;     // [0] = done flag (sweep number at which tolerance was met), [1] = ticket
  size_t smem_cb = 0;        // k_pr_cb<CB_MAIN> and <CB_FUSED>: a source block and its zero slot
  size_t smem_vb = 0;        // pass B: its window of V and the zero slot
  std::vector<cudaEvent_t> prof_events;
  // GB_PR_TRACE=1 (diagnostics): CUDA events between the kernels of every sweep; averages are printed
  // to stderr when the layout is released
  bool trace = false;
  mutable std::vector<cudaEvent_t> trace_events;  // 5 per traced sweep
  uint64_t bytes() const {
    return new_id.bytes() + outdeg.bytes() + hot.bytes() + rem.bytes() + fin_kb.bytes() + sell.bytes() +
           slice_meta.bytes() + x[0].bytes() + x[1].bytes() + scores.bytes() + block_err.bytes() + err_hist.bytes() +
           v.bytes();
  }
  // task cursors: k_pr_cb's ranges, then pass B's (the finish kernel resets them all)
  uint32_t task_ranges() const { return grid_cb + grid_vb; }
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
// The largest node count + 1 a JACOBI PageRank takes.  Its layout build sorts the n rows and scans n + 1
// counts with CUB in single passes of int-sized counts, and needs about 24 bytes per node for the order sort
// alone, so node counts of 2^31 - 1 and more are refused rather than widened.
constexpr uint32_t PR_MAX_NODES = 0x7FFFFFFFu;
// GB_OK when n < PR_MAX_NODES, else GB_ERR_INVALID with the one message every PageRank entry point gives.
// check_pr_host_csr checks it first, so the host-CSR calls (one-shot, shard and communicator) refuse before
// they upload or copy any offsets; layout_begin checks it for the twin's paths (gb_page_rank, the shards of
// gb_pr_shard_create), before the plan's first allocation.  Either way the caller's scores stay unwritten.
gb_status require_pr_node_count(uint32_t n);
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

// ---- the rules every PageRank call keeps (pagerank.cu) -----------------------------------------------------
// GB_ERR_INVALID for a config that cannot stop: max_iterations == 0 (no sweep limit) with tolerance <= 0
gb_status require_pr_config(const gb_page_rank_config* cfg);
// max_iterations == 0 never satisfies `iteration == max_iterations` (page_rank.rs:107): the
// reference then runs until the tolerance is met; we bound that at 100000 sweeps.
uint64_t pr_sweep_limit(const gb_page_rank_config* cfg);
// gb_page_rank / gb_page_rank_device: the ranks of g into d_scores (device) or h_scores (host), whichever is
// given.  A g->pr_plan the caller has put there is used as it is; otherwise JACOBI builds it from g's in-CSR.
gb_status page_rank_impl(const gb_graph* g, const gb_page_rank_config* cfg, float* d_scores, float* h_scores,
                         uint64_t* ran, double* error);

// a shard of the sweep API that owns `plan` (pagerank.cu); takes the plan, whatever it returns
gb_status shard_from_plan(int device, PrPlan* plan, gb_pr_shard** out);
// The shards of one call, freed together
struct ShardSet {
  std::vector<gb_pr_shard*> v;
  explicit ShardSet(uint32_t count) : v(count, nullptr) {}
  void clear() {
    for (gb_pr_shard* sh : v)
      if (sh) gb_pr_shard_free(sh);
    v.clear();
  }
  ~ShardSet() { clear(); }
};

// ---- PageRank from a host CSR (pr_csr.cu) ------------------------------------------------------------------
// The O(1) host checks of a host PageRank CSR (n + 1 in- and out-offsets, the in-targets), in the order and
// with the messages of every entry point that takes one
gb_status check_pr_host_csr(uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt, const uint32_t* out_off);
// The layouts of ranks 0 .. U-1 (U = devs.size() * V, rank r on devs[r / V]) of a host CSR that passed
// check_pr_host_csr.  Part u of the split (pr_split, targets in chunks of about chunk_edges >= 1
// edges) is uploaded by the device of rank u; the offsets are checked on the device.  A lone rank builds its
// layout from its part as the chunks land; with several, every rank gathers the rows it owns from all parts into
// a local in-CSR first.  On success plans holds U plans, the caller's to free; on failure nothing is left.
gb_status pr_csr_plans(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                       const uint32_t* in_tgt, const uint32_t* out_off, uint64_t chunk_edges,
                       std::vector<PrPlan*>* plans);
// check_pr_host_csr, then the plans of pr_csr_plans (chunks of GB_PR_PART_CHUNK_EDGES edges) as the shards of
// ranks 0 .. U-1 of the sweep API: shards (U entries) are the caller's to free.
gb_status pr_csr_shards(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                        const uint32_t* in_tgt, const uint32_t* out_off, std::vector<gb_pr_shard*>& shards);

// launch shapes of the sweep kernels, their error buffers and k_pr_cb's shared-memory size (pagerank.cu).
// h_nrows / h_poff: the staircase (nrows[], poff[]) as the layout build holds it on the host.
gb_status plan_sweep_shape(PrPlan* p, const std::vector<uint32_t>& h_nrows, const std::vector<uint32_t>& h_poff,
                           int dev_sms, cudaStream_t s);
// The largest window of V pass B can take on `device` (a multiple of VB_ALIGN slots): its shared-memory block,
// the zero slot and k_pr_cb's static shared memory within the per-block opt-in limit, and below 0xFFFF, since
// pass B's ids and pad id are 16-bit (58048 slots on an H100).
// GB_PR_VB_WINDOW (tests): a smaller window, in slots.
gb_status pr_vb_window(int device, uint32_t* window);

}  // namespace gb
