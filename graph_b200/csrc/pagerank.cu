// pagerank.cu — PageRank over the device in-CSR.
//
// Replaces crates/algos/src/page_rank.rs:58-168 (`page_rank`, `page_rank_iteration`).
//
// Two schedules (gb_pr_mode, include/graph_b200.h):
//   EXACT  — the reference's sweep as one thread executes it: in place, CSR-order f32 sums, separate
//            multiply/add (no FMA), IEEE division.  One warp walks the vertices in id order; lanes
//            only parallelise the gather loads, the additions stay sequential.  Bit-exact with the
//            reference wherever the reference is deterministic (n <= 16384 = one chunk).
//   JACOBI — the throughput path (double-buffered, deterministic).
//
// JACOBI design.  A pull sweep issues one 4-byte gather per edge, and divergent gathers that miss L1
// are limited by the L1TEX->XBAR request rate (profiles/microbench/gather_ceiling.cu), whatever the
// layout of the index stream, far below the HBM roofline.  Shared memory serves several random 4-byte
// reads per clock.  So the sweep is COLUMN
// BLOCKED: vertices are renumbered by in-degree descending, then out-degree descending (hot sources
// first); the source vector is cut into blocks of B entries that fit in shared memory, and every
// (row, block) pair that is expected to hold at least tau edges gets a SEGMENT of 16-bit block-local
// source ids in that block's stream.  A persistent CTA brings a block into shared memory with TMA bulk
// copies (cp.async.bulk + mbarrier), then its warps stream the segments (coalesced 128-bit loads, 8 ids per lane), gather from
// shared memory, and reduce lanes that belong to the same row with a segmented warp scan; one f32
// partial per (row, block) pair goes back to HBM.  Edges of pairs below the threshold (and all edges
// of short rows) stay in a SELL-32 layout with 32-bit ids: one lane per row, gathers through L1/L2
// (no shared memory: the whole L1 / shared-memory array serves as L1); that kernel also completes every row whose
// segments lie in at most 4 blocks.  A finish kernel adds the hub rows' partials in a fixed order
// (f64), applies the update of page_rank.rs:148-158 and reduces the sweep error.
// Everything is deterministic: bit-identical run to run for a given shard count; across shard counts the
// ranks agree to ~2e-7 (DESIGN.md §2).
//
// Multi-GPU (1-D edge-cut by destination): the 32-row slices of the internal order are dealt
// round-robin to the P ranks, so every rank holds the same mix of hub and tail rows; a rank builds the
// layout of its own rows only and stores each finished out_score into every peer's next vector
// (multimem.st through the NVSwitch when a multicast mapping is given, else one store per peer).
// The shard API at the end of this file is one rank's side of that; multi.cu drives the ranks of one process,
// and pr_csr.cu builds layouts and shards straight from a host CSR.
//
// Algorithmic bytes per sweep: 4m (targets) + 4(n+1) (offsets) + 5*4n (out_scores read+write,
// scores read+write, out-degree read) = 4m + 24n + 4  (BASELINE.md §3).
#include <algorithm>
#include <cmath>

#include "pr_plan.cuh"

namespace gb {

void free_pr_plan(PrPlan* p) {
  if (!p) return;
  if (p->trace && p->trace_events.size() >= 5) {
    cudaDeviceSynchronize();
    double acc[4] = {0, 0, 0, 0};
    const size_t sweeps = p->trace_events.size() / 5;
    for (size_t i = 0; i < sweeps; ++i)
      for (int k = 0; k < 4; ++k) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, p->trace_events[5 * i + k], p->trace_events[5 * i + k + 1]);
        acc[k] += ms;
      }
    if (p->vb)  // nothing runs between the fused k_pr_cb and pass B
      fprintf(stderr, "[gb trace] shard %u/%u, %zu sweeps: k_pr_cb with pass A %.4f  pass B %.4f  k_pr_finish %.4f ms\n",
              p->deal.p, p->deal.P, sweeps, acc[0] / sweeps, acc[2] / sweeps, acc[3] / sweeps);
    else
      fprintf(stderr, "[gb trace] shard %u/%u, %zu sweeps: k_pr_cb %.4f  k_pr_fixup %.4f  k_pr_sell %.4f  k_pr_finish %.4f ms\n",
              p->deal.p, p->deal.P, sweeps, acc[0] / sweeps, acc[1] / sweeps, acc[2] / sweeps, acc[3] / sweeps);
  }
  for (cudaEvent_t e : p->trace_events) cudaEventDestroy(e);
  for (cudaEvent_t e : p->prof_events) cudaEventDestroy(e);
  delete p;
}
uint64_t pr_plan_bytes(const PrPlan* p) { return p ? p->bytes() : 0; }

// ---- small device helpers --------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_stream_u4(const uint32_t* p) {
  uint4 r;  // streamed once per sweep: keep it out of L1 so the gathered vector stays there
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_stream_u2(const uint2* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
// a fused task of k_pr_cb<CB_FUSED>, read afresh wherever it is needed (an L1 hit): a coherent load in volatile
// asm, so that the compiler cannot merge the reads into one value that would live (and spill) across the walks
__device__ __forceinline__ uint4 ld_task(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}

// ---- sweep kernels (JACOBI) ------------------------------------------------------------------
// What k_pr_cb's task scheduler reads: the block of each rank, the tasks and this pass's task cursors
struct CbSched {
  const uint32_t* blk;  // CbStream::blk (CB_FUSED: unused, its tasks name their source block)
  const uint2* tasks;
  uint32_t n_tasks;     // CB_FUSED: PrVBlocks::n_tasks (the tasks are PrArgs::fused_tasks)
  uint32_t* task_ctr;
};
// What the walker, the fixup of cut segments and k_pr_finish read of a stream (CbStream)
struct CbWalk {
  const uint32_t* nrows;
  const uint32_t* poff;
  const uint2* ids;
  const uint32_t* bits;
  float* partial;
  const uint4* chunks;
  uint32_t n_chunks;
  const uint32_t* tail_slot;
  double* side;
  const uint32_t* fix_list;
  uint32_t n_fix;
};
struct PrArgs {
  const uint32_t* outdeg;
  const float* x_cur;
  float* x_next;
  float* mc_next;       // multicast mapping of x_next on every rank (NULL: unicast peer stores)
  float* peer_next[7];  // peer-mapped copies of x_next (fused allgather over NVLink); n_peers used
  uint32_t n_peers;
  uint32_t n;
  float* scores;
  PrDeal deal;
  uint32_t n_loc, n_cb;
  uint32_t n_fin_warp;  // rows [0, n_fin_warp) own segments in many blocks (finish: one CTA per 32 rows)
  uint32_t fin_hub_ctas;  // finish: CTAs [0, fin_hub_ctas) take those groups, the rest the other rows
  uint32_t n_fin;       // rows [0, n_fin) are completed by k_pr_finish (rem[] + partials); rows [n_fin, n_cb) own
                        // segments in at most SELL_FEW blocks and are completed by their k_pr_sell lane
  uint32_t few_kb, few_nrows[SELL_FEW], few_poff[SELL_FEW];  // the first blocks' row prefixes / partial offsets
  uint32_t fix_in_sell; // k_pr_sell adds the parts of cut segments first (PrPlan::fix_at == PrFix::SELL)
  const uint32_t* fin_kb;  // [ceil(n_cb / 32)] blocks in which the first row of each 32-row group owns a segment
  // column blocks: the stream a k_pr_cb pass walks, or the hot blocks' (k_pr_fixup, k_pr_sell, k_pr_finish)
  uint32_t B;
  CbSched sched;
  CbWalk walk;
  CbWalk fix;              // pass B: the hot blocks' stream, whose cut segments its first warps add (PrFix::PASS_B)
  uint32_t n_task_ranges;  // all passes' task cursors, from sched.task_ctr of the hot blocks
  float* rem;
  // pass A of the virtual blocks (k_pr_cb<CB_FUSED>)
  const uint4* fused_tasks;  // PrVBlocks::tasks
  float* vals;
  const uint16_t* bin_ids;
  const uint32_t* bin_bits;
  const uint32_t* bin_grun;
  const uint32_t* bin_runs;
  const uint2* bin_chunks;
  uint32_t bin_fill;    // runs start on 32-byte sectors of V: zero each run's pad slots (PrVBlocks::sectors)
  // SELL rows
  const uint4* sell;
  const uint2* slice_meta;
  uint32_t num_slices;
  // error / stop rule
  double* block_err;
  double* err_hist;
  uint32_t* ctrl;
  uint32_t err_base_fin;  // block_err slots [0, err_base_fin) belong to the SELL CTAs
  float base, damping;
  double tolerance;
  double extra_err;   // closed-form error of the skipped zero-in-degree rows (first sweep only)
  uint32_t sweep;     // index inside the current batch
  uint32_t sweep_no;  // 1-based global sweep number
};

// 8 gathers per lane in straight-line predicated code (padding id ~0 reads nothing): per-target if/else
// makes every load wait for a scoreboard slot of the previous one, and every pending miss holds an L1
// line — so this kernel uses NO shared memory at all and leaves the whole L1 / shared-memory array to L1
// (a 128 KB shared-memory mirror of the hottest sources was slower than two mirror-less CTAs per SM).
__device__ __forceinline__ void pr_gather(const float* x, const uint4& ta, const uint4& tb, float (&v)[8]) {
  const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.u32 p, %1, 0xffffffff;\n\t"
        "mov.f32 %0, 0f00000000;\n\t"
        "@p ld.global.nc.f32 %0, [%2];\n\t}"
        : "=f"(v[j])
        : "r"(t[j]), "l"(x + t[j]));
  }
}
__device__ __forceinline__ float pr_sum8(const float (&v)[8]) {
  return ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
}
__device__ __forceinline__ uint4 pr_ld4(const uint4* p) { return ld_stream_u4(reinterpret_cast<const uint32_t*>(p)); }

// the per-vertex update of page_rank.rs:148-158 with the reference's rounding sequence; gr = global row
template <bool PEERS>
__device__ __forceinline__ double pr_update(uint32_t gr, float sum, float old, uint32_t deg, const PrArgs& a) {
  const float nw = __fadd_rn(a.base, __fmul_rn(a.damping, sum));
  a.scores[gr] = nw;
  const float xo = __fdiv_rn(nw, (float)deg);
  if (PEERS && a.mc_next) {
    // one store, replicated by the NVSwitch into every rank's next vector (this rank's included)
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(a.mc_next + gr), "f"(xo) : "memory");
  } else {
    a.x_next[gr] = xo;
    if (PEERS)
      for (uint32_t p = 0; p < a.n_peers; ++p) a.peer_next[p][gr] = xo;
  }
  return fabs((double)__fsub_rn(nw, old));
}

// ---- column blocks ------------------------------------------------------------------------------------
// One warp, one chunk: groups [g0, g1) of block j's stream, in steps of 32 G groups from the even-aligned
// g0 & ~1 (G = cb_step_groups: 4, or 2 in the short chunks of thin blocks so that their lanes do not idle).
// Lane L owns the ADJACENT positions G L .. G L + G - 1 of the step (G / 2 128-bit loads) and adds the
// runs inside the lane in f32; across lanes the value of the run that is open at the end of each lane goes
// through ONE segmented inclusive scan (5 shuffles, one ballot and one read of the start bits per step); a
// run that spans steps is carried in f64.  The row of a group follows from counting segment-start bits.
// A lane ends at most G runs per step: one at each position followed by a segment start, and the one open
// at its end.
// SPECIAL = the chunk starts or ends inside a segment (rare: segments longer than a chunk); the common
// instantiation carries none of the side-buffer logic.
template <bool SPECIAL>
__device__ __forceinline__ void cb_emit(const PrArgs& a, uint32_t c, bool is_end, uint32_t q, uint32_t last,
                                        bool run_continues, bool last_step, bool tail_cont, bool in_head,
                                        uint32_t cum, uint32_t slot0, double tot) {
  if (!is_end) return;
  if (SPECIAL) {
    if (q == last && run_continues && !last_step) return;  // carried into the next step
    if (in_head && cum == 0) a.walk.side[2 * (size_t)c] = tot;                        // tail part of a cut segment
    else if (q == last && last_step && tail_cont) a.walk.side[2 * (size_t)c + 1] = tot;  // head part of one
    else a.walk.partial[slot0 + cum] = (float)tot;
  } else {
    if (q == last && run_continues) return;  // carried into the next step
    a.walk.partial[slot0 + cum] = (float)tot;
  }
}
// A lane's k-th load of a step.  With one load per lane (G = 2) the ids are streamed past L1, so that
// the gathered vector stays there; with two (G = 4) the second load reads the other half of the sectors
// of the first one, so they are kept in L1.
template <uint32_t G>
__device__ __forceinline__ uint4 cb_ld_ids(const uint4* p) {
  if constexpr (G == 2) {
    return ld_stream_u4(reinterpret_cast<const uint32_t*>(p));
  } else {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
  }
}
__device__ __forceinline__ float cb_group_sum(const float* xs, uint32_t lo, uint32_t hi) {
  return xs[lo & 0xFFFFu] + xs[lo >> 16] + (xs[hi & 0xFFFFu] + xs[hi >> 16]);
}
template <uint32_t G, bool SPECIAL>
__device__ __forceinline__ void cb_walk(const PrArgs& a, const float* xs, uint32_t c, const uint4 ch, uint32_t lane,
                                        uint32_t pad2) {
  constexpr uint32_t NL = G / 2;    // 128-bit loads and 64-bit start-bit words per lane and step
  constexpr uint32_t STEP = 32 * G;  // groups per step
  const uint32_t g0 = ch.x, g1 = ch.y;
  const uint32_t j = ch.w & 0xFFFFFFu, fl = ch.w >> 24;
  const bool head_cont = SPECIAL && (fl & CB_HEAD_CONT), tail_cont = SPECIAL && (fl & CB_TAIL_CONT);
  uint32_t slot0 = a.walk.poff[j] + ch.z;  // staircase slot of the row "before" the first segment start
  bool in_head = head_cont;
  double carry = 0.0;
  const uint32_t le_mask = 0xFFFFFFFFu >> (31u - lane);
  const uint32_t q0 = G * lane;  // the lane's first position in the step
  const uint4* ids16 = reinterpret_cast<const uint4*>(a.walk.ids) + NL * lane;  // pairs of groups
  const uint4 padv = make_uint4(pad2, pad2, pad2, pad2);
  const auto load = [&](uint4(&d)[NL], uint32_t gs) {  // the lane's pairs of the step at gs that start below g1
#pragma unroll
    for (uint32_t k = 0; k < NL; ++k) d[k] = gs + q0 + 2 * k < g1 ? cb_ld_ids<G>(ids16 + (gs >> 1) + k) : padv;
  };
  uint4 ids[NL], nids[NL];
  load(ids, g0 & ~1u);
  for (uint32_t gs = g0 & ~1u; gs < g1; gs += STEP) {
    load(nids, gs + STEP);
    // groups outside [g0, g1) belong to the neighbouring chunks: only position 0 can lie before g0, and the
    // loads above already left out the pairs that start past g1
    if (gs + q0 < g0) ids[0].x = ids[0].y = pad2;
#pragma unroll
    for (uint32_t k = 0; k < NL; ++k)
      if (gs + q0 + 2 * k + 1 >= g1) ids[k].z = ids[k].w = pad2;
    const uint32_t wi = gs >> 5, sh = gs & 31u;
    uint32_t w[G + 1];
#pragma unroll
    for (uint32_t k = 0; k <= G; ++k) w[k] = __ldg(a.walk.bits + wi + k);
    const uint32_t nvalid = min(STEP, g1 - gs);
    unsigned long long W[NL];  // segment starts at the step's positions 64 k .. 64 k + 63, inside [g0, g1)
#pragma unroll
    for (uint32_t k = 0; k < NL; ++k) {
      W[k] = ((unsigned long long)__funnelshift_r(w[2 * k + 1], w[2 * k + 2], sh) << 32) |
             __funnelshift_r(w[2 * k], w[2 * k + 1], sh);
      if (nvalid < 64 * k + 64) W[k] = k == 0 || nvalid > 64 * k ? W[k] & ((1ull << (nvalid - 64 * k)) - 1ull) : 0ull;
    }
    if (gs < g0) W[0] &= ~1ull;
    const uint32_t last = nvalid - 1;
    const bool last_step = gs + STEP >= g1;
    // does the run of the last valid group go on after this step (inside the chunk / past its end)?
    const bool run_continues = last_step ? tail_cont : !((w[G] >> sh) & 1u);
    // the word of the lane's positions, the word of the position after them, and the starts before them
    const uint32_t s = q0 & 63u, e = q0 + G;
    unsigned long long Wm = W[0], We = W[0];
    uint32_t pre = 0;
#pragma unroll
    for (uint32_t k = 1; k < NL; ++k) {
      if (q0 >= 64 * k) {
        pre += __popcll(W[k - 1]);
        Wm = W[k];
      }
      if (e >= 64 * k) We = W[k];
    }
    pre += __popcll(Wm & ((1ull << s) - 1ull));
    const uint32_t F = (uint32_t)(Wm >> s) & ((1u << G) - 1u);  // segment starts at the lane's G positions
    const bool nxt = lane < 31 && ((We >> (e & 63u)) & 1ull);   // and at the position after them
    float v[G], r[G];  // group sums; runs inside the lane (restarted at every start)
#pragma unroll
    for (uint32_t i = 0; i < G; ++i) v[i] = i & 1 ? cb_group_sum(xs, ids[i / 2].z, ids[i / 2].w)
                                                  : cb_group_sum(xs, ids[i / 2].x, ids[i / 2].y);
    r[0] = v[0];
#pragma unroll
    for (uint32_t i = 1; i < G; ++i) r[i] = (F >> i) & 1u ? v[i] : r[i - 1] + v[i];
    float incl = r[G - 1];  // this lane's share of the run open at its end
    const uint32_t below = __ballot_sync(0xFFFFFFFFu, F != 0) & le_mask;
    const int seg_start = below ? 31 - __clz(below) : -1;
    const int lo = seg_start < 0 ? 0 : seg_start;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const float t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if ((int)lane - d >= lo) incl += t;
    }
    const double incl_d = (double)incl + (seg_start < 0 ? carry : 0.0);
    double x_in = __shfl_up_sync(0xFFFFFFFFu, incl_d, 1);  // the run open at the end of the previous lane
    if (lane == 0) x_in = carry;
#pragma unroll
    for (uint32_t i = 0; i < G; ++i) {
      const uint32_t q = q0 + i, Fi = F & ((2u << i) - 1u);  // segment starts at the lane's positions <= q
      const bool valid = q <= last && (i > 0 || gs + q0 >= g0);
      const bool ends = i + 1 < G ? ((F >> (i + 1)) & 1u) != 0 : nxt;
      cb_emit<SPECIAL>(a, c, valid && (q == last || ends), q, last, run_continues, last_step, tail_cont, in_head,
                       pre + __popc(Fi), slot0, i + 1 < G ? (double)r[i] + (Fi ? 0.0 : x_in) : incl_d);
    }
    const double tl = __shfl_sync(0xFFFFFFFFu, incl_d, 31);
    carry = (run_continues && !last_step) ? tl : 0.0;
    unsigned long long any = 0;
#pragma unroll
    for (uint32_t k = 0; k < NL; ++k) {
      any |= W[k];
      slot0 += __popcll(W[k]);
      ids[k] = nids[k];
    }
    if (SPECIAL && any) in_head = false;
  }
}
__device__ __forceinline__ void cb_chunk(const PrArgs& a, const float* xs, uint32_t c, uint32_t lane, uint32_t pad2) {
  const uint4 ch = a.walk.chunks[c];
  if (ch.x >= ch.y) return;
  const bool special = (ch.w >> 24) & (CB_HEAD_CONT | CB_TAIL_CONT);
  if (cb_step_groups(ch.x, ch.y) == 4) {
    if (special) cb_walk<4, true>(a, xs, c, ch, lane, pad2);
    else cb_walk<4, false>(a, xs, c, ch, lane, pad2);
  } else {
    if (special) cb_walk<2, true>(a, xs, c, ch, lane, pad2);
    else cb_walk<2, false>(a, xs, c, ch, lane, pad2);
  }
}

// V[slot] = xs[sid] unless sid is BIN_PAD, predicated: a branch per position would split the warp's stores
__device__ __forceinline__ void bin_store(float* v, uint32_t xs_smem, uint32_t sid) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .f32 x;\n\t"
      "setp.ne.u32 p, %0, %3;\n\t"
      "mov.f32 x, 0f00000000;\n\t"
      "@p ld.shared.f32 x, [%1];\n\t"
      "@p st.global.f32 [%2], x;\n\t}" ::"r"(sid),
      "r"(xs_smem + 4 * sid), "l"(v), "n"((uint32_t)BIN_PAD)
      : "memory");
}
// V[e .. e rounded up to VB_RUN_ALIGN) = 0: the pad slots after a run, with at most one 4-, one 8- and one 16-byte
// store, so that the run's last 32-byte sector is written whole in the step that stores the run's last value
__device__ __forceinline__ void bin_fill_pad(float* v, uint32_t e) {
  if (e & 1u) v[e++] = 0.0f;
  if (e & 2u) {
    *reinterpret_cast<float2*>(v + e) = make_float2(0.0f, 0.0f);
    e += 2;
  }
  if (e & 4u) *reinterpret_cast<float4*>(v + e) = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}
// Pass A of the virtual blocks, one warp per chunk of steps of one source block.  In a step of BIN_STEP positions
// lane L stores the values of positions 32 k + L (k < 8) to their slots of V: slot = position + delta of the
// position's run.  A run's slots are consecutive, so each of the 8 stores of a step is coalesced.  A step lies in
// one block's share, so its runs are consecutive from r0, the first run of its first group, and the run of a
// position is r0 plus the run starts after the step's first position up to it.  Lane L holds the delta of run
// r0 + L and every lane takes the delta of its run from there by shuffle; a step with more than 32 runs loops over
// 32-run windows instead.  The loads run ahead of the stores, so that no load waits on another one in the steady
// state: while step s stores, the ids and start bits of step s + 1 are in flight, and so are its deltas, from its
// r0, which was loaded during step s - 1.
// FILL (sector-aligned runs): the lane of a run's last position also zeroes the run's pad slots.  A run ends where
// the next position starts a run (nbit: the first position of the next step) or is a pad; the pads of a step
// follow its valid positions, so the step's last valid position is where they begin.
template <bool WIDE, bool FILL>
__device__ __forceinline__ void bin_step(const PrArgs& a, uint32_t xs_smem, uint32_t p0, uint32_t lane, const uint4 id,
                                         const uint4 b0, const uint4 b1, uint32_t nbit, uint32_t r0, uint32_t d,
                                         uint32_t runs) {
  const uint32_t bits[9] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, nbit};
  const uint32_t w[4] = {id.x, id.y, id.z, id.w};
  const uint32_t upto = 0xFFFFFFFFu >> (31u - lane);  // positions 0 .. lane of a group
  uint32_t before = 0u - (bits[0] & 1u);  // run starts after the step's first position, before group k
  uint32_t nvalid = 0;                    // FILL: the step's positions that hold a pair
  if (FILL) {
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k)
      nvalid += __popc(__ballot_sync(0xFFFFFFFFu, ((w[k / 2] >> (16 * (k & 1))) & 0xFFFFu) != BIN_PAD));
  }
#pragma unroll
  for (uint32_t k = 0; k < 8; ++k) {
    const uint32_t r = before + __popc(bits[k] & upto);  // the position's run - r0
    before += __popc(bits[k]);
    uint32_t dk;
    if (!WIDE) {
      dk = __shfl_sync(0xFFFFFFFFu, d, r);
    } else {
      // a window of 32 runs at a time, the first one in d
      dk = __shfl_sync(0xFFFFFFFFu, d, r & 31u);
#pragma unroll 1
      for (uint32_t w0 = 32; w0 <= runs; w0 += 32) {
        const uint32_t t = __shfl_sync(0xFFFFFFFFu, __ldg(a.bin_runs + r0 + w0 + lane), (r - w0) & 31u);
        if (r - w0 < 32) dk = t;
      }
    }
    const uint32_t sid = (w[k / 2] >> (16 * (k & 1))) & 0xFFFFu;
    bin_store(a.vals + (p0 + 32 * k + dk), xs_smem, sid);
    if (FILL) {
      const uint32_t q = 32 * k + lane;  // the position in the step
      const bool last = sid != BIN_PAD && (((__funnelshift_rc(bits[k], bits[k + 1], lane + 1) & 1u) != 0) ||
                                           (q + 1 == nvalid && nvalid < BIN_STEP));
      if (last) bin_fill_pad(a.vals, p0 + 32 * k + dk + 1);
    }
  }
}
template <bool FILL>
__device__ __forceinline__ void bin_chunk(const PrArgs& a, const float* xs, uint32_t c, uint32_t lane) {
  constexpr uint32_t GS = BIN_STEP / 32;  // groups per step
  const uint2 ch = a.bin_chunks[c];       // steps [ch.x, ch.y)
  const uint32_t* ids = reinterpret_cast<const uint32_t*>(a.bin_ids) + 4 * lane;  // 128 words per step
  const uint4* bits4 = reinterpret_cast<const uint4*>(a.bin_bits);               // 2 per step
  const uint32_t xs_smem = (uint32_t)__cvta_generic_to_shared(xs);
  uint4 id = ld_stream_u4(ids + 128 * (size_t)ch.x);
  uint4 b0 = __ldg(bits4 + 2 * ch.x), b1 = __ldg(bits4 + 2 * ch.x + 1);
  uint32_t r0 = __ldg(a.bin_grun + GS * ch.x);
  uint32_t r0n = ch.x + 1 < ch.y ? __ldg(a.bin_grun + GS * (ch.x + 1)) : 0u;
  uint32_t d = __ldg(a.bin_runs + r0 + lane);
  for (uint32_t s = ch.x; s < ch.y; ++s) {
    uint4 nid = id, nb0 = b0, nb1 = b1;
    uint32_t nd = d, r0nn = r0n;
    if (s + 1 < ch.y) {
      nid = ld_stream_u4(ids + 128 * (size_t)(s + 1));
      nb0 = __ldg(bits4 + 2 * (s + 1));
      nb1 = __ldg(bits4 + 2 * (s + 1) + 1);
      nd = __ldg(a.bin_runs + r0n + lane);
      if (s + 2 < ch.y) r0nn = __ldg(a.bin_grun + GS * (s + 2));
    }
    // FILL: the start bits of the next step's first 32 positions (past the last step: a run start)
    const uint32_t nbit = !FILL ? 0u : s + 1 < ch.y ? nb0.x : __ldg(a.bin_bits + 8 * (s + 1));
    // runs of the step after its first one: the run starts after its first position
    const uint32_t runs = __popc(b0.x & ~1u) + __popc(b0.y) + __popc(b0.z) + __popc(b0.w) + __popc(b1.x) +
                          __popc(b1.y) + __popc(b1.z) + __popc(b1.w);
    if (runs < 32) bin_step<false, FILL>(a, xs_smem, s * BIN_STEP + lane, lane, id, b0, b1, nbit, r0, d, runs);
    else bin_step<true, FILL>(a, xs_smem, s * BIN_STEP + lane, lane, id, b0, b1, nbit, r0, d, runs);
    id = nid, b0 = nb0, b1 = nb1, d = nd, r0 = r0n, r0n = r0nn;
  }
}

// Segments cut by chunk boundaries (segments longer than a chunk): one warp per segment adds its parts
// in a fixed order — the head part of the first chunk, then lanes over the following chunks (a fixed
// xor tree per batch of 32).  Tiny; runs after k_pr_cb (as k_pr_fixup, or as the prologue of k_pr_sell or of
// pass B).  w = the hot blocks' stream.
__device__ __forceinline__ void cb_fix_segment(const CbWalk& w, uint32_t c0, uint32_t lane) {
  double t = w.side[2 * (size_t)c0 + 1];
  for (uint32_t k0 = c0 + 1;; k0 += 32) {
    const uint32_t k = k0 + lane;
    // the walk ends at the first chunk that is not entirely inside the segment (sentinel chunk after the last)
    const uint32_t fl = w.chunks[min(k, w.n_chunks)].w >> 24;
    const bool inside = k < w.n_chunks && (fl & CB_INTERIOR) && (fl & CB_TAIL_CONT);
    const uint32_t stop = __ballot_sync(0xFFFFFFFFu, !inside);
    const uint32_t upto = stop ? (uint32_t)__ffs(stop) - 1 : 31u;  // last lane that contributes
    t += warp_sum(lane <= upto ? w.side[2 * (size_t)k] : 0.0);
    if (stop) break;
  }
  if (lane == 0) w.partial[w.tail_slot[c0]] = (float)t;
}

// ---- TMA bulk copy of a source block into shared memory (cp.async.bulk + mbarrier) -----------------
// One thread asks the copy engine for the block's 192 KB and every thread waits on the mbarrier's phase:
// no load/store instruction of the CTA is spent on the transfer and it runs at the SM's L2 bandwidth
// (the LDG.128 -> STS.128 loop it replaces kept one 16 KB wave in flight: 12 round trips per block).
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(arrivals) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(mbar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(mbar)
               : "memory");
}

// Persistent CTAs pull TASKS (32 consecutive chunks of one block).  The task list (fattest blocks first)
// is split into one contiguous RANGE per CTA, each with its own atomic cursor: a CTA first drains its own
// range — consecutive tasks of one block, so the 192 KB block is loaded once, not once per task — and then
// steals from the other ranges' cursors.  Self-balancing whatever else shares the SM and however uneven the
// thin blocks are (a purely static split leaves thin blocks at single-warp latency, one global cursor reloads the
// block for every task).  Claiming the next task one task ahead (to hide the atomic's
// round trip) was measured and dropped: a claimed task cannot be stolen, which costs more at the tail.
// KIND: CB_MAIN = the column blocks of x_cur; CB_FUSED = the same, with pass A of the virtual blocks: a task
// holds a source block's hot chunks and its pass-A chunks (PrVBlocks::tasks), interleaved so that the warps of a
// CTA stream ids through cb_chunk and scatter values through bin_chunk at the same time, from one load of the
// block; CB_VIRT = pass B (block j is V[blk[j] .. blk[j + 1]), the column-block walker as in CB_MAIN; its first
// warps add the cut segments of the hot blocks, which CB_FUSED has finished).
constexpr uint32_t CB_MAIN = 0, CB_VIRT = 1, CB_FUSED = 2;

// the next task of a CTA that drains range r (whole warp): from r's cursor, else from the first range after r that
// has tasks left, which becomes r.  CB_NONE when every range is drained.
__device__ __forceinline__ uint32_t cb_claim_task(const CbSched& s, uint32_t& r, uint32_t lane) {
  const uint32_t R = gridDim.x;  // ranges = CTAs
  for (;;) {
    const uint32_t lo = (uint32_t)((uint64_t)s.n_tasks * r / R), hi = (uint32_t)((uint64_t)s.n_tasks * (r + 1) / R);
    uint32_t k = CB_NONE;
    if (lane == 0) {
      k = lo + atomicAdd(s.task_ctr + r, 1u);
      if (k >= hi) k = CB_NONE;
    }
    const uint32_t t = __shfl_sync(0xFFFFFFFFu, k, 0);
    if (t != CB_NONE) return t;
    // this range is drained: the lanes probe the other ranges' cursors 32 at a time (plain loads)
    uint32_t found = CB_NONE;
    for (uint32_t base = 1; base < R && found == CB_NONE; base += 32) {
      uint32_t q = r + base + lane;
      if (q >= R) q -= R;
      bool ok = false;
      if (base + lane < R) {
        const uint32_t qlo = (uint32_t)((uint64_t)s.n_tasks * q / R), qhi = (uint32_t)((uint64_t)s.n_tasks * (q + 1) / R);
        ok = *((volatile uint32_t*)(s.task_ctr + q)) < qhi - qlo;
      }
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
      if (m) found = __shfl_sync(0xFFFFFFFFu, q, __ffs(m) - 1);
    }
    if (found == CB_NONE) return CB_NONE;  // every range is drained
    r = found;
  }
}
// the block of task t: a source block (CB_FUSED), else a block rank of the stream
template <uint32_t KIND>
__device__ __forceinline__ uint32_t cb_task_block(const PrArgs& a, uint32_t t) {
  return KIND == CB_FUSED ? ld_task(a.fused_tasks + t).w : a.sched.tasks[t].y >> 8;
}

// Inside a block the chunks of the CTA's tasks FLOW: s_flow = (task << 32 | next chunk) is the one cursor, and a
// warp claims a chunk with one shared atomicAdd, which gives it the task and the chunk's index in it together
// (CB_FUSED: hot, pass A, hot, .. while both kinds last, then the rest of the longer kind).  The warp that draws
// the last index, n - 1, of an n-chunk task claims the CTA's next task before it walks that chunk (cb_claim_task:
// only once the current task has no chunk left to hand out, so a claimed task is taken up by the next warp that
// finishes a chunk and is not withheld from stealing for longer; the claim's round trip overlaps the walk).  If
// that task is in the block in shared memory, the warp swaps it into s_flow with index 0 and the warps go on
// without waiting; otherwise it leaves the task in s_task and CB_NONE in s_flow, and every warp leaves the flow
// when it draws CB_NONE (the claiming warp after its chunk).  A warp that draws an index past n - 1 waits until
// s_flow names another task.  Ordering rules:
//  * a task and its chunk index come from one atomic on s_flow: no warp reads a task that is not published;
//  * s_range (the range being drained) is written by a claimer before its atomicExch on s_flow, behind a
//    __threadfence_block, and read by the next claimer after its atomicAdd, behind another: the claims are ordered;
//  * the block is replaced only between two __syncthreads, which a warp reaches only after it drew CB_NONE, i.e.
//    with no chunk of the block left; s_task is read after the first and s_flow is reset before the second.
template <uint32_t KIND>
__global__ void __launch_bounds__(PR_THREADS, 1) k_pr_cb(const PrArgs a) {
  extern __shared__ __align__(128) float smem[];
  float* xs = smem;  // B entries of x_cur + one zero slot (the pad id)
  __shared__ uint32_t s_task, s_range;
  __shared__ __align__(8) unsigned long long s_flow;
  __shared__ __align__(8) unsigned long long s_mbar;
  if (a.ctrl[0] != 0) return;  // tolerance already met by an earlier sweep of this batch
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (KIND == CB_VIRT)  // k_pr_cb<CB_FUSED> has finished (PrFix::PASS_B; n_fix = 0 otherwise)
    for (uint32_t i = blockIdx.x * PR_WARPS + warp; i < a.fix.n_fix; i += gridDim.x * PR_WARPS)
      cb_fix_segment(a.fix, a.fix.fix_list[i], lane);
  const uint32_t B = a.B;
  const uint32_t pad2 = B | (B << 16);
  const uint32_t mbar = (uint32_t)__cvta_generic_to_shared(&s_mbar);
  const uint32_t xs_smem = (uint32_t)__cvta_generic_to_shared(xs);
  const bool bulk_ok = (reinterpret_cast<uintptr_t>(a.x_cur) & 15u) == 0;  // cp.async.bulk moves 16-byte units
  uint32_t phase = 0;
  if (threadIdx.x == 0) mbar_init(mbar, 1);
  if (threadIdx.x < 4) xs[B + threadIdx.x] = 0.0f;  // the pad id's zero slot: never overwritten
  if (warp == 0) {
    uint32_t r = blockIdx.x;
    const uint32_t t = cb_claim_task(a.sched, r, lane);
    if (lane == 0) s_task = t, s_range = r;
  }
  for (;;) {
    __syncthreads();  // s_task is set, and every warp has left the flow of the previous block
    const uint32_t t0 = s_task;
    if (t0 == CB_NONE) break;
    const uint32_t j = cb_task_block<KIND>(a, t0);
    const uint64_t x0 = KIND == CB_VIRT    ? (uint64_t)a.sched.blk[j]
                        : KIND == CB_FUSED ? (uint64_t)j * B
                                           : (uint64_t)a.sched.blk[j] * B;
    const uint32_t cnt = KIND == CB_VIRT ? a.sched.blk[j + 1] - a.sched.blk[j]
                                         : (uint32_t)min((uint64_t)B, (uint64_t)a.n - x0);
    if (bulk_ok) {
      const uint32_t bulk = cnt & ~3u;
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the block's old contents were read through the generic proxy
        mbar_expect_tx(mbar, bulk * 4u);
        for (uint32_t off = 0; off < bulk; off += 4096u)  // 16 KB pieces
          bulk_g2s(xs_smem + off * 4u, a.x_cur + x0 + off, min(4096u, bulk - off) * 4u, mbar);
      }
      if (threadIdx.x >= 32 && threadIdx.x - 32 < cnt - bulk) xs[bulk + threadIdx.x - 32] = a.x_cur[x0 + bulk + threadIdx.x - 32];
      mbar_wait(mbar, phase);
      phase ^= 1u;
    } else {
      for (uint32_t i = threadIdx.x; i < cnt; i += PR_THREADS) xs[i] = a.x_cur[x0 + i];
    }
    if (threadIdx.x == 0) s_flow = (unsigned long long)t0 << 32;
    __syncthreads();
    // the flow of block j.  The task is read again for every chunk, so that none of it stays live across a walk
    // (the walkers use every register of the 64 that one 1024-thread CTA per SM leaves)
    for (;;) {
      unsigned long long f = 0;
      if (lane == 0) f = atomicAdd(&s_flow, 1ull);
      f = __shfl_sync(0xFFFFFFFFu, f, 0);
      const uint32_t t = (uint32_t)(f >> 32), k = (uint32_t)f;
      if (t == CB_NONE) break;
      // (first chunk, chunk count | block rank << 8); CB_FUSED: (first hot chunk, first pass-A chunk, hot chunks |
      // pass-A chunks << 8, source block)
      uint32_t n;
      if constexpr (KIND == CB_FUSED) {
        const uint32_t z = ld_task(a.fused_tasks + t).z;
        n = (z & 0xFFu) + (z >> 8);
      } else {
        n = a.sched.tasks[t].y & 0xFFu;
      }
      if (k >= max(n, 1u)) {  // past the task's chunks: wait until the claiming warp has swapped the next task in
        uint32_t cur = t;
        while (cur == t) {
          __nanosleep(64);
          if (lane == 0) cur = (uint32_t)(*(volatile unsigned long long*)&s_flow >> 32);
          cur = __shfl_sync(0xFFFFFFFFu, cur, 0);
        }
        continue;
      }
      bool leave = false;
      if (k + 1 == max(n, 1u)) {  // the task's last chunk: none is left to hand out, so claim the CTA's next task
        uint32_t r = 0;
        if (lane == 0) {
          __threadfence_block();
          r = *(volatile uint32_t*)&s_range;
        }
        r = __shfl_sync(0xFFFFFFFFu, r, 0);
        const uint32_t nt = cb_claim_task(a.sched, r, lane);
        leave = nt == CB_NONE || cb_task_block<KIND>(a, nt) != j;
        if (lane == 0) {
          *(volatile uint32_t*)&s_range = r;
          if (leave) s_task = nt;
          __threadfence_block();
          atomicExch(&s_flow, (unsigned long long)(leave ? CB_NONE : nt) << 32);
        }
      }
      if (k < n) {
        if constexpr (KIND == CB_FUSED) {
          const uint4 ft = ld_task(a.fused_tasks + t);
          const uint32_t n_hot = ft.z & 0xFFu, n_bin = ft.z >> 8, pairs = min(n_hot, n_bin);
          const bool hot = k < 2 * pairs ? (k & 1u) == 0 : n_hot > n_bin;
          const uint32_t i = k < 2 * pairs ? k >> 1 : k - pairs;
          if (hot) cb_chunk(a, xs, ft.x + i, lane, pad2);
          else if (a.bin_fill) bin_chunk<true>(a, xs, ft.y + i, lane);
          else bin_chunk<false>(a, xs, ft.y + i, lane);
        } else {
          cb_chunk(a, xs, a.sched.tasks[t].x + k, lane, pad2);
        }
      }
      if (leave) break;
    }
  }
}

__global__ void k_pr_fixup(const PrArgs a) {
  if (a.ctrl[0] != 0) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = gw; i < a.walk.n_fix; i += nw) cb_fix_segment(a.walk, a.walk.fix_list[i], lane);
}

// ---- SELL-32 sweep: one lane per row ------------------------------------------------------------
// A lane reads its row four targets at a time (128-bit, coalesced: the slice is stored group-major,
// lane-minor), gathers, and adds in row order.  The next slice's first targets and row metadata are
// requested while the current slice is processed.  Rows below n_cb only hold the edges that are not in
// a column-block segment: their sum goes to rem[] and the finish kernel completes them.
// The kernel needs no shared memory: two 512-thread CTAs per SM.
template <bool PEERS>
__global__ void __launch_bounds__(PR_SELL_THREADS, 2) k_pr_sell(const PrArgs a) {
  constexpr int NT = PR_SELL_THREADS;
  constexpr int NW = NT / 32;
  __shared__ double warp_err[NW];
  if (a.ctrl[0] != 0) return;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (a.fix_in_sell) {
    // segments cut by chunk boundaries (hub rows only: they are completed by k_pr_finish, after this kernel)
    const uint32_t gw0 = blockIdx.x * NW + warp, nw0 = gridDim.x * NW;
    for (uint32_t i = gw0; i < a.walk.n_fix; i += nw0) cb_fix_segment(a.walk, a.walk.fix_list[i], lane);
  }
  const float* __restrict__ x = a.x_cur;
  double err = 0.0;
  const uint32_t stride = gridDim.x * NW;
  const uint4 pad = make_uint4(~0u, ~0u, ~0u, ~0u);
  const uint32_t P = a.deal.P, pp = a.deal.p;
  // slices are dealt CTA-minor: the widest slices (the first ones) land on different SMs, not on the 16
  // warps of CTA 0 (an eighth-shard ran with its busiest SM 31 % above the average otherwise)
  uint32_t sidx = warp * gridDim.x + blockIdx.x;
  // pipeline state: metadata of this and the next slice, first two target groups + row data of this one
  uint2 meta = make_uint2(0, 0), nmeta = meta;
  uint4 ta = pad, tb = pad;
  float old = 0.0f;
  uint32_t deg = 1;
  if (sidx < a.num_slices) {
    meta = __ldg(a.slice_meta + sidx);
    if (sidx + stride < a.num_slices) nmeta = __ldg(a.slice_meta + sidx + stride);
    const uint4* base = a.sell + meta.x + lane;
    if (0 < meta.y) ta = pr_ld4(base);
    if (1 < meta.y) tb = pr_ld4(base + 32);
    const uint32_t l = 32 * sidx + lane;
    if (l >= a.n_fin && l < a.n_loc) {
      const uint32_t gr = deal_global(l, P, pp);
      old = a.scores[gr];
      deg = a.outdeg[gr];
    }
  }
  while (sidx < a.num_slices) {
    const uint32_t w4 = meta.y;
    const uint4* base = a.sell + meta.x + lane;
    const uint32_t l = 32 * sidx + lane;
    // next slice: first groups, row data; metadata of the slice after it
    const uint32_t nidx = sidx + stride;
    uint4 nta = pad, ntb = pad;
    float nold = 0.0f;
    uint32_t ndeg = 1;
    uint2 nnmeta = make_uint2(0, 0);
    if (nidx < a.num_slices) {
      const uint4* nbase = a.sell + nmeta.x + lane;
      if (0 < nmeta.y) nta = pr_ld4(nbase);
      if (1 < nmeta.y) ntb = pr_ld4(nbase + 32);
      const uint32_t nl = 32 * nidx + lane;
      if (nl >= a.n_fin && nl < a.n_loc) {
        const uint32_t ngr = deal_global(nl, P, pp);
        nold = a.scores[ngr];
        ndeg = a.outdeg[ngr];
      }
      if (nidx + stride < a.num_slices) nnmeta = __ldg(a.slice_meta + nidx + stride);
    }
    // a row with segments in at most SELL_FEW blocks is completed here: its partials (written by k_pr_cb,
    // which ran before) are requested now and added after the gathers, in block order like k_pr_finish
    float part[SELL_FEW];
#pragma unroll
    for (uint32_t j = 0; j < SELL_FEW; ++j) {
      part[j] = 0.0f;
      if (l >= a.n_fin && j < a.few_kb && l < a.few_nrows[j]) part[j] = a.walk.partial[(size_t)a.few_poff[j] + l];
    }
    float acc = 0.0f;
    for (uint32_t q = 0; q < w4; q += 2) {
      // targets of the next two groups are requested before this group's gathers are consumed
      const uint4 na = (q + 2 < w4) ? pr_ld4(base + (q + 2) * 32) : pad;
      const uint4 nb = (q + 3 < w4) ? pr_ld4(base + (q + 3) * 32) : pad;
      float v[8];
      pr_gather(x, ta, tb, v);
      acc += pr_sum8(v);
      ta = na;
      tb = nb;
    }
    if (l < a.n_fin) {
      a.rem[l] = acc;
    } else if (l < a.n_loc) {
      if (l < a.n_cb) {
        double sum = (double)acc;
#pragma unroll
        for (uint32_t j = 0; j < SELL_FEW; ++j)
          if (j < a.few_kb && l < a.few_nrows[j]) sum += (double)part[j];
        acc = (float)sum;
      }
      err += pr_update<PEERS>(deal_global(l, P, pp), acc, old, deg, a);
    }
    sidx = nidx;
    meta = nmeta;
    nmeta = nnmeta;
    ta = nta;
    tb = ntb;
    old = nold;
    deg = ndeg;
  }
  err = warp_sum(err);
  if (lane == 0) warp_err[warp] = err;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tt = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) tt += warp_err[w];
    a.block_err[blockIdx.x] = tt;
  }
}

// FIN_U = 32-row groups per warp iteration of the rows that are not hub groups: 2 (and 16 blocks' partials
// in flight) when every warp has a single iteration to do — the walk is a latency chain, fewer rounds win;
// 4 (4 blocks in flight) when the grid is capped and the kernel is throughput bound (RMAT-26 on one GPU).
template <bool PEERS, uint32_t FIN_U>
__global__ void __launch_bounds__(PR_FIN_THREADS) k_pr_finish(const PrArgs a) {
  constexpr int FIN_WARPS = PR_FIN_THREADS / 32;
  __shared__ double warp_err[FIN_WARPS];
  __shared__ bool is_last;
  if (a.ctrl[0] != 0) return;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double err = 0.0;
  const uint32_t P = a.deal.P, pp = a.deal.p;
  if (blockIdx.x == 0)  // next sweep's column-block task cursors
    for (uint32_t i = threadIdx.x; i < a.n_task_ranges; i += PR_FIN_THREADS) a.sched.task_ctr[i] = 0;
  // hub rows (segments in more than FIN_CTA_BLOCKS blocks): one CTA per 32-row group — lane = row,
  // warp w adds blocks w, w + 8, ... (independent coalesced loads), warp 0 adds the 8 sums in order
  __shared__ double part[FIN_WARPS][32];
  // fin_hub_ctas != 0: CTAs [0, fin_hub_ctas) take the hub groups, the others the remaining rows
  const bool split = a.fin_hub_ctas != 0;  // else every CTA does both parts
  const uint32_t H = split ? a.fin_hub_ctas : gridDim.x, T0 = split ? a.fin_hub_ctas : 0u;
  for (uint32_t g = blockIdx.x; blockIdx.x < H && g * 32 < a.n_fin_warp; g += H) {
    const uint32_t l = g * 32 + lane;
    const uint32_t kb = __ldg(a.fin_kb + g);  // blocks of the group's first row (it has the most)
    double s = 0.0;
#pragma unroll 8
    for (uint32_t j = warp; j < kb; j += FIN_WARPS)
      if (l < __ldg(a.walk.nrows + j)) s += (double)a.walk.partial[(size_t)__ldg(a.walk.poff + j) + l];
    part[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && l < a.n_fin) {
      double t = (double)a.rem[l];
#pragma unroll
      for (int w = 0; w < FIN_WARPS; ++w) t += part[w][lane];
      const uint32_t gr = deal_global(l, P, pp);
      err += pr_update<PEERS>(gr, (float)t, a.scores[gr], a.outdeg[gr], a);
    }
    __syncthreads();
  }
  // all other rows with segments: one lane per row, FIN_U consecutive 32-row groups per warp iteration,
  // 16 blocks' partials requested at a time (the walk is latency bound, not bandwidth bound: rounds count)
  const uint32_t tail_groups = (a.n_fin - a.n_fin_warp + 31) / 32;
  const uint32_t tw = (blockIdx.x - T0) * FIN_WARPS + warp, tnw = (gridDim.x - T0) * FIN_WARPS;
  for (uint32_t w = tw * FIN_U; blockIdx.x >= T0 && w < tail_groups; w += tnw * FIN_U) {
    const uint32_t l0 = a.n_fin_warp + 32 * w;
    const uint32_t kb = __ldg(a.fin_kb + (l0 >> 5));  // blocks of the first row (it has the most)
    uint32_t l[FIN_U], gr[FIN_U], deg[FIN_U];
    float old[FIN_U];
    double s[FIN_U];
#pragma unroll
    for (uint32_t u = 0; u < FIN_U; ++u) {
      l[u] = l0 + 32 * u + lane;
      gr[u] = 0;
      deg[u] = 1;
      old[u] = 0.0f;
      s[u] = 0.0;
      if (l[u] < a.n_fin) {
        gr[u] = deal_global(l[u], P, pp);
        old[u] = a.scores[gr[u]];
        deg[u] = a.outdeg[gr[u]];
        s[u] = (double)a.rem[l[u]];
      }
    }
#pragma unroll(FIN_U == 2 ? 16 : 4)
    for (uint32_t j = 0; j < kb; ++j) {
      const uint32_t nr = __ldg(a.walk.nrows + j);
      const float* __restrict__ pj = a.walk.partial + __ldg(a.walk.poff + j);
#pragma unroll
      for (uint32_t u = 0; u < FIN_U; ++u)
        if (l[u] < nr) s[u] += (double)pj[l[u]];
    }
#pragma unroll
    for (uint32_t u = 0; u < FIN_U; ++u)
      if (l[u] < a.n_fin) err += pr_update<PEERS>(gr[u], (float)s[u], old[u], deg[u], a);
  }
  err = warp_sum(err);
  if (lane == 0) warp_err[warp] = err;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < FIN_WARPS; ++w) t += warp_err[w];
    a.block_err[a.err_base_fin + blockIdx.x] = t;
    __threadfence();
    unsigned ticket = atomicAdd(&a.ctrl[1], 1u);
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // fixed-order reduction of all CTA partials (deterministic error)
  const uint32_t total = a.err_base_fin + gridDim.x;
  double t = 0.0;
  for (uint32_t i = threadIdx.x; i < total; i += PR_FIN_THREADS) t += ((volatile double*)a.block_err)[i];
  t = warp_sum(t);
  if (lane == 0) warp_err[warp] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double e = a.extra_err;
#pragma unroll
    for (int w = 0; w < FIN_WARPS; ++w) e += warp_err[w];
    a.err_hist[a.sweep] = e;
    a.ctrl[1] = 0;
    if (e < a.tolerance) a.ctrl[0] = a.sweep_no;
  }
}

// ---- inter-sweep barrier of the sharded path, on the device -------------------------------------------
// Every rank owns a control block in peer-mapped (symmetric) memory: arrive[q] = the last sweep rank q has
// finished, errs[sweep & 1][q] = rank q's share of that sweep's error.  After its finish kernel a rank
// publishes its error share and then its arrival into EVERY rank's block (release, system scope), waits
// until all ranks have arrived at this sweep (acquire) and adds the P shares in rank order — every rank
// gets the same total, without a host round trip or a collective.  Two error banks suffice: a rank can
// be at most one sweep ahead of the slowest (it cannot pass barrier k+1 before everyone left barrier k).
struct PrSyncBlock {
  uint32_t arrive[8];
  double errs[2][8];
};
__global__ void k_pr_sync(PrSyncBlock* self, PrSyncBlock* const* peers_dev, uint32_t P, uint32_t rank,
                          uint32_t sweep_no, const double* __restrict__ local_err, double* __restrict__ total_err,
                          uint32_t slot) {
  const uint32_t q = threadIdx.x;
  const double mine = *local_err;
  __threadfence_system();  // this rank's stores of the sweep (previous kernels) before its arrival
  if (q < P) {
    PrSyncBlock* dst = (q == rank) ? self : peers_dev[q];
    volatile double* e = &dst->errs[sweep_no & 1u][rank];
    *e = mine;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(&dst->arrive[rank]), "r"(sweep_no) : "memory");
  }
  if (q < P) {
    uint32_t seen;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(&self->arrive[q]) : "memory");
    } while ((int32_t)(seen - sweep_no) < 0);
  }
  __syncthreads();
  if (q == 0) {
    double t = 0.0;
    for (uint32_t r = 0; r < P; ++r) t += ((volatile double*)self->errs[sweep_no & 1u])[r];
    total_err[slot] = t;
  }
}

// own == 0: scores of rows this rank does not own stay 0 so that the ranks' vectors can be summed
__global__ void k_pr_init(uint32_t n, uint32_t n_active, float init, float base, PrDeal deal,
                          const uint32_t* __restrict__ outdeg, float* __restrict__ x0,
                          float* __restrict__ x1, float* __restrict__ scores) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    float d = (float)outdeg[r];
    x0[r] = __fdiv_rn(init, d);  // page_rank.rs:75-79; +inf for dangling vertices, never gathered
    const bool mine = ((r >> 5) % deal.P) == deal.p;
    if (r < n_active) {
      scores[r] = mine ? init : 0.0f;
    } else {
      // no in-edges: after the first sweep score == base + damping * 0 == base, for ever
      scores[r] = deal.p == 0 ? base : 0.0f;
      x1[r] = __fdiv_rn(base, d);
    }
  }
}
__global__ void k_pr_fill_inactive(uint32_t n, uint32_t n_active, float base,
                                   const uint32_t* __restrict__ outdeg, float* __restrict__ x) {
  for (uint32_t r = n_active + blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x)
    x[r] = __fdiv_rn(base, (float)outdeg[r]);
}
__global__ void k_unpermute(const float* __restrict__ src, const uint32_t* __restrict__ new_id,
                            uint32_t n, float* __restrict__ dst) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    dst[v] = src[new_id[v]];
}

// ---- EXACT: the reference sweep on one warp ---------------------------------------------------
// page_rank.rs:58-168 with the loop of :142-160 executed in id order.  Lanes fetch 32 gathered values
// at a time; every lane then performs the same sequential f32 additions in CSR order.
__global__ void __launch_bounds__(32) k_pr_exact(const uint32_t* __restrict__ in_off,
                                                 const uint32_t* __restrict__ in_tgt,
                                                 const uint32_t* __restrict__ out_off, uint32_t n,
                                                 uint64_t max_iterations, double tolerance, float damping,
                                                 float* scores, float* out, uint64_t* ran,
                                                 double* error) {
  const uint32_t lane = threadIdx.x;
  const float nf = (float)n;
  const float init = __fdiv_rn(1.0f, nf);
  const float base = __fdiv_rn(__fsub_rn(1.0f, damping), nf);
  for (uint32_t v = lane; v < n; v += 32) {
    out[v] = __fdiv_rn(init, (float)(out_off[v + 1] - out_off[v]));
    scores[v] = init;
  }
  __syncwarp();
  uint64_t it = 0;
  double err = 0.0;
  for (;;) {
    err = 0.0;
    for (uint32_t u = 0; u < n; ++u) {
      const uint32_t b = in_off[u], e = in_off[u + 1];
      float tot = 0.0f;
      for (uint32_t i = b; i < e; i += 32) {
        const uint32_t cnt = min(32u, e - i);
        float val = 0.0f;
        if (lane < cnt) val = ((volatile float*)out)[in_tgt[i + lane]];
        for (uint32_t j = 0; j < cnt; ++j) tot = __fadd_rn(tot, __shfl_sync(0xFFFFFFFFu, val, j));
      }
      const float old = scores[u];
      const float nw = __fadd_rn(base, __fmul_rn(damping, tot));
      err += fabs((double)__fsub_rn(nw, old));
      __syncwarp();
      if (lane == 0) {
        scores[u] = nw;
        ((volatile float*)out)[u] = __fdiv_rn(nw, (float)(out_off[u + 1] - out_off[u]));
      }
      __syncwarp();
    }
    ++it;
    if (err < tolerance || it == max_iterations) break;  // page_rank.rs:107
  }
  if (lane == 0) {
    *ran = it;
    *error = err;
  }
}

// The dynamic shared memory k_pr_cb<KIND> can take on `device`: the per-block opt-in limit less its static
// shared memory
template <uint32_t KIND>
static gb_status cb_smem_limit(int device, size_t* bytes) {
  int optin = 0;
  GB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  cudaFuncAttributes fa{};
  GB_CUDA(cudaFuncGetAttributes(&fa, k_pr_cb<KIND>));
  *bytes = (size_t)optin - fa.sharedSizeBytes;
  return GB_OK;
}
// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the kernel, for the whole process, and every plan's
// launches need it at least as large as their own shared memory (smem_cb, smem_vb).  So it is set to the
// device's limit, not to the plan's size: a plan built later (another B, another window of V) never lowers it
// below what an earlier plan, still cached, launches with.
template <uint32_t KIND>
static gb_status cb_smem_ceiling(int device, size_t need) {
  size_t lim = 0;
  GB_TRY(cb_smem_limit<KIND>(device, &lim));
  GB_REQUIRE(need <= lim, "k_pr_cb needs %zu bytes of shared memory, the device allows %zu", need, lim);
  GB_CUDA(cudaFuncSetAttribute(k_pr_cb<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lim));
  return GB_OK;
}

// ---- launch shapes: the last stage of the layout build --------------------------------------------
gb_status plan_sweep_shape(PrPlan* p, const std::vector<uint32_t>& h_nrows, const std::vector<uint32_t>& h_poff,
                           int dev_sms, cudaStream_t s) {
  p->trace = (uint32_t)env_u64("GB_PR_TRACE", 0) != 0;
  p->smem_cb = ((size_t)p->B + 4) * sizeof(float);
  p->smem_vb = p->vb ? ((size_t)p->v.window + 4) * sizeof(float) : p->smem_cb;
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  GB_TRY(cb_smem_ceiling<CB_MAIN>(dev, p->smem_cb));
  GB_TRY(cb_smem_ceiling<CB_VIRT>(dev, p->smem_vb));
  GB_TRY(cb_smem_ceiling<CB_FUSED>(dev, p->smem_cb));
  const uint64_t want_sell = ((uint64_t)p->num_slices + PR_SELL_THREADS / 32 - 1) / (PR_SELL_THREADS / 32);
  p->grid_sell = (unsigned)std::min<uint64_t>(want_sell, (uint64_t)dev_sms * 2);
  // rows with segments in more than SELL_FEW blocks are a prefix (nrows[] is non-increasing): k_pr_finish
  // completes them; all others are completed by their k_pr_sell lane (k_pr_cb is done by then).  With virtual
  // blocks k_pr_finish completes every local row.
  p->n_fin = p->hot.KB > SELL_FEW ? std::min<uint32_t>(p->n_cb, (h_nrows[SELL_FEW] + 31) / 32 * 32) : 0;
  if (p->vb) p->n_fin = p->n_loc;
  for (uint32_t j = 0; j < SELL_FEW && j < p->hot.KB; ++j) {
    p->few_nrows[j] = h_nrows[j];
    p->few_poff[j] = h_poff[j];
  }
  p->n_fin_warp =
      p->hot.KB > FIN_CTA_BLOCKS ? std::min<uint32_t>(p->n_fin, (h_nrows[FIN_CTA_BLOCKS] + 31) / 32 * 32) : 0;
  const uint64_t fin_warps2 = (uint64_t)p->n_fin_warp / 32 * (PR_FIN_THREADS / 32) + (p->n_fin - p->n_fin_warp + 63) / 64;
  const uint64_t fin_warps4 = (uint64_t)p->n_fin_warp / 32 * (PR_FIN_THREADS / 32) + (p->n_fin - p->n_fin_warp + 127) / 128;
  p->fin_u = (fin_warps2 + PR_FIN_THREADS / 32 - 1) / (PR_FIN_THREADS / 32) <= (uint64_t)dev_sms * 8 ? 2 : 4;
  // GB_PR_FIN_U (experiment / tests): 2 or 4 forces that instantiation of k_pr_finish; anything else = automatic
  const uint32_t force_u = (uint32_t)env_u64("GB_PR_FIN_U", 0);
  if (force_u == 2 || force_u == 4) p->fin_u = force_u;
  const uint64_t fin_tasks = p->fin_u == 2 ? fin_warps2 : fin_warps4;
  const uint64_t want_fin = (fin_tasks + PR_FIN_THREADS / 32 - 1) / (PR_FIN_THREADS / 32);
  p->grid_fin = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want_fin, (uint64_t)dev_sms * 8));
  // Role split of the finish CTAs: when every CTA has at most one pass of each kind to do (the grid is not
  // capped) and the hub chain is long (hundreds of blocks per row), CTAs [0, hub groups) take one hub
  // group each and the others the remaining rows — the two latency chains then run side by side instead
  // of one after the other in every CTA.  It pays on a shard of a large graph; there is nothing to gain
  // when the grid is capped (RMAT-26 on one GPU) or the hub chain is short (RMAT-22), where every CTA keeps
  // doing both parts.
  // GB_PR_FIN_SPLIT (experiment / tests): 1 forces the split, 2 never splits, 0 = automatic.  Forcing waives
  // only the two conditions above that decide whether it pays; the structural ones stay (a hub group to
  // take, rows left for the others, and at least one CTA beyond the hub CTAs: else no CTA would update
  // the tail rows).
  p->fin_hub_ctas = 0;
  const uint32_t split = (uint32_t)env_u64("GB_PR_FIN_SPLIT", 0);
  const bool split_pays = want_fin <= (uint64_t)dev_sms * 8 && p->hot.KB > 4 * FIN_CTA_BLOCKS;
  if (p->n_fin_warp && p->n_fin > p->n_fin_warp && p->grid_fin > p->n_fin_warp / 32 &&
      (split == 1 || (split == 0 && split_pays)))
    p->fin_hub_ctas = p->n_fin_warp / 32;
  // the kernel that adds the parts of cut segments (PrFix): k_pr_sell only when it completes none of their rows
  if (!p->hot.n_fix) p->fix_at = PrFix::NONE;
  else if (p->vb) p->fix_at = PrFix::PASS_B;
  else if (p->grid_sell && p->hot.fix_max_row < p->n_fin) p->fix_at = PrFix::SELL;
  else p->fix_at = PrFix::FIXUP;
  const size_t nerr = (size_t)p->grid_sell + p->grid_fin;
  GB_TRY(p->block_err.alloc(nerr));
  GB_CUDA(cudaMemsetAsync(p->block_err.p, 0, nerr * sizeof(double), s));
  GB_TRY(p->err_hist.alloc(64));
  GB_TRY(p->ctrl.alloc(2));
  GB_CUDA(cudaMemsetAsync(p->ctrl.p, 0, 8, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

gb_status pr_vb_window(int device, uint32_t* window) {
  size_t lim = 0;
  GB_TRY(cb_smem_limit<CB_VIRT>(device, &lim));
  uint32_t W = (uint32_t)(lim / sizeof(float) - 4) / VB_ALIGN * VB_ALIGN;
  // pass B's ids are 16-bit: every V-local slot and the pad id W itself stay below 0xFFFF
  W = std::min<uint32_t>(W, 0xFFFFu & ~(VB_ALIGN - 1));
  const uint64_t force = env_u64("GB_PR_VB_WINDOW", 0);
  if (force) W = (uint32_t)std::min<uint64_t>(W, force / VB_ALIGN * VB_ALIGN);
  *window = W;
  return GB_OK;
}

// a stream's scheduler and walker groups of PrArgs
static CbSched sched_of(const CbStream& st, uint32_t* task_ctr) {
  return CbSched{st.blk.p, st.tasks.p, st.n_tasks, task_ctr};
}
static CbWalk walk_of(const CbStream& st) {
  return CbWalk{st.nrows.p, st.poff.p, st.ids.p, st.bits.p, st.partial.p, st.chunks.p, st.n_chunks,
                st.tail_slot.p, st.side.p, st.fix_list.p, st.n_fix};
}
// the arguments of k_pr_cb<CB_MAIN>, k_pr_fixup, k_pr_sell and k_pr_finish: the hot blocks' stream, for every
// sweep (the per-sweep fields are set by enqueue_sweep)
static PrArgs make_args(const PrPlan* p, float base, float damping, double tolerance) {
  PrArgs a{};
  a.outdeg = p->outdeg.p;
  a.n = p->n;
  a.deal = p->deal;
  a.n_loc = p->n_loc;
  a.n_cb = p->n_cb;
  a.n_fin_warp = p->n_fin_warp;
  a.fin_hub_ctas = p->fin_hub_ctas;
  a.n_fin = p->n_fin;
  a.few_kb = std::min<uint32_t>(p->hot.KB, SELL_FEW);
  for (uint32_t j = 0; j < SELL_FEW; ++j) {
    a.few_nrows[j] = p->few_nrows[j];
    a.few_poff[j] = p->few_poff[j];
  }
  a.fix_in_sell = p->fix_at == PrFix::SELL ? 1u : 0u;
  a.B = p->B;
  a.sched = sched_of(p->hot, p->task_ctr.p);
  a.walk = walk_of(p->hot);
  a.n_task_ranges = p->task_ranges();
  a.rem = p->vb ? p->v.virt.partial.p : p->rem.p;
  a.fin_kb = p->fin_kb.p;
  a.sell = p->sell.p;
  a.slice_meta = p->slice_meta.p;
  a.num_slices = p->num_slices;
  a.block_err = p->block_err.p;
  a.err_hist = p->err_hist.p;
  a.ctrl = p->ctrl.p;
  a.err_base_fin = p->grid_sell;
  a.base = base;
  a.damping = damping;
  a.tolerance = tolerance;
  a.n_peers = 0;
  a.mc_next = nullptr;
  return a;
}
// k_pr_cb<CB_FUSED>: the hot blocks' walker and pass A of the virtual blocks, over the fused tasks
static PrArgs fused_args(const PrPlan* p, PrArgs a) {
  const PrVBlocks& v = p->v;
  a.sched = CbSched{nullptr, nullptr, v.n_tasks, p->task_ctr.p};
  a.fused_tasks = v.tasks.p;
  a.vals = v.val.p;
  a.bin_ids = v.bin_ids.p;
  a.bin_bits = v.bin_bits.p;
  a.bin_grun = v.bin_grun.p;
  a.bin_runs = v.bin_runs.p;
  a.bin_chunks = v.bin_chunks.p;
  a.bin_fill = v.sectors ? 1u : 0u;
  return a;
}
// pass B: the virtual blocks' stream, over V, in blocks of its window; its partials are the rows' cold sums
// (k_pr_finish's rem).  Its first warps add the hot blocks' cut segments (PrFix::PASS_B).
static PrArgs pass_b_args(const PrPlan* p, PrArgs a) {
  a.x_cur = p->v.val.p;
  a.B = p->v.window;
  a.sched = sched_of(p->v.virt, p->task_ctr.p + p->grid_cb);
  a.walk = walk_of(p->v.virt);
  a.fix = walk_of(p->hot);
  if (p->fix_at != PrFix::PASS_B) a.fix.n_fix = 0;
  return a;
}

// one sweep = column blocks (+ fixup of cut segments) and SELL rows, or column blocks fused with pass A of the
// virtual blocks and pass B; then finish.  *launches is advanced by the kernels launched
template <bool PEERS>
static gb_status launch_sweep(const PrPlan* p, const PrArgs& a, cudaStream_t s, uint64_t* launches) {
  cudaEvent_t* ev = nullptr;
  if (p->trace && p->trace_events.size() < 5 * 256) {
    const size_t base = p->trace_events.size();
    p->trace_events.resize(base + 5);
    for (int k = 0; k < 5; ++k) GB_CUDA(cudaEventCreate(&p->trace_events[base + k]));
    ev = &p->trace_events[base];
    GB_CUDA(cudaEventRecord(ev[0], s));
  }
  if (p->grid_cb) {
    if (p->vb) k_pr_cb<CB_FUSED><<<p->grid_cb, PR_THREADS, p->smem_cb, s>>>(fused_args(p, a));
    else k_pr_cb<CB_MAIN><<<p->grid_cb, PR_THREADS, p->smem_cb, s>>>(a);
    *launches += 1;
  }
  if (ev) GB_CUDA(cudaEventRecord(ev[1], s));
  if (p->fix_at == PrFix::FIXUP) {
    k_pr_fixup<<<grid_for((uint64_t)p->hot.n_fix * 32, 128, 296), 128, 0, s>>>(a);
    *launches += 1;
  }
  if (ev) GB_CUDA(cudaEventRecord(ev[2], s));
  if (p->grid_sell) {
    k_pr_sell<PEERS><<<p->grid_sell, PR_SELL_THREADS, 0, s>>>(a);
    *launches += 1;
  }
  if (p->vb) {
    k_pr_cb<CB_VIRT><<<p->grid_vb, PR_THREADS, p->smem_vb, s>>>(pass_b_args(p, a));
    *launches += 1;
  }
  if (ev) GB_CUDA(cudaEventRecord(ev[3], s));
  if (p->fin_u == 2) k_pr_finish<PEERS, 2><<<p->grid_fin, PR_FIN_THREADS, 0, s>>>(a);
  else k_pr_finish<PEERS, 4><<<p->grid_fin, PR_FIN_THREADS, 0, s>>>(a);
  if (ev) GB_CUDA(cudaEventRecord(ev[4], s));
  *launches += 1;
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

struct PrStart {  // init and base of page_rank.rs:70-71
  float init, base;
  PrStart(uint32_t n, float damping) : init(1.0f / (float)n), base((1.0f - damping) / (float)n) {}
};
// x0 = init / outdeg, the constant part of x1, the scores (k_pr_init), and the stop flag and task cursors
static gb_status pr_reset(const PrPlan* p, PrStart v, float* x0, float* x1, float* scores, cudaStream_t s) {
  k_pr_init<<<grid_for(p->n, 256), 256, 0, s>>>(p->n, p->n_active, v.init, v.base, p->deal, p->outdeg.p, x0, x1,
                                                scores);
  GB_CUDA(cudaMemsetAsync(p->ctrl.p, 0, 8, s));
  GB_CUDA(cudaMemsetAsync(p->task_ctr.p, 0, (size_t)std::max<unsigned>(p->task_ranges(), 1) * 4, s));
  return GB_OK;
}
// the closed-form error of the rows without in-edges, contributed to sweep 1 once, by rank 0
static double first_sweep_err(const PrPlan* p, uint64_t sweep_no, PrStart v) {
  return (sweep_no == 1 && p->deal.p == 0) ? (double)(p->n - p->n_active) * fabs((double)(v.base - v.init)) : 0.0;
}
// Sweep sweep_no, entry `sweep` of a.err_hist, from x_cur into x_next (a: make_args and the caller's vectors).
// `done` (if any) is recorded after the sweep's kernels.  Sources without in-edges change exactly once
// (init/deg -> base/deg): after sweep 1, the vector that sweep has just finished reading is patched.
template <bool PEERS>
static gb_status enqueue_sweep(const PrPlan* p, PrArgs a, PrStart v, const float* x_cur, float* x_next,
                               uint32_t sweep, uint64_t sweep_no, cudaEvent_t done, cudaStream_t s,
                               uint64_t* launches) {
  a.x_cur = x_cur;
  a.x_next = x_next;
  a.sweep = sweep;
  a.sweep_no = (uint32_t)std::min<uint64_t>(sweep_no, 0xFFFFFFFFull);
  a.extra_err = first_sweep_err(p, sweep_no, v);
  GB_TRY(launch_sweep<PEERS>(p, a, s, launches));
  if (done) GB_CUDA(cudaEventRecord(done, s));
  if (sweep_no == 1 && p->n_active < p->n) {
    k_pr_fill_inactive<<<grid_for(p->n - p->n_active, 256), 256, 0, s>>>(p->n, p->n_active, v.base, p->outdeg.p,
                                                                       const_cast<float*>(x_cur));
    *launches += 1;
  }
  return GB_OK;
}

// ---- drivers ---------------------------------------------------------------------------------
gb_status require_pr_config(const gb_page_rank_config* cfg) {
  GB_REQUIRE(!(cfg->max_iterations == 0 && !(cfg->tolerance > 0.0)),
             "max_iterations == 0 with tolerance <= 0 never terminates (page_rank.rs:107)");
  return GB_OK;
}
uint64_t pr_sweep_limit(const gb_page_rank_config* cfg) {
  return cfg->max_iterations ? cfg->max_iterations : 100000ull;
}

static gb_status run_exact(const gb_graph* g, const gb_page_rank_config* cfg, float* d_scores,
                           uint64_t* ran, double* error) {
  cudaStream_t s = g->stream;
  DevBuf<float> out;
  DevBuf<uint64_t> d_ran;
  DevBuf<double> d_err;
  GB_TRY(out.alloc(g->n));
  GB_TRY(d_ran.alloc(1));
  GB_TRY(d_err.alloc(1));
  k_pr_exact<<<1, 32, 0, s>>>(g->in.off.p, g->in.tgt.p, g->out.off.p, g->n, cfg->max_iterations,
                             cfg->tolerance, cfg->damping_factor, d_scores, out.p, d_ran.p, d_err.p);
  GB_CUDA(cudaGetLastError());
  g->timing.kernel_launches += 1;
  GB_CUDA(cudaMemcpyAsync(ran, d_ran.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(error, d_err.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

static gb_status run_jacobi(const gb_graph* g, const gb_page_rank_config* cfg, float* d_scores,
                            uint64_t* ran, double* error) {
  PrPlan* p = g->pr_plan;  // built by page_rank_impl
  cudaStream_t s = g->stream;
  const uint32_t n = p->n;
  const PrStart v(n, cfg->damping_factor);
  const bool profile = profiling_on();
  if (!p->x[0].p) {
    GB_TRY(p->x[0].alloc(n));
    GB_TRY(p->x[1].alloc(n));
    GB_TRY(p->scores.alloc(n));
  }

  GB_TRY(pr_reset(p, v, p->x[0].p, p->x[1].p, p->scores.p, s));
  g->timing.kernel_launches += 1;

  PrArgs a = make_args(p, v.base, cfg->damping_factor, cfg->tolerance);
  a.scores = p->scores.p;

  const uint64_t limit = pr_sweep_limit(cfg);
  const bool can_stop_early = cfg->tolerance > 0.0;
  const uint32_t batch_cap = 64;
  uint64_t done = 0;      // sweeps launched so far
  uint64_t stopped = 0;   // sweep number at which the tolerance was met (0 = not yet)
  double last_err = 0.0;
  size_t ev_used = 0;
  while (done < limit && !stopped) {
    const uint32_t batch = (uint32_t)std::min<uint64_t>(limit - done, can_stop_early ? 8 : batch_cap);
    for (uint32_t b = 0; b < batch; ++b) {
      const uint64_t sweep_no = done + b + 1;
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      if (profile && ev_used + 2 <= 2 * PR_MAX_PROFILE_EVENTS) {
        while (p->prof_events.size() < ev_used + 2) {
          cudaEvent_t e;
          GB_CUDA(cudaEventCreate(&e));
          p->prof_events.push_back(e);
        }
        e0 = p->prof_events[ev_used];
        e1 = p->prof_events[ev_used + 1];
        ev_used += 2;
        GB_CUDA(cudaEventRecord(e0, s));
      }
      GB_TRY(enqueue_sweep<false>(p, a, v, p->x[(sweep_no - 1) & 1].p, p->x[sweep_no & 1].p, b, sweep_no, e1, s,
                                  &g->timing.kernel_launches));
    }
    GB_CUDA(cudaGetLastError());
    done += batch;
    if (can_stop_early || done >= limit) {
      uint32_t ctrl0 = 0;
      GB_CUDA(cudaMemcpyAsync(&ctrl0, p->ctrl.p, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      if (ctrl0 != 0) stopped = ctrl0;
      const uint64_t last = stopped ? stopped : done;
      const uint32_t slot = (uint32_t)(last - (done - batch) - 1);
      GB_CUDA(cudaMemcpyAsync(&last_err, p->err_hist.p + slot, 8, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
    }
  }
  *ran = stopped ? stopped : done;
  *error = last_err;
  k_unpermute<<<grid_for(n, 256), 256, 0, s>>>(p->scores.p, p->new_id.p, n, d_scores);
  g->timing.kernel_launches += 1;
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  if (profile) {
    double ms = 0.0;
    for (size_t i = 0; i + 1 < ev_used; i += 2) {
      float t = 0.0f;
      GB_CUDA(cudaEventElapsedTime(&t, p->prof_events[i], p->prof_events[i + 1]));
      ms += t;
    }
    g->timing.hot_kernel_ms = ms;
    g->timing.hot_kernel_launches = ev_used / 2;
  }
  return GB_OK;
}

static gb_status ensure_plan(const gb_graph* g) {
  if (!g->pr_plan) GB_TRY(build_pr_plan(g, PrDeal{}, &g->pr_plan));
  return GB_OK;
}
static void plan_stats(const PrPlan* p, gb_pr_shard_stats* stats) {
  stats->rank = p->deal.p;
  stats->world = p->deal.P;
  stats->active_rows = p->n_active;
  stats->local_rows = p->n_loc;
  stats->local_edges = p->loc_edges;
  stats->block_edges = p->cb_edges;
  stats->block_entries = p->B;
  stats->hot_blocks = p->hot.KB;
  stats->segments = p->hot.S;
  stats->groups = p->hot.NG;
  stats->chunks = p->hot.n_chunks;
  stats->tasks = p->vb ? p->v.n_tasks : p->hot.n_tasks;  // k_pr_cb's tasks (CB_FUSED's with virtual blocks)
  stats->cut_segments = p->hot.n_fix;
  stats->chunk_groups = p->hot.chunk_groups;
  stats->launches_per_sweep = 1 + (p->grid_cb ? 1 : 0) + (p->grid_sell ? 1 : 0) +
                              (p->fix_at == PrFix::FIXUP ? 1 : 0) + (p->vb ? 1 : 0);
  stats->device_bytes = p->bytes();
  stats->vblock_parts = p->vb ? p->v.virt.KB : 0;
  stats->vblock_pairs = p->vb ? p->v.pairs : 0;
  stats->vblock_edges = p->vb ? p->v.edges : 0;
  stats->vblock_wide_steps = p->vb ? p->v.wide_steps : 0;
  stats->vblock_slots = p->vb ? p->v.slots : 0;
  stats->vblock_sectors = p->vb && p->v.sectors ? 1u : 0u;
}
static void plan_shape(const PrPlan* p, gb_pr_plan_shape* shape) {
  shape->hot_blocks = p->hot.KB;
  shape->n_cb = p->n_cb;
  shape->n_fin = p->n_fin;
  shape->n_fin_warp = p->n_fin_warp;
  shape->fin_u = p->fin_u;
  shape->fin_hub_ctas = p->fin_hub_ctas;
  shape->grid_cb = p->grid_cb;
  shape->grid_sell = p->grid_sell;
  shape->grid_fin = p->grid_fin;
  shape->n_mega = p->n_mega;
  shape->n_fix = p->hot.n_fix;
  shape->fix_in_sell = p->fix_at == PrFix::SELL ? 1u : 0u;
  shape->dual = 0;
  shape->last_hot_block = p->last_hot_block;
}
// the value buffer V of a plan's virtual blocks: poison it with 0xFFFFFFFF, and / or copy it to the host
static gb_status plan_values(const PrPlan* p, int poison, float* values, uint64_t count) {
  const PrVBlocks& v = p->v;
  GB_REQUIRE(p->vb, "the layout has no virtual blocks");
  GB_REQUIRE(count == v.slots, "count %llu is not the value buffer's %llu slots", (unsigned long long)count,
             (unsigned long long)v.slots);
  if (poison) {
    GB_CUDA(cudaMemsetAsync(v.val.p, 0xFF, v.slots * sizeof(float), 0));
    GB_CUDA(cudaStreamSynchronize(0));
  }
  if (values) GB_CUDA(cudaMemcpy(values, v.val.p, v.slots * sizeof(float), cudaMemcpyDeviceToHost));
  return GB_OK;
}

gb_status page_rank_impl(const gb_graph* g, const gb_page_rank_config* cfg, float* d_scores, float* h_scores,
                         uint64_t* ran, double* error) {
  GB_REQUIRE(g && cfg && ran && error, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED)
    return fail(GB_ERR_UNSUPPORTED, "page_rank needs a directed graph (page_rank.rs:61)");
  GB_REQUIRE(cfg->mode <= GB_PR_JACOBI, "bad page rank mode %u", cfg->mode);
  GB_TRY(require_pr_config(cfg));
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  uint32_t mode = cfg->mode;
  if (mode == GB_PR_AUTO) mode = (g->n <= 16384) ? GB_PR_EXACT : GB_PR_JACOBI;
  if (mode == GB_PR_JACOBI) GB_TRY(ensure_plan(g));  // not timed; refuses n >= 2^31 - 1 before any allocation
  DevBuf<float> tmp_scores;
  if (!d_scores) {
    GB_TRY(tmp_scores.alloc(g->n));
    d_scores = tmp_scores.p;
  }
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  if (mode == GB_PR_EXACT) GB_TRY(run_exact(g, cfg, d_scores, ran, error));
  else GB_TRY(run_jacobi(g, cfg, d_scores, ran, error));
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  if (h_scores) GB_CUDA(cudaMemcpyAsync(h_scores, d_scores, (size_t)g->n * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
  return GB_OK;
}

}  // namespace gb

// ---- multi-GPU shard (1-D edge-cut by destination, 32-row slices dealt round-robin) ----------------
struct gb_pr_shard {
  int device = 0;                     // the plan's device: a shard holds no graph, which may be freed before it
  gb::PrPlan* plan = nullptr;
  gb::DevBuf<void*> sync_table;       // device copy of the ranks' control-block pointers (gb_pr_shard_sync)
  void* sync_table_host[8] = {nullptr};
};

namespace gb {
gb_status shard_from_plan(int device, PrPlan* plan, gb_pr_shard** out) {
  gb_pr_shard* sh = new (std::nothrow) gb_pr_shard();
  if (!sh) {
    DeviceGuard guard(device);
    free_pr_plan(plan);
    return fail(GB_ERR_OOM, "host allocation failed");
  }
  sh->device = device;
  sh->plan = plan;
  *out = sh;
  return GB_OK;
}
}  // namespace gb

extern "C" {

gb_status gb_pr_shard_create(const gb_graph* g, uint32_t rank, uint32_t world, gb_pr_shard** shard) {
  GB_REQUIRE(g && shard, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED) return gb::fail(GB_ERR_UNSUPPORTED, "page rank shards need a directed graph");
  GB_REQUIRE(world >= 1 && rank < world, "bad shard %u of %u", rank, world);
  gb::DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  gb_pr_shard* sh = new (std::nothrow) gb_pr_shard();
  if (!sh) return gb::fail(GB_ERR_OOM, "host allocation failed");
  sh->device = g->device;
  gb_status st = gb::build_pr_plan(g, gb::PrDeal(world, rank), &sh->plan);
  if (st != GB_OK) {
    delete sh;
    return st;
  }
  *shard = sh;
  return GB_OK;
}

gb_status gb_pr_shard_free(gb_pr_shard* shard) {
  if (!shard) return GB_OK;
  // the plan owns all its memory: freeing it needs the device, not the graph, which may be gone already
  gb::DeviceGuard guard(shard->device);
  gb::free_pr_plan(shard->plan);
  delete shard;
  return GB_OK;
}

gb_status gb_pr_shard_init(const gb_pr_shard* shard, float damping, float* d_x0, float* d_x1,
                           float* d_scores, void* cuda_stream) {
  GB_REQUIRE(shard && d_x0 && d_x1 && d_scores, "NULL argument");
  const gb::PrPlan* p = shard->plan;
  gb::DeviceGuard guard(shard->device);
  // every rank fills the whole initial vector itself (no exchange needed before sweep 1)
  GB_TRY(gb::pr_reset(p, gb::PrStart(p->n, damping), d_x0, d_x1, d_scores, (cudaStream_t)cuda_stream));
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

gb_status gb_pr_shard_step(const gb_pr_shard* shard, float damping, uint64_t sweep_no, const float* d_x_cur,
                           float* d_x_next, float* const* d_peer_x_next, uint32_t peer_count,
                           float* d_mc_x_next, float* d_scores, double* d_error, void* cuda_stream) {
  GB_REQUIRE(shard && d_x_cur && d_x_next && d_scores && d_error, "NULL argument");
  GB_REQUIRE(peer_count <= 7, "at most 7 peers");
  GB_REQUIRE(peer_count == 0 || d_peer_x_next || d_mc_x_next, "peer pointer array is NULL");
  GB_REQUIRE(sweep_no >= 1, "sweep_no is 1-based");
  const gb::PrPlan* p = shard->plan;
  gb::DeviceGuard guard(shard->device);
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const gb::PrStart v(p->n, damping);
  gb::PrArgs a = gb::make_args(p, v.base, damping, -1.0 /* the caller owns the stop rule */);
  a.scores = d_scores;
  a.n_peers = d_mc_x_next ? 0 : peer_count;
  a.mc_next = d_mc_x_next;
  for (uint32_t i = 0; i < a.n_peers; ++i) a.peer_next[i] = d_peer_x_next[i];
  a.err_hist = d_error;
  uint64_t launches = 0;
  if (peer_count || d_mc_x_next)
    GB_TRY(gb::enqueue_sweep<true>(p, a, v, d_x_cur, d_x_next, 0, sweep_no, nullptr, s, &launches));
  else GB_TRY(gb::enqueue_sweep<false>(p, a, v, d_x_cur, d_x_next, 0, sweep_no, nullptr, s, &launches));
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

gb_status gb_pr_shard_sync(const gb_pr_shard* shard, uint64_t sweep_no, const double* d_local_error,
                           void* d_self_block, void* const* d_peer_blocks, double* d_total_error,
                           uint32_t slot, void* cuda_stream) {
  GB_REQUIRE(shard && d_local_error && d_self_block && d_total_error, "NULL argument");
  const gb::PrPlan* p = shard->plan;
  GB_REQUIRE(p->deal.P <= 8, "at most 8 ranks");
  GB_REQUIRE(p->deal.P == 1 || d_peer_blocks, "peer block array is NULL");
  GB_REQUIRE(sweep_no >= 1 && sweep_no < 0x7FFFFFFFull, "bad sweep number");
  gb::DeviceGuard guard(shard->device);
  cudaStream_t s = (cudaStream_t)cuda_stream;
  // the peer pointer table lives in the shard (device copy, refreshed when the pointers change)
  gb_pr_shard* sh = const_cast<gb_pr_shard*>(shard);
  void* table[8] = {nullptr};
  for (uint32_t q = 0; q < p->deal.P; ++q) table[q] = (q == p->deal.p) ? d_self_block : d_peer_blocks[q];
  if (!sh->sync_table.p || memcmp(table, sh->sync_table_host, sizeof table) != 0) {
    if (!sh->sync_table.p) GB_TRY(sh->sync_table.alloc(8));
    memcpy(sh->sync_table_host, table, sizeof table);
    GB_CUDA(cudaMemcpyAsync(sh->sync_table.p, table, sizeof table, cudaMemcpyHostToDevice, s));
  }
  gb::k_pr_sync<<<1, 32, 0, s>>>(static_cast<gb::PrSyncBlock*>(d_self_block),
                                reinterpret_cast<gb::PrSyncBlock* const*>(sh->sync_table.p), p->deal.P, p->deal.p,
                                (uint32_t)sweep_no, d_local_error, d_total_error, slot);
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

gb_status gb_pr_shard_finish(const gb_pr_shard* shard, const float* d_scores_internal, float* d_scores_out,
                             void* cuda_stream) {
  GB_REQUIRE(shard && d_scores_internal && d_scores_out, "NULL argument");
  const gb::PrPlan* p = shard->plan;
  gb::DeviceGuard guard(shard->device);
  gb::k_unpermute<<<gb::grid_for(p->n, 256), 256, 0, (cudaStream_t)cuda_stream>>>(d_scores_internal, p->new_id.p,
                                                                                 p->n, d_scores_out);
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

gb_status gb_pr_shard_info(const gb_pr_shard* shard, gb_pr_shard_stats* stats) {
  GB_REQUIRE(shard && stats, "NULL argument");
  gb::plan_stats(shard->plan, stats);
  return GB_OK;
}

gb_status gb_page_rank_plan_info(const gb_graph* g, gb_pr_shard_stats* stats) {
  GB_REQUIRE(g && stats, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED) return gb::fail(GB_ERR_UNSUPPORTED, "page rank needs a directed graph");
  gb::DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_TRY(gb::ensure_plan(g));
  gb::plan_stats(g->pr_plan, stats);
  return GB_OK;
}

gb_status gb_page_rank_plan_values(const gb_graph* g, int poison, float* values, uint64_t count) {
  GB_REQUIRE(g, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED) return gb::fail(GB_ERR_UNSUPPORTED, "page rank needs a directed graph");
  gb::DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_TRY(gb::ensure_plan(g));
  return gb::plan_values(g->pr_plan, poison, values, count);
}

gb_status gb_pr_shard_plan_values(const gb_pr_shard* shard, int poison, float* values, uint64_t count) {
  GB_REQUIRE(shard, "NULL argument");
  gb::DeviceGuard guard(shard->device);
  return gb::plan_values(shard->plan, poison, values, count);
}

gb_status gb_pr_shard_plan_shape(const gb_pr_shard* shard, gb_pr_plan_shape* shape) {
  GB_REQUIRE(shard && shape, "NULL argument");
  gb::plan_shape(shard->plan, shape);
  return GB_OK;
}

gb_status gb_page_rank_plan_shape(const gb_graph* g, gb_pr_plan_shape* shape) {
  GB_REQUIRE(g && shape, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED) return gb::fail(GB_ERR_UNSUPPORTED, "page rank needs a directed graph");
  gb::DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_TRY(gb::ensure_plan(g));
  gb::plan_shape(g->pr_plan, shape);
  return GB_OK;
}

gb_status gb_page_rank_plan_reset(const gb_graph* g) {
  GB_REQUIRE(g, "NULL argument");
  gb::DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  gb::free_pr_plan(g->pr_plan);
  g->pr_plan = nullptr;
  return GB_OK;
}

gb_status gb_page_rank(const gb_graph* graph, const gb_page_rank_config* config, float* scores,
                       uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(scores != nullptr, "scores is NULL");
  return gb::page_rank_impl(graph, config, nullptr, scores, ran_iterations, error);
}

gb_status gb_page_rank_device(const gb_graph* graph, const gb_page_rank_config* config, float* d_scores,
                              uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(d_scores != nullptr, "d_scores is NULL");
  return gb::page_rank_impl(graph, config, d_scores, nullptr, ran_iterations, error);
}

}  // extern "C"
