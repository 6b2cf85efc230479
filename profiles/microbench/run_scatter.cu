// run_scatter.cu — do pass A's run-scattered stores into the value buffer V lose their time to partial 32-byte sectors?
// A synthetic V of 5275 partitions x 1366 source blocks of runs (lengths with mean ~35 slots, fixed seed, ~1 GB) is
// written the way k_pr_cb<CB_BIN> writes it: persistent 1024-thread CTAs take source blocks from an atomic cursor,
// each warp walks 8-step chunks of its block's share in 256-position steps, and every store instruction covers 32
// consecutive positions.  The positions, ids, start bits and first runs are the same in every variant; only where
// a run's slots lie in V changes:
//   packed   runs of one partition back to back (the layout before sector alignment)
//   aligned  every run starts at a multiple of 8 slots (one 32-byte sector), pad slots left unwritten
//   filled   aligned, and the warp stores zeros to the run's pad slots in the step that stores its last value
//   dense    V[position]: no scatter at all
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o run_scatter run_scatter.cu
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s failed: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

constexpr uint32_t NBLK = 1366, NPART = 5275, STEP = 256, CHUNK = 8, XB = 49152, PAD = 0xFFFFu;
constexpr uint32_t PACKED = 0, ALIGNED = 1, FILLED = 2, DENSE = 3;

__host__ __device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}
__host__ __device__ __forceinline__ uint32_t id_index(uint32_t pos) {  // position 32 k + L of a step at 8 L + k
  return (pos & ~(STEP - 1)) | (pos & 31u) << 3 | (pos >> 5 & 7u);
}

struct Args {
  float* v;
  const uint16_t* ids;
  const uint32_t* bits;  // per 32 positions: run starts
  const uint32_t* grun;  // per 32 positions: run of its first position
  const uint32_t* runs;  // [runs + 32] slot - position of each run's first position
  const uint32_t* bstep; // [NBLK + 1] first step of each block's share
  uint32_t steps;
  uint32_t* cursor;
};

__device__ __forceinline__ uint4 ld_stream_u4(const uint32_t* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void store(float* v, uint32_t xs_smem, uint32_t sid) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .f32 x;\n\t"
      "setp.ne.u32 p, %0, %3;\n\t"
      "mov.f32 x, 0f00000000;\n\t"
      "@p ld.shared.f32 x, [%1];\n\t"
      "@p st.global.f32 [%2], x;\n\t}" ::"r"(sid), "r"(xs_smem + 4 * sid), "l"(v), "n"(PAD)
      : "memory");
}
// zeros to slots [e, e rounded up to 8): at most one 4-, one 8- and one 16-byte store
__device__ __forceinline__ void fill_tail(float* v, uint32_t e) {
  if (e & 1u) v[e++] = 0.0f;
  if (e & 2u) { *reinterpret_cast<float2*>(v + e) = make_float2(0.0f, 0.0f); e += 2; }
  if (e & 4u) *reinterpret_cast<float4*>(v + e) = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

template <uint32_t VAR, bool WIDE>
__device__ __forceinline__ void step(const Args& a, uint32_t xs_smem, uint32_t p0, uint32_t lane, const uint4 id,
                                     const uint4 b0, const uint4 b1, uint32_t nbit, uint32_t r0, uint32_t d, uint32_t runs) {
  const uint32_t bits[9] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, nbit};
  const uint32_t w[4] = {id.x, id.y, id.z, id.w};
  const uint32_t upto = 0xFFFFFFFFu >> (31u - lane);
  uint32_t before = 0u - (bits[0] & 1u);
  uint32_t nvalid = 0;  // valid positions form a prefix of the step
  if (VAR == FILLED) {
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) nvalid += __popc(__ballot_sync(0xFFFFFFFFu, ((w[k / 2] >> (16 * (k & 1))) & 0xFFFFu) != PAD));
  }
#pragma unroll
  for (uint32_t k = 0; k < 8; ++k) {
    const uint32_t r = before + __popc(bits[k] & upto);
    before += __popc(bits[k]);
    uint32_t dk;
    if (!WIDE) {
      dk = __shfl_sync(0xFFFFFFFFu, d, r);
    } else {
      dk = __shfl_sync(0xFFFFFFFFu, d, r & 31u);
#pragma unroll 1
      for (uint32_t w0 = 32; w0 <= runs; w0 += 32) {
        const uint32_t t = __shfl_sync(0xFFFFFFFFu, __ldg(a.runs + r0 + w0 + lane), (r - w0) & 31u);
        if (r - w0 < 32) dk = t;
      }
    }
    const uint32_t sid = (w[k / 2] >> (16 * (k & 1))) & 0xFFFFu;
    if (VAR == DENSE) dk = 0;
    const uint32_t slot = p0 + 32 * k + dk;
    store(a.v + slot, xs_smem, sid);
    if (VAR == FILLED) {
      const uint32_t q = 32 * k + lane;  // the position in the step; does its run end here?
      const bool ends = q < nvalid && (q + 1 == nvalid || (__funnelshift_rc(bits[k], bits[k + 1], lane + 1) & 1u));
      if (ends) fill_tail(a.v, slot + 1);
    }
  }
}

template <uint32_t VAR>
__device__ __forceinline__ void chunk(const Args& a, uint32_t xs_smem, uint32_t s0, uint32_t s1, uint32_t lane) {
  const uint32_t* ids = reinterpret_cast<const uint32_t*>(a.ids) + 4 * lane;
  const uint4* bits4 = reinterpret_cast<const uint4*>(a.bits);
  uint4 id = ld_stream_u4(ids + 128 * (size_t)s0);
  uint4 b0 = __ldg(bits4 + 2 * s0), b1 = __ldg(bits4 + 2 * s0 + 1);
  uint32_t r0 = __ldg(a.grun + 8 * s0);
  uint32_t r0n = s0 + 1 < s1 ? __ldg(a.grun + 8 * (s0 + 1)) : 0u;
  uint32_t d = __ldg(a.runs + r0 + lane);
  for (uint32_t s = s0; s < s1; ++s) {
    uint4 nid = id, nb0 = b0, nb1 = b1;
    uint32_t nd = d, r0nn = r0n;
    if (s + 1 < s1) {
      nid = ld_stream_u4(ids + 128 * (size_t)(s + 1));
      nb0 = __ldg(bits4 + 2 * (s + 1));
      nb1 = __ldg(bits4 + 2 * (s + 1) + 1);
      nd = __ldg(a.runs + r0n + lane);
      if (s + 2 < s1) r0nn = __ldg(a.grun + 8 * (s + 2));
    }
    // start bit of the position after the step (a step after the last one starts a run)
    const uint32_t nbit = VAR != FILLED ? 0u : s + 1 < s1 ? nb0.x : s + 1 < a.steps ? __ldg(a.bits + 8 * (s + 1)) : 1u;
    const uint32_t runs = __popc(b0.x & ~1u) + __popc(b0.y) + __popc(b0.z) + __popc(b0.w) + __popc(b1.x) +
                          __popc(b1.y) + __popc(b1.z) + __popc(b1.w);
    if (runs < 32) step<VAR, false>(a, xs_smem, s * STEP + lane, lane, id, b0, b1, nbit, r0, d, runs);
    else step<VAR, true>(a, xs_smem, s * STEP + lane, lane, id, b0, b1, nbit, r0, d, runs);
    id = nid, b0 = nb0, b1 = nb1, d = nd, r0 = r0n, r0n = r0nn;
  }
}

template <uint32_t VAR>
__global__ void __launch_bounds__(1024, 1) k_scatter(const Args a) {
  extern __shared__ __align__(128) float xs[];
  __shared__ uint32_t s_blk, s_next;
  for (uint32_t i = threadIdx.x; i < XB; i += blockDim.x) xs[i] = 1.0f + (float)i;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, xs_smem = (uint32_t)__cvta_generic_to_shared(xs);
  for (;;) {
    __syncthreads();  // every warp is done with the previous block
    if (threadIdx.x == 0) {
      s_blk = atomicAdd(a.cursor, 1u);
      s_next = blockDim.x / 32;
    }
    __syncthreads();
    const uint32_t b = s_blk;
    if (b >= NBLK) break;
    const uint32_t s0 = a.bstep[b], s1 = a.bstep[b + 1], nch = (s1 - s0 + CHUNK - 1) / CHUNK;
    for (uint32_t k = warp; k < nch;) {
      chunk<VAR>(a, xs_smem, s0 + CHUNK * k, min(s1, s0 + CHUNK * k + CHUNK), lane);
      uint32_t nx = 0;
      if (lane == 0) nx = atomicAdd(&s_next, 1u);
      k = __shfl_sync(0xFFFFFFFFu, nx, 0);
    }
  }
}

__global__ void k_ids(uint16_t* ids, const uint32_t* bpos, const uint32_t* bcnt, uint32_t npos) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < npos; p += gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = NBLK;  // last block with bpos <= p
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (bpos[mid] <= p) lo = mid;
      else hi = mid;
    }
    ids[id_index(p)] = p - bpos[lo] < bcnt[lo] ? (uint16_t)(hash32(p) % XB) : (uint16_t)PAD;
  }
}
__global__ void k_count_unwritten(const uint32_t* v, uint64_t n, unsigned long long* cnt) {
  unsigned long long c = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    c += v[i] == 0xFFFFFFFFu;
  atomicAdd(cnt, c);
}

int main() {
  // run lengths: 1 + exponential with mean 34 (many short runs, a long tail), fixed seed
  std::vector<uint32_t> len((size_t)NBLK * NPART);
  uint64_t total = 0;
  for (size_t i = 0; i < len.size(); ++i) {
    const double u = (hash32((uint32_t)i * 2654435761u + 977u) + 0.5) / 4294967296.0;
    len[i] = 1 + (uint32_t)std::min(1000.0, -34.0 * std::log(u));
    total += len[i];
  }
  // pass A positions (identical in every variant): block b's share, runs in partition order, padded to a step
  std::vector<uint32_t> bpos(NBLK), bcnt(NBLK), bstep(NBLK + 1);
  uint64_t npos = 0;
  for (uint32_t b = 0; b < NBLK; ++b) {
    uint64_t c = 0;
    for (uint32_t k = 0; k < NPART; ++k) c += len[(size_t)b * NPART + k];
    bpos[b] = (uint32_t)npos, bcnt[b] = (uint32_t)c, bstep[b] = (uint32_t)(npos / STEP);
    npos += (c + STEP - 1) / STEP * STEP;
  }
  bstep[NBLK] = (uint32_t)(npos / STEP);
  const uint32_t steps = (uint32_t)(npos / STEP), nruns = NBLK * NPART;
  std::vector<uint32_t> bits(npos / 32, 0), grun(npos / 32), rpos(nruns);
  for (uint32_t b = 0; b < NBLK; ++b) {
    uint32_t p = bpos[b];
    for (uint32_t k = 0; k < NPART; ++k) {
      const uint32_t r = b * NPART + k;
      rpos[r] = p;
      bits[p / 32] |= 1u << (p % 32);
      p += len[r];
    }
  }
  for (uint32_t b = 0, r = 0; b < NBLK; ++b) {  // the run of each group's first position; pads keep the last run
    const uint32_t g0 = bpos[b] / 32, g1 = bstep[b + 1] * (STEP / 32);
    for (uint32_t g = g0; g < g1; ++g) {
      while (r + 1 < (b + 1) * NPART && rpos[r + 1] <= 32 * g) ++r;
      grun[g] = r;
    }
    r = (b + 1) * NPART;
  }
  // slots: partition-major, blocks in order inside a partition, partitions at multiples of 32 slots
  std::vector<uint32_t> runs_packed(nruns + 32, 0), runs_aligned(nruns + 32, 0);
  uint64_t vlen[2] = {0, 0}, written = total;
  for (int al = 0; al < 2; ++al) {
    uint64_t slot = 0;
    for (uint32_t k = 0; k < NPART; ++k) {
      slot = (slot + 31) / 32 * 32;
      for (uint32_t b = 0; b < NBLK; ++b) {
        const uint32_t r = b * NPART + k;
        (al ? runs_aligned : runs_packed)[r] = (uint32_t)(slot - rpos[r]);
        slot += al ? (len[r] + 7) / 8 * 8 : len[r];
      }
    }
    vlen[al] = (slot + 31) / 32 * 32;
  }
  vlen[1] = std::max<uint64_t>(vlen[1], npos);
  printf("runs %u, pairs %llu (mean run %.1f), positions %llu, V %.3f GB packed, %.3f GB aligned\n", nruns,
         (unsigned long long)total, (double)total / nruns, (unsigned long long)npos, vlen[0] * 4e-9, vlen[1] * 4e-9);

  uint32_t *d_bits, *d_grun, *d_runs[2], *d_bpos, *d_bcnt, *d_bstep, *d_cursor;
  uint16_t* d_ids;
  float* d_v;
  unsigned long long* d_cnt;
  CK(cudaMalloc(&d_bits, bits.size() * 4)); CK(cudaMalloc(&d_grun, grun.size() * 4));
  for (int al = 0; al < 2; ++al) CK(cudaMalloc(&d_runs[al], (nruns + 32) * 4ull));
  CK(cudaMalloc(&d_bpos, NBLK * 4)); CK(cudaMalloc(&d_bcnt, NBLK * 4)); CK(cudaMalloc(&d_bstep, (NBLK + 1) * 4));
  CK(cudaMalloc(&d_cursor, 4)); CK(cudaMalloc(&d_cnt, 8));
  CK(cudaMalloc(&d_ids, npos * 2));
  CK(cudaMalloc(&d_v, vlen[1] * 4));
  CK(cudaMemcpy(d_bits, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_grun, grun.data(), grun.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_runs[0], runs_packed.data(), (nruns + 32) * 4ull, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_runs[1], runs_aligned.data(), (nruns + 32) * 4ull, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_bpos, bpos.data(), NBLK * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_bcnt, bcnt.data(), NBLK * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_bstep, bstep.data(), (NBLK + 1) * 4, cudaMemcpyHostToDevice));
  k_ids<<<132 * 8, 256>>>(d_ids, d_bpos, d_bcnt, (uint32_t)npos);
  CK(cudaDeviceSynchronize());

  int sms = 132;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const size_t smem = XB * 4;
  CK(cudaFuncSetAttribute(k_scatter<PACKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(k_scatter<ALIGNED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(k_scatter<FILLED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(k_scatter<DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const char* names[4] = {"packed", "aligned", "filled", "dense"};
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto launch = [&](uint32_t var) {
    Args a{d_v, d_ids, d_bits, d_grun, d_runs[var == PACKED ? 0 : 1], d_bstep, steps, d_cursor};
    CK(cudaMemsetAsync(d_cursor, 0, 4));
    CK(cudaEventRecord(e0));
    if (var == PACKED) k_scatter<PACKED><<<sms, 1024, smem>>>(a);
    else if (var == ALIGNED) k_scatter<ALIGNED><<<sms, 1024, smem>>>(a);
    else if (var == FILLED) k_scatter<FILLED><<<sms, 1024, smem>>>(a);
    else k_scatter<DENSE><<<sms, 1024, smem>>>(a);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms;
  };
  // check the walk: slots that no store reached, against the layout (alignment gaps; pads unless filled)
  for (uint32_t var = 0; var < 4; ++var) {
    const uint64_t n = var == PACKED ? vlen[0] : var == DENSE ? npos : vlen[1];
    CK(cudaMemset(d_v, 0xFF, n * 4)); CK(cudaMemset(d_cnt, 0, 8));
    launch(var);
    k_count_unwritten<<<sms * 8, 256>>>(reinterpret_cast<const uint32_t*>(d_v), n, d_cnt);
    unsigned long long got = 0;
    CK(cudaMemcpy(&got, d_cnt, 8, cudaMemcpyDeviceToHost));
    uint64_t want = n - written;
    if (var == FILLED) {
      uint64_t padded = 0;
      for (uint32_t r = 0; r < nruns; ++r) padded += (len[r] + 7) / 8 * 8;
      want = n - padded;
    }
    printf("%-8s unwritten slots %llu (expected %llu)%s\n", names[var], got, (unsigned long long)want, got == want ? "" : "  MISMATCH");
    if (got != want) return 1;
  }
  // timing: 3 warm-up launches, then 20 timed launches per variant, variants interleaved
  std::vector<float> t[4];
  for (int w = 0; w < 3; ++w)
    for (uint32_t var = 0; var < 4; ++var) launch(var);
  for (int i = 0; i < 20; ++i)
    for (uint32_t var = 0; var < 4; ++var) t[var].push_back(launch(var));
  float med[4];
  for (uint32_t var = 0; var < 4; ++var) {
    std::sort(t[var].begin(), t[var].end());
    med[var] = 0.5f * (t[var][9] + t[var][10]);
  }
  for (uint32_t var = 0; var < 4; ++var) {
    const double bytes = npos * 2.0 + total * 4.0;
    printf("%-8s median %.3f ms  (min %.3f, max %.3f)  %.2fx packed  ids + values %.2f TB/s\n", names[var], med[var],
           t[var].front(), t[var].back(), med[var] / med[0], bytes / (med[var] * 1e-3) / 1e12);
  }
  return 0;
}
