// multi.cu — single-process multi-GPU PageRank behind the C ABI (gb_comm_*, gb_page_rank_multi).
//
// The reference is one process (SURVEY.md §2.3); a Rust host that owns N devices needs the N-GPU sweep
// without torch or NCCL.  One host thread drives all devices: peer access is enabled all-to-all, every
// device gets two full-length out_scores vectors and a control block that all peers can address (unified
// virtual addressing: the peer pointer IS the pointer), and a sweep is gb_pr_shard_step + gb_pr_shard_sync
// enqueued on every device's stream — the sync kernel spins on the peers' arrival flags on the device, so
// the host never waits inside the loop (tolerance 0) and no collective library is involved.  On an NVSwitch
// box whose driver offers multicast objects the next vectors are additionally mapped through one multicast
// address per device (cuMulticast*), so that a finished out_score is ONE store replicated by the switch.
#include <cuda.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include <cub/cub.cuh>

#include "pr_plan.cuh"

struct gb_comm {
  std::vector<int> devs;
  std::vector<cudaStream_t> streams;
  uint32_t n = 0, n_pad = 0;                  // vectors are sized lazily for the first graph
  std::vector<float*> x;                      // per device: 2 * n_pad floats
  std::vector<void*> ctl;                     // per device: control block of gb_pr_shard_sync
  std::vector<float*> scores;                 // per device: n floats (internal order)
  std::vector<double*> err, total_err;        // per device: 1 / 64 doubles
  uint64_t sync_seq = 0;
  // multicast (optional)
  bool multicast = false;
  CUmemGenericAllocationHandle mc_handle = 0;
  std::vector<CUmemGenericAllocationHandle> phys;  // per device physical allocation behind x (VMM path)
  std::vector<CUdeviceptr> mc_va;                  // per device mapping of the multicast object
  size_t vmm_bytes = 0;
};

namespace gb {

// The driver API (virtual memory management + multicast objects) is resolved at run time: the library
// must load on a box without a driver (the CPU-only checks), so it does not link libcuda.
struct DriverApi {
  bool ok = false;
#define GB_DRV(name) decltype(&::name) name = nullptr
  GB_DRV(cuInit);
  GB_DRV(cuDeviceGet);
  GB_DRV(cuDeviceGetAttribute);
  GB_DRV(cuMulticastGetGranularity);
  GB_DRV(cuMulticastCreate);
  GB_DRV(cuMulticastAddDevice);
  GB_DRV(cuMulticastBindMem);
  GB_DRV(cuMemCreate);
  GB_DRV(cuMemAddressReserve);
  GB_DRV(cuMemMap);
  GB_DRV(cuMemSetAccess);
  GB_DRV(cuMemUnmap);
  GB_DRV(cuMemAddressFree);
  GB_DRV(cuMemRelease);
#undef GB_DRV
};
static const DriverApi& driver() {
  static DriverApi api = [] {
    DriverApi a;
    void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return a;
    bool all = true;
#define GB_LOAD(name, sym)                                        \
  a.name = reinterpret_cast<decltype(a.name)>(dlsym(h, sym));     \
  all = all && a.name != nullptr
    GB_LOAD(cuInit, "cuInit");
    GB_LOAD(cuDeviceGet, "cuDeviceGet");
    GB_LOAD(cuDeviceGetAttribute, "cuDeviceGetAttribute");
    GB_LOAD(cuMulticastGetGranularity, "cuMulticastGetGranularity");
    GB_LOAD(cuMulticastCreate, "cuMulticastCreate");
    GB_LOAD(cuMulticastAddDevice, "cuMulticastAddDevice");
    GB_LOAD(cuMulticastBindMem, "cuMulticastBindMem");
    GB_LOAD(cuMemCreate, "cuMemCreate");
    GB_LOAD(cuMemAddressReserve, "cuMemAddressReserve");
    GB_LOAD(cuMemMap, "cuMemMap");
    GB_LOAD(cuMemSetAccess, "cuMemSetAccess");
    GB_LOAD(cuMemUnmap, "cuMemUnmap");
    GB_LOAD(cuMemAddressFree, "cuMemAddressFree");
    GB_LOAD(cuMemRelease, "cuMemRelease");
#undef GB_LOAD
    a.ok = all;
    return a;
  }();
  return api;
}

__global__ void k_add_f32(float* __restrict__ dst, const float* __restrict__ src, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] += src[i];
}

static void comm_release_buffers(gb_comm* c) {
  const DriverApi& D = driver();
  for (size_t i = 0; i < c->devs.size(); ++i) {
    cudaSetDevice(c->devs[i]);
    cudaDeviceSynchronize();
    if (c->multicast && i < c->mc_va.size() && c->mc_va[i]) {
      D.cuMemUnmap(c->mc_va[i], c->vmm_bytes);
      D.cuMemAddressFree(c->mc_va[i], c->vmm_bytes);
    }
    if (i < c->phys.size() && c->phys[i]) {
      if (i < c->x.size() && c->x[i]) {
        D.cuMemUnmap((CUdeviceptr)c->x[i], c->vmm_bytes);
        D.cuMemAddressFree((CUdeviceptr)c->x[i], c->vmm_bytes);
      }
      D.cuMemRelease(c->phys[i]);
    } else if (i < c->x.size() && c->x[i]) {
      cudaFree(c->x[i]);
    }
    if (i < c->ctl.size() && c->ctl[i]) cudaFree(c->ctl[i]);
    if (i < c->scores.size() && c->scores[i]) cudaFree(c->scores[i]);
    if (i < c->err.size() && c->err[i]) cudaFree(c->err[i]);
    if (i < c->total_err.size() && c->total_err[i]) cudaFree(c->total_err[i]);
  }
  if (c->multicast && c->mc_handle) D.cuMemRelease(c->mc_handle);
  c->x.clear();
  c->ctl.clear();
  c->scores.clear();
  c->err.clear();
  c->total_err.clear();
  c->phys.clear();
  c->mc_va.clear();
  c->mc_handle = 0;
  c->multicast = false;
  c->n = c->n_pad = 0;
}

// Tries to back the x vectors with VMM allocations bound to one multicast object.  Any failure leaves
// the communicator on plain cudaMalloc buffers + unicast peer stores (returns false, nothing allocated).
static bool comm_try_multicast(gb_comm* c, size_t bytes_per_dev) {
  const int P = (int)c->devs.size();
  if (P < 2 || getenv("GB_NO_MULTICAST")) return false;
  const DriverApi& D = driver();
  if (!D.ok || D.cuInit(0) != CUDA_SUCCESS) return false;
  for (int d : c->devs) {
    int ok = 0;
    CUdevice dev;
    if (D.cuDeviceGet(&dev, d) != CUDA_SUCCESS) return false;
    if (D.cuDeviceGetAttribute(&ok, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS || !ok) return false;
  }
  CUmulticastObjectProp mp{};
  mp.numDevices = (unsigned)P;
  mp.handleTypes = 0;
  mp.flags = 0;
  size_t gran = 0;
  mp.size = bytes_per_dev;
  if (D.cuMulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || !gran) return false;
  const size_t bytes = (bytes_per_dev + gran - 1) / gran * gran;
  mp.size = bytes;
  CUmemGenericAllocationHandle mc = 0;
  if (D.cuMulticastCreate(&mc, &mp) != CUDA_SUCCESS) return false;
  std::vector<CUmemGenericAllocationHandle> phys(P, 0);
  std::vector<CUdeviceptr> va(P, 0), mva(P, 0);
  bool ok = true;
  for (int i = 0; i < P && ok; ++i) {
    CUdevice dev;
    D.cuDeviceGet(&dev, c->devs[i]);
    ok = D.cuMulticastAddDevice(mc, dev) == CUDA_SUCCESS;
  }
  std::vector<CUmemAccessDesc> access(P);
  for (int i = 0; i < P; ++i) {
    access[i].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    access[i].location.id = c->devs[i];
    access[i].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  }
  for (int i = 0; i < P && ok; ++i) {
    cudaSetDevice(c->devs[i]);
    CUmemAllocationProp ap{};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = c->devs[i];
    ok = D.cuMemCreate(&phys[i], bytes, &ap, 0) == CUDA_SUCCESS;
    ok = ok && D.cuMemAddressReserve(&va[i], bytes, gran, 0, 0) == CUDA_SUCCESS;
    ok = ok && D.cuMemMap(va[i], bytes, 0, phys[i], 0) == CUDA_SUCCESS;
    ok = ok && D.cuMemSetAccess(va[i], bytes, access.data(), (size_t)P) == CUDA_SUCCESS;  // every device may address it
    ok = ok && D.cuMulticastBindMem(mc, 0, phys[i], 0, bytes, 0) == CUDA_SUCCESS;
  }
  for (int i = 0; i < P && ok; ++i) {
    cudaSetDevice(c->devs[i]);
    ok = D.cuMemAddressReserve(&mva[i], bytes, gran, 0, 0) == CUDA_SUCCESS;
    ok = ok && D.cuMemMap(mva[i], bytes, 0, mc, 0) == CUDA_SUCCESS;
    ok = ok && D.cuMemSetAccess(mva[i], bytes, &access[i], 1) == CUDA_SUCCESS;
  }
  if (!ok) {
    for (int i = 0; i < P; ++i) {
      if (mva[i]) {
        D.cuMemUnmap(mva[i], bytes);
        D.cuMemAddressFree(mva[i], bytes);
      }
      if (va[i]) {
        D.cuMemUnmap(va[i], bytes);
        D.cuMemAddressFree(va[i], bytes);
      }
      if (phys[i]) D.cuMemRelease(phys[i]);
    }
    D.cuMemRelease(mc);
    cudaGetLastError();
    return false;
  }
  c->multicast = true;
  c->mc_handle = mc;
  c->phys = phys;
  c->mc_va = mva;
  c->vmm_bytes = bytes;
  c->x.resize(P);
  for (int i = 0; i < P; ++i) c->x[i] = reinterpret_cast<float*>(va[i]);
  return true;
}

static gb_status comm_prepare(gb_comm* c, uint32_t n) {
  const uint32_t P = (uint32_t)c->devs.size();
  const uint32_t grid = 32 * P;
  const uint32_t n_pad = (uint32_t)(((uint64_t)n + grid - 1) / grid * grid);
  if (c->n == n && !c->x.empty()) return GB_OK;
  comm_release_buffers(c);
  c->n = n;
  c->n_pad = n_pad;
  const size_t xbytes = (size_t)2 * n_pad * sizeof(float);
  if (!comm_try_multicast(c, xbytes)) {
    c->x.assign(P, nullptr);
    for (uint32_t i = 0; i < P; ++i) {
      GB_CUDA(cudaSetDevice(c->devs[i]));
      GB_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->x[i]), xbytes));
    }
  }
  c->ctl.assign(P, nullptr);
  c->scores.assign(P, nullptr);
  c->err.assign(P, nullptr);
  c->total_err.assign(P, nullptr);
  for (uint32_t i = 0; i < P; ++i) {
    GB_CUDA(cudaSetDevice(c->devs[i]));
    GB_CUDA(cudaMemset(c->x[i], 0, xbytes));
    GB_CUDA(cudaMalloc(&c->ctl[i], GB_PR_SYNC_BLOCK_BYTES));
    GB_CUDA(cudaMemset(c->ctl[i], 0, GB_PR_SYNC_BLOCK_BYTES));
    GB_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->scores[i]), (size_t)n * sizeof(float)));
    GB_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->err[i]), sizeof(double)));
    GB_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->total_err[i]), 64 * sizeof(double)));
    GB_CUDA(cudaMemset(c->total_err[i], 0, 64 * sizeof(double)));
    GB_CUDA(cudaDeviceSynchronize());
  }
  c->sync_seq = 0;
  return GB_OK;
}

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

// The sweeps of the sharded JACOBI schedule over the communicator, one shard per device (shards[i] on
// devs[i]), and the assembly of the ranks on device 0.  scores, *ran and *error are written only on success.
static gb_status comm_sweeps(gb_comm* c, uint32_t n, const std::vector<gb_pr_shard*>& shards,
                             const gb_page_rank_config* cfg, float* scores, uint64_t* ran, double* error) {
  const uint32_t P = (uint32_t)c->devs.size();
  GB_TRY(comm_prepare(c, n));
  const uint32_t n_pad = c->n_pad;
  for (uint32_t i = 0; i < P; ++i)
    GB_TRY(gb_pr_shard_init(shards[i], cfg->damping_factor, c->x[i], c->x[i] + n_pad, c->scores[i], c->streams[i]));
  // every device has finished its init before anybody's sweep-2 stores could land in its x0
  for (uint32_t i = 0; i < P; ++i) {
    GB_CUDA(cudaSetDevice(c->devs[i]));
    GB_CUDA(cudaStreamSynchronize(c->streams[i]));
  }
  const uint64_t limit = cfg->max_iterations ? cfg->max_iterations : 100000ull;
  const bool can_stop = cfg->tolerance > 0.0;
  uint64_t sweep = 0;
  double total = 0.0;
  std::vector<float*> peers(8, nullptr);
  std::vector<void*> blocks(8, nullptr);
  for (;;) {
    ++sweep;
    const uint32_t cur = (uint32_t)((sweep - 1) & 1), nxt = (uint32_t)(sweep & 1);
    for (uint32_t i = 0; i < P; ++i) {
      uint32_t np = 0;
      for (uint32_t q = 0; q < P; ++q)
        if (q != i) peers[np++] = c->x[q] + (size_t)nxt * n_pad;
      float* mc = c->multicast ? reinterpret_cast<float*>(c->mc_va[i]) + (size_t)nxt * n_pad : nullptr;
      GB_TRY(gb_pr_shard_step(shards[i], cfg->damping_factor, sweep, c->x[i] + (size_t)cur * n_pad,
                              c->x[i] + (size_t)nxt * n_pad, peers.data(), P - 1, P > 1 ? mc : nullptr, c->scores[i],
                              c->err[i], c->streams[i]));
    }
    for (uint32_t i = 0; i < P; ++i) {
      for (uint32_t q = 0; q < P; ++q) blocks[q] = c->ctl[q];
      GB_TRY(gb_pr_shard_sync(shards[i], c->sync_seq + sweep, c->err[i], c->ctl[i], blocks.data(), c->total_err[i],
                              (uint32_t)(sweep % 64), c->streams[i]));
    }
    const bool last = sweep == limit;
    if (can_stop || last) {
      GB_CUDA(cudaSetDevice(c->devs[0]));
      GB_CUDA(cudaMemcpyAsync(&total, c->total_err[0] + (sweep % 64), sizeof(double), cudaMemcpyDeviceToHost,
                              c->streams[0]));
      GB_CUDA(cudaStreamSynchronize(c->streams[0]));
      if ((can_stop && total < cfg->tolerance) || last) break;
    }
  }
  c->sync_seq += sweep;
  *ran = sweep;
  *error = total;
  // every device holds its own rows' scores (zero elsewhere): sum them on device 0, then original ids
  for (uint32_t i = 0; i < P; ++i) {
    GB_CUDA(cudaSetDevice(c->devs[i]));
    GB_CUDA(cudaStreamSynchronize(c->streams[i]));
  }
  GB_CUDA(cudaSetDevice(c->devs[0]));
  float* tmp = c->x[0];  // the out_scores vectors are free again: staging for the peers' score vectors
  for (uint32_t q = 1; q < P; ++q) {
    GB_CUDA(cudaMemcpyPeerAsync(tmp, c->devs[0], c->scores[q], c->devs[q], (size_t)n * sizeof(float), c->streams[0]));
    k_add_f32<<<grid_for(n, 256), 256, 0, c->streams[0]>>>(c->scores[0], tmp, n);
  }
  GB_TRY(gb_pr_shard_finish(shards[0], c->scores[0], tmp, c->streams[0]));
  GB_CUDA(cudaMemcpyAsync(scores, tmp, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->streams[0]));
  GB_CUDA(cudaStreamSynchronize(c->streams[0]));
  return GB_OK;
}

// ---- shards from a host in-CSR (gb_pr_shards_csr_u32) ----------------------------------------------------
// Rank r's in-degree of every original row, 0 for the rows another rank owns (the deal of 32-row slices of the
// internal order over U ranks); entry n is 0, so that an exclusive scan gives the local offsets
__global__ void k_pr_owned_deg(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ new_id, uint32_t n,
                               uint32_t U, uint32_t r, uint32_t* __restrict__ deg) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += gridDim.x * blockDim.x)
    deg[v] = v < n && (new_id[v] >> 5) % U == r ? in_off[v + 1] - in_off[v] : 0u;
}

constexpr uint32_t GATHER_ILP = 8;  // 32-entry loads in flight per warp while it copies one row
// One landed chunk of one part, rows [v0, v1) of the original order: a warp takes 32 consecutive rows, ballots
// those rank r owns and copies each with the whole warp, 32 entries per step, from the part's targets (a peer
// pointer when the part lives on another device; part_tgt[0] is edge part_e0) to loc_tgt + loc_off[v].  Every
// copied target is checked against n; a warp adds its count of bad ones to *bad once.
__global__ void __launch_bounds__(256) k_pr_gather_rows(const uint32_t* __restrict__ in_off,
                                                        const uint32_t* __restrict__ part_tgt, uint64_t part_e0,
                                                        uint32_t v0, uint32_t v1, const uint32_t* __restrict__ new_id,
                                                        uint32_t U, uint32_t r, const uint32_t* __restrict__ loc_off,
                                                        uint32_t* __restrict__ loc_tgt, uint32_t n,
                                                        unsigned int* __restrict__ bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t nbad = 0;
  for (uint64_t base = (uint64_t)v0 + 32ull * warp; base < v1; base += 32ull * nwarps) {
    const uint64_t v = base + lane;
    uint32_t b0 = 0, d = 0, dst = 0;
    if (v < v1 && (new_id[v] >> 5) % U == r) {
      b0 = in_off[v];
      d = in_off[v + 1] - b0;
      dst = loc_off[v];
    }
    uint32_t todo = __ballot_sync(0xFFFFFFFFu, d != 0);
    while (todo) {
      const int src_lane = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t rb = __shfl_sync(0xFFFFFFFFu, b0, src_lane);
      const uint32_t rd = __shfl_sync(0xFFFFFFFFu, d, src_lane);
      const uint32_t rdst = __shfl_sync(0xFFFFFFFFu, dst, src_lane);
      const uint32_t* __restrict__ from = part_tgt + (rb - part_e0);
      uint32_t* __restrict__ to = loc_tgt + rdst;
      for (uint64_t i = lane; i < rd; i += 32 * GATHER_ILP) {
        uint32_t t[GATHER_ILP];
#pragma unroll
        for (uint32_t u = 0; u < GATHER_ILP; ++u) t[u] = i + 32 * u < rd ? from[i + 32 * u] : 0u;
#pragma unroll
        for (uint32_t u = 0; u < GATHER_ILP; ++u)
          if (i + 32 * u < rd) {
            nbad += t[u] >= n;
            to[i + 32 * u] = t[u];
          }
      }
    }
  }
  nbad = __reduce_add_sync(0xFFFFFFFFu, nbad);
  if (lane == 0 && nbad) atomicAdd(bad, nbad);
}

constexpr uint64_t PR_PART_CHUNK_EDGES = 1u << 23;  // 32 MiB of targets per chunk (GB_PR_PART_CHUNK_EDGES)

// One rank r on device dev: the full offsets gathered from the parts, the order stage of its layout, and the
// compact local in-CSR of the rows it owns (loc_off by original id, loc_tgt in CSR order).  A lone rank needs
// neither the gathered offsets nor the local CSR: its part is all of them.
struct PrCsrRank {
  int dev = -1;
  cudaStream_t s = nullptr;
  PeerBuf in_off, out_off;     // [n + 1] each
  LayoutBuild* build = nullptr;
  PrPlan* plan = nullptr;      // the finished layout, until the caller takes it
  DevBuf<uint32_t> loc_off, loc_tgt;
  uint64_t entries = 0;        // loc_off[n]
  DevBuf<unsigned int> bad;    // [0] in rows whose offsets decrease, [1] out rows, [2] targets >= n
  unsigned int h_bad[3] = {0, 0, 0};
  ~PrCsrRank() {
    if (dev < 0) return;
    cudaSetDevice(dev);
    if (s) cudaStreamSynchronize(s);
    layout_free(build);
    free_pr_plan(plan);
    loc_tgt.release();
    loc_off.release();
    bad.release();
    out_off.release();
    in_off.release();
    if (s) cudaStreamDestroy(s);
  }
};

gb_status check_pr_host_csr(uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt, const uint32_t* out_off) {
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GB_REQUIRE(in_off && out_off, "offset arrays are NULL");
  GB_REQUIRE(in_off[n] == out_off[n], "in and out offsets disagree on the edge count");
  GB_TRY(require_host_csr(n, in_off, in_tgt, "in"));
  return require_host_csr(n, out_off, nullptr, "out", true);
}

gb_status pr_csr_plans(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                       const uint32_t* in_tgt, const uint32_t* out_off, uint64_t chunk_edges,
                       std::vector<PrPlan*>* plans) {
  const uint64_t m = in_off[n];
  const uint32_t U = (uint32_t)devs.size() * V;
  const bool peers = U > 1;
  const std::vector<PrPart> split = pr_split(in_off, n, U, chunk_edges);
  DeviceGuard guard(devs[0]);
  // declared after the parts, the ranks go first on any return, and each drains its stream as it goes: the
  // gathers and a lone rank's layout read the parts
  std::vector<std::unique_ptr<CsrFeed>> parts;
  std::vector<std::unique_ptr<PrCsrRank>> ranks;
  // 1. every part's in and out offsets, then its targets chunk by chunk, round robin over the parts: the copies go
  // out before the host waits for any check, so every bus is busy from the start
  uint32_t max_chunks = 0;
  for (uint32_t u = 0; u < U; ++u) {
    parts.emplace_back(new (std::nothrow) CsrFeed());
    GB_REQUIRE(parts.back() != nullptr, "host allocation failed");
    CsrFeed& q = *parts.back();
    GB_TRY(q.open(devs[u / V], split[u].r_begin, split[u].r_end, peers, true));
    GB_TRY(q.resident(split[u].e_begin, split[u].e_end, split[u].chunks.count(), peers));
    GB_TRY(q.send_offsets(in_off, out_off));
    max_chunks = std::max(max_chunks, split[u].chunks.count());
  }
  for (uint32_t k = 0; k < max_chunks; ++k)
    for (uint32_t u = 0; u < U; ++u) {
      const CsrChunks& ch = split[u].chunks;
      if (k >= ch.count()) continue;
      GB_CUDA(cudaSetDevice(parts[u]->dev));
      GB_TRY(parts[u]->send(k, in_tgt, ch.edge[k], ch.edge[k + 1] - ch.edge[k]));
    }
  // 2. rank u checks part u's rows (the slices tile [0, n]: every row once, whatever the host arrays hold), and
  // with several ranks every rank assembles the full offsets from the parts
  for (uint32_t r = 0; r < U; ++r) {
    ranks.emplace_back(new (std::nothrow) PrCsrRank());
    GB_REQUIRE(ranks.back() != nullptr, "host allocation failed");
    PrCsrRank& k = *ranks.back();
    k.dev = devs[r / V];
    GB_CUDA(cudaSetDevice(k.dev));
    GB_CUDA(cudaStreamCreateWithFlags(&k.s, cudaStreamNonBlocking));
    GB_TRY(k.bad.alloc(3));
    GB_CUDA(cudaMemsetAsync(k.bad.p, 0, 12, k.s));
    GB_TRY(parts[r]->check_monotone(k.s, split[r].r_begin, split[r].r_end, k.bad.p));
    GB_CUDA(cudaMemcpyAsync(k.h_bad, k.bad.p, 8, cudaMemcpyDeviceToHost, k.s));
    if (!peers) continue;
    GB_TRY(k.in_off.alloc((size_t)n + 1, peers));
    GB_TRY(k.out_off.alloc((size_t)n + 1, peers));
    for (uint32_t u = 0; u < U; ++u) {
      const CsrFeed& q = *parts[u];
      const size_t count = (size_t)(q.r_end - q.r_begin) + (u + 1 == U ? 1 : 0);
      if (!count) continue;
      GB_CUDA(cudaStreamWaitEvent(k.s, q.offsets_in, 0));
      GB_CUDA(cudaMemcpyPeerAsync(k.in_off.p + q.r_begin, k.dev, q.off.p, q.dev, count * 4, k.s));
      GB_CUDA(cudaMemcpyPeerAsync(k.out_off.p + q.r_begin, k.dev, q.off2.p, q.dev, count * 4, k.s));
    }
  }
  unsigned int nbad[2] = {0, 0};
  for (auto& k : ranks) {
    GB_CUDA(cudaSetDevice(k->dev));
    GB_CUDA(cudaStreamSynchronize(k->s));
    nbad[0] += k->h_bad[0];
    nbad[1] += k->h_bad[1];
  }
  GB_TRY(require_monotone("in", nbad[0]));
  GB_TRY(require_monotone("out", nbad[1]));
  // 3. order stage.  A lone rank owns every row: its part is its in-CSR, whose chunks the layout build checks
  // and classifies as they land.  Otherwise the local offsets, and the gathers of every chunk as it lands.
  for (uint32_t r = 0; r < U; ++r) {
    PrCsrRank& k = *ranks[r];
    GB_CUDA(cudaSetDevice(k.dev));
    PrSource src;
    src.device = k.dev;
    src.stream = k.s;
    src.n = n;
    src.m = m;
    src.in_off = peers ? k.in_off.p : parts[0]->off.p;
    src.out_off = peers ? k.out_off.p : parts[0]->off2.p;
    src.feed = peers ? nullptr : parts[0].get();
    src.chunks = peers ? nullptr : &split[0].chunks;
    PrDeal deal;
    deal.P = U;
    deal.p = r;
    GB_TRY(layout_begin(src, deal, &k.build));
    if (!peers) {
      LayoutBuild* b = k.build;
      k.build = nullptr;
      GB_TRY(layout_end(b, src.in_off, parts[0]->tgt.p, m, &k.plan));
      continue;
    }
    const uint32_t* new_id = layout_new_id(k.build);
    {
      DevBufStreamScope scope(k.s);  // the copy streams may still be busy: release waits for this stream only
      GB_TRY(k.loc_off.alloc((size_t)n + 1));
      k_pr_owned_deg<<<grid_for((uint64_t)n + 1, 256), 256, 0, k.s>>>(k.in_off.p, new_id, n, U, r, k.loc_off.p);
      DevBuf<uint8_t> tmp;
      GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
        return cub::DeviceScan::ExclusiveSum(t, tb, k.loc_off.p, k.loc_off.p, (int)(n + 1), k.s);
      }));
      uint32_t total = 0;
      GB_CUDA(cudaMemcpyAsync(&total, k.loc_off.p + n, 4, cudaMemcpyDeviceToHost, k.s));
      GB_CUDA(cudaStreamSynchronize(k.s));
      k.entries = total;
      GB_TRY(k.loc_tgt.alloc(std::max<uint64_t>(k.entries, 1)));
    }
    for (uint32_t c = 0; c < max_chunks; ++c)
      for (uint32_t u = 0; u < U; ++u) {
        const CsrChunks& ch = split[u].chunks;
        if (c >= ch.count()) continue;
        const uint32_t v0 = ch.row[c], v1 = ch.row[c + 1];
        if (v1 == v0) continue;
        GB_CUDA(cudaStreamWaitEvent(k.s, parts[u]->landed[c], 0));
        k_pr_gather_rows<<<grid_for((uint64_t)(v1 - v0), 256), 256, 0, k.s>>>(
            k.in_off.p, parts[u]->tgt.p, split[u].e_begin, v0, v1, new_id, U, r, k.loc_off.p, k.loc_tgt.p, n,
            k.bad.p + 2);
      }
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaMemcpyAsync(k.h_bad + 2, k.bad.p + 2, 4, cudaMemcpyDeviceToHost, k.s));
  }
  if (peers) {
    unsigned int nbad_tgt = 0;
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      GB_CUDA(cudaStreamSynchronize(k->s));
      nbad_tgt += k->h_bad[2];
    }
    GB_TRY(require_ids("in", nbad_tgt, n));
    // 4. every rank has gathered: the parts and the full offsets go (the order stage has read the degrees), and
    // each rank builds its layout from its local CSR, which goes too
    parts.clear();
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      k->in_off.release();
      k->out_off.release();
    }
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      LayoutBuild* b = k->build;
      k->build = nullptr;
      GB_TRY(layout_end(b, k->loc_off.p, k->loc_tgt.p, k->entries, &k->plan));
      DevBufStreamScope scope(k->s);
      k->loc_tgt.release();
      k->loc_off.release();
    }
  }
  plans->clear();
  for (auto& k : ranks) {
    plans->push_back(k->plan);
    k->plan = nullptr;
  }
  return GB_OK;
}

// The shards of ranks 0 .. U-1 (U = devs.size() * V, rank r on devs[r / V]) of a host in-CSR: shards (U entries)
// are the caller's to free.
static gb_status pr_csr_shards(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                               const uint32_t* in_tgt, const uint32_t* out_off, std::vector<gb_pr_shard*>& shards) {
  GB_TRY(check_pr_host_csr(n, in_off, in_tgt, out_off));
  GB_REQUIRE(n < 0x7FFFFFFFu, "node_count %u: the local offsets are scanned in one pass of < 2^31 items", n);
  const uint64_t chunk_edges = std::max<uint64_t>((uint32_t)env_u64("GB_PR_PART_CHUNK_EDGES", PR_PART_CHUNK_EDGES), 1);
  std::vector<PrPlan*> plans;
  GB_TRY(pr_csr_plans(devs, V, n, in_off, in_tgt, out_off, chunk_edges, &plans));
  gb_status st = GB_OK;
  for (size_t r = 0; r < plans.size(); ++r) {  // shard_from_plan takes its plan, whatever it returns
    if (st == GB_OK) {
      st = shard_from_plan(devs[r / V], plans[r], &shards[r]);
    } else {
      DeviceGuard guard(devs[r / V]);
      free_pr_plan(plans[r]);
    }
  }
  return st;
}

const std::vector<int>& comm_devices(const gb_comm* c) { return c->devs; }

}  // namespace gb

extern "C" {

gb_status gb_comm_init(int ndev, const int* devices, gb_comm** comm) {
  GB_REQUIRE(comm != nullptr, "comm is NULL");
  GB_REQUIRE(ndev >= 1 && ndev <= 8, "a communicator spans 1..8 devices");
  int count = 0;
  GB_CUDA(cudaGetDeviceCount(&count));
  gb_comm* c = new (std::nothrow) gb_comm();
  if (!c) return gb::fail(GB_ERR_OOM, "host allocation failed");
  for (int i = 0; i < ndev; ++i) {
    const int d = devices ? devices[i] : i;
    if (d < 0 || d >= count || std::find(c->devs.begin(), c->devs.end(), d) != c->devs.end()) {
      delete c;
      return gb::fail(GB_ERR_INVALID, "bad or repeated device %d (the box has %d)", d, count);
    }
    c->devs.push_back(d);
  }
  int prev = 0;
  cudaGetDevice(&prev);
  gb_status st = [&]() -> gb_status {
    for (int a : c->devs)
      for (int b : c->devs) {
        if (a == b) continue;
        int can = 0;
        GB_CUDA(cudaDeviceCanAccessPeer(&can, a, b));
        GB_REQUIRE(can, "device %d cannot address device %d (no peer access)", a, b);
        GB_CUDA(cudaSetDevice(a));
        cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else GB_CUDA(e);
      }
    for (int d : c->devs) {
      GB_CUDA(cudaSetDevice(d));
      cudaStream_t s = nullptr;
      GB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      c->streams.push_back(s);
    }
    return GB_OK;
  }();
  cudaSetDevice(prev);
  if (st != GB_OK) {
    gb_comm_free(c);
    return st;
  }
  *comm = c;
  return GB_OK;
}

gb_status gb_comm_free(gb_comm* c) {
  if (!c) return GB_OK;
  int prev = 0;
  cudaGetDevice(&prev);
  gb::comm_release_buffers(c);
  for (size_t i = 0; i < c->streams.size(); ++i) {
    cudaSetDevice(c->devs[i]);
    cudaStreamDestroy(c->streams[i]);
  }
  cudaSetDevice(prev);
  delete c;
  return GB_OK;
}

gb_status gb_comm_info(const gb_comm* c, int* ndev, int* multicast) {
  GB_REQUIRE(c, "NULL argument");
  if (ndev) *ndev = (int)c->devs.size();
  if (multicast) *multicast = c->multicast ? 1 : 0;
  return GB_OK;
}

gb_status gb_page_rank_multi(gb_comm* c, const gb_graph* const* graphs, const gb_page_rank_config* cfg,
                             float* scores, uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(c && graphs && cfg && scores && ran_iterations && error, "NULL argument");
  GB_REQUIRE(!(cfg->max_iterations == 0 && !(cfg->tolerance > 0.0)),
             "max_iterations == 0 with tolerance <= 0 never terminates (page_rank.rs:107)");
  const uint32_t P = (uint32_t)c->devs.size();
  gb_graph_info info0{};
  for (uint32_t i = 0; i < P; ++i) {
    GB_REQUIRE(graphs[i] != nullptr, "graphs[%u] is NULL", i);
    gb_graph_info gi{};
    GB_TRY(gb_graph_get_info(graphs[i], &gi));
    GB_REQUIRE(gi.device == c->devs[i], "graphs[%u] lives on device %d, the communicator's device %u is %d", i,
               gi.device, i, c->devs[i]);
    if (i == 0) info0 = gi;
    GB_REQUIRE(gi.node_count == info0.node_count && gi.edge_count == info0.edge_count,
               "graphs[%u] is not the same graph as graphs[0]", i);
  }
  const uint32_t n = info0.node_count;
  int prev = 0;
  cudaGetDevice(&prev);
  gb::ShardSet shards(P);
  gb_status st = [&]() -> gb_status {
    for (uint32_t i = 0; i < P; ++i) GB_TRY(gb_pr_shard_create(graphs[i], i, P, &shards.v[i]));
    return gb::comm_sweeps(c, n, shards.v, cfg, scores, ran_iterations, error);
  }();
  shards.clear();
  cudaSetDevice(prev);
  return st;
}

gb_status gb_pr_shards_csr_u32(gb_comm* c, uint32_t ranks_per_device, uint32_t n, const uint32_t* in_off,
                               const uint32_t* in_tgt, const uint32_t* out_off, gb_pr_shard** shards) {
  GB_REQUIRE(c != nullptr, "comm is NULL");
  GB_REQUIRE(shards != nullptr, "shards is NULL");
  GB_REQUIRE(ranks_per_device >= 1, "ranks_per_device must be >= 1");
  const uint64_t U = (uint64_t)c->devs.size() * ranks_per_device;
  GB_REQUIRE(U <= 8, "%zu devices x %u ranks per device: at most 8 ranks", c->devs.size(), ranks_per_device);
  gb::ShardSet set((uint32_t)U);
  GB_TRY(gb::pr_csr_shards(c->devs, ranks_per_device, n, in_off, in_tgt, out_off, set.v));
  for (uint32_t r = 0; r < U; ++r) shards[r] = set.v[r];
  set.v.clear();
  return GB_OK;
}

gb_status gb_page_rank_csr_multi_u32(gb_comm* c, uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt,
                                     const uint32_t* out_off, const gb_page_rank_config* cfg, float* scores,
                                     uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(c != nullptr, "comm is NULL");
  GB_REQUIRE(scores != nullptr, "scores is NULL");
  GB_REQUIRE(cfg && ran_iterations && error, "NULL argument");
  GB_REQUIRE(!(cfg->max_iterations == 0 && !(cfg->tolerance > 0.0)),
             "max_iterations == 0 with tolerance <= 0 never terminates (page_rank.rs:107)");
  const uint32_t P = (uint32_t)c->devs.size();
  int prev = 0;
  cudaGetDevice(&prev);
  gb::ShardSet shards(P);
  gb_status st = [&]() -> gb_status {
    GB_TRY(gb::pr_csr_shards(c->devs, 1, n, in_off, in_tgt, out_off, shards.v));
    return gb::comm_sweeps(c, n, shards.v, cfg, scores, ran_iterations, error);
  }();
  shards.clear();
  cudaSetDevice(prev);
  return st;
}

}  // extern "C"
