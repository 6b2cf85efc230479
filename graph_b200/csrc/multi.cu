// multi.cu — the communicator: the devices of one process, their streams and peer-addressable sweep buffers
// (gb_comm_*), and the PageRank calls that sweep over them (gb_page_rank_multi, gb_page_rank_csr_multi_u32).
// Where the shards of a call come from is not decided here: resident graphs give them through
// gb_pr_shard_create (pagerank.cu), a host CSR through pr_csr_shards (pr_csr.cu).
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

#include "pr_plan.cuh"

struct gb_comm {
  std::vector<int> devs;
  std::vector<cudaStream_t> streams;
  // held by a PageRank call from its shard fill through the copy of the scores: the buffers below, which
  // comm_prepare frees and reallocates for another n, and sync_seq are one call's at a time
  mutable std::mutex mu;
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
  const uint64_t limit = pr_sweep_limit(cfg);
  const bool can_stop = cfg->tolerance > 0.0;
  uint64_t sweep = 0;
  double total = 0.0;
  // peers[nxt][i]: buffer nxt of every device but devs[i], in device order (a communicator spans at most 8)
  float* peers[2][8][8] = {};
  void* blocks[8] = {};
  for (uint32_t q = 0; q < P; ++q) blocks[q] = c->ctl[q];
  for (uint32_t nxt = 0; nxt < 2; ++nxt)
    for (uint32_t i = 0; i < P; ++i) {
      uint32_t np = 0;
      for (uint32_t q = 0; q < P; ++q)
        if (q != i) peers[nxt][i][np++] = c->x[q] + (size_t)nxt * n_pad;
    }
  for (;;) {
    ++sweep;
    const uint32_t cur = (uint32_t)((sweep - 1) & 1), nxt = (uint32_t)(sweep & 1);
    for (uint32_t i = 0; i < P; ++i) {
      float* mc = c->multicast ? reinterpret_cast<float*>(c->mc_va[i]) + (size_t)nxt * n_pad : nullptr;
      GB_TRY(gb_pr_shard_step(shards[i], cfg->damping_factor, sweep, c->x[i] + (size_t)cur * n_pad,
                              c->x[i] + (size_t)nxt * n_pad, peers[nxt][i], P - 1, P > 1 ? mc : nullptr,
                              c->scores[i], c->err[i], c->streams[i]));
    }
    for (uint32_t i = 0; i < P; ++i)
      GB_TRY(gb_pr_shard_sync(shards[i], c->sync_seq + sweep, c->err[i], c->ctl[i], blocks, c->total_err[i],
                              (uint32_t)(sweep % 64), c->streams[i]));
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

// One PageRank call over the communicator: fill(shards) makes the P shards (shards[i] on devs[i]), comm_sweeps
// runs them, and the shards go before the caller's device is current again, whatever either returned.  Calls
// on one communicator run one after the other, on its lock.
template <class Fill>
static gb_status comm_page_rank(gb_comm* c, uint32_t n, const gb_page_rank_config* cfg, float* scores, uint64_t* ran,
                                double* error, Fill fill) {
  DeviceGuard guard(c->devs[0]);  // fill and comm_sweeps move from device to device
  std::lock_guard<std::mutex> lock(c->mu);
  ShardSet shards((uint32_t)c->devs.size());
  GB_TRY(fill(shards.v));
  return comm_sweeps(c, n, shards.v, cfg, scores, ran, error);
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
  gb::DeviceGuard guard(c->devs[0]);
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
  if (st != GB_OK) {
    gb_comm_free(c);
    return st;
  }
  *comm = c;
  return GB_OK;
}

gb_status gb_comm_free(gb_comm* c) {
  if (!c) return GB_OK;
  gb::DeviceGuard guard(c->devs[0]);
  gb::comm_release_buffers(c);
  for (size_t i = 0; i < c->streams.size(); ++i) {
    cudaSetDevice(c->devs[i]);
    cudaStreamDestroy(c->streams[i]);
  }
  delete c;
  return GB_OK;
}

gb_status gb_comm_info(const gb_comm* c, int* ndev, int* multicast) {
  GB_REQUIRE(c, "NULL argument");
  std::lock_guard<std::mutex> lock(c->mu);  // comm_prepare sets multicast
  if (ndev) *ndev = (int)c->devs.size();
  if (multicast) *multicast = c->multicast ? 1 : 0;
  return GB_OK;
}

gb_status gb_page_rank_multi(gb_comm* c, const gb_graph* const* graphs, const gb_page_rank_config* cfg,
                             float* scores, uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(c && graphs && cfg && scores && ran_iterations && error, "NULL argument");
  GB_TRY(gb::require_pr_config(cfg));
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
  auto from_graphs = [&](std::vector<gb_pr_shard*>& shards) -> gb_status {
    for (uint32_t i = 0; i < P; ++i) GB_TRY(gb_pr_shard_create(graphs[i], i, P, &shards[i]));
    return GB_OK;
  };
  return gb::comm_page_rank(c, info0.node_count, cfg, scores, ran_iterations, error, from_graphs);
}

gb_status gb_page_rank_csr_multi_u32(gb_comm* c, uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt,
                                     const uint32_t* out_off, const gb_page_rank_config* cfg, float* scores,
                                     uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(c != nullptr, "comm is NULL");
  GB_REQUIRE(scores != nullptr, "scores is NULL");
  GB_REQUIRE(cfg && ran_iterations && error, "NULL argument");
  GB_TRY(gb::require_pr_config(cfg));
  return gb::comm_page_rank(c, n, cfg, scores, ran_iterations, error, [&](std::vector<gb_pr_shard*>& shards) {
    return gb::pr_csr_shards(c->devs, 1, n, in_off, in_tgt, out_off, shards);
  });
}

}  // extern "C"
