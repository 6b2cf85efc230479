// gather_ceiling.cu — what does an H100 SM sustain for divergent 4-byte gathers?
// Measures random gathers from an f32 table (16 MiB: L2 resident; 256 MiB: larger than L2) through
// (a) ld.global.nc, (b) tex1Dfetch, (c) half/half, (d) cp.async 4-byte global->shared, at several
// occupancies.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_ceiling gather_ceiling.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s failed: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}

template <int MODE, int UNROLL>
__global__ void k_gather(const float* __restrict__ table, cudaTextureObject_t tex, const uint32_t* __restrict__ idx,
                         uint64_t count, float* out) {
  extern __shared__ float sm[];
  const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  float acc = 0.0f;
  for (uint64_t base = tid; base + (UNROLL - 1) * nthreads < count; base += UNROLL * nthreads) {
    uint32_t t[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) t[u] = idx[base + u * nthreads];
    float v[UNROLL];
    if (MODE == 3) {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        uint32_t saddr = (uint32_t)__cvta_generic_to_shared(sm + threadIdx.x + u * blockDim.x);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(saddr), "l"(table + t[u]));
      }
      asm volatile("cp.async.commit_group;");
      asm volatile("cp.async.wait_group 0;");
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) v[u] = sm[threadIdx.x + u * blockDim.x];
    } else {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (MODE == 0) v[u] = __ldg(table + t[u]);
        else if (MODE == 1) v[u] = tex1Dfetch<float>(tex, (int)t[u]);
        else v[u] = (u & 1) ? tex1Dfetch<float>(tex, (int)t[u]) : __ldg(table + t[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) acc += v[u];
  }
  if (acc == 123.456f) out[0] = acc;
}

template <int MODE>
void run(const char* name, const float* table, cudaTextureObject_t tex, const uint32_t* idx, uint64_t count, float* out,
         int threads, int blocks_per_sm) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int grid = sms * blocks_per_sm;
  size_t smem = (MODE == 3) ? (size_t)threads * 8 * 4 : 0;
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(k_gather<MODE, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int w = 0; w < 2; ++w) k_gather<MODE, 8><<<grid, threads, smem>>>(table, tex, idx, count, out);
  CK(cudaDeviceSynchronize());
  cudaEventRecord(e0);
  const int reps = 5;
  for (int r = 0; r < reps; ++r) k_gather<MODE, 8><<<grid, threads, smem>>>(table, tex, idx, count, out);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= reps;
  double gps = count / (ms * 1e-3) / 1e9;
  int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  printf("%-10s threads/SM=%5d  %8.3f ms  %7.1f Ggathers/s  %.3f gathers/clk/SM (at %d MHz)\n", name, threads * blocks_per_sm,
         ms, gps, gps * 1e9 / sms / (clk * 1e3), clk / 1000);
}

__global__ void k_fill_idx(uint32_t* idx, uint64_t count, uint32_t mask) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
    idx[i] = hash32((uint32_t)i * 2654435761u + 12345u) & mask;
}

int main() {
  const uint64_t count = 1ull << 28;  // 268M gathers per launch
  uint32_t* idx; float* out;
  CK(cudaMalloc(&idx, count * 4)); CK(cudaMalloc(&out, 4));
  for (int log_n : {22, 26}) {
    const uint64_t n = 1ull << log_n;
    float* table; CK(cudaMalloc(&table, n * 4)); CK(cudaMemset(table, 0, n * 4));
    k_fill_idx<<<132 * 8, 256>>>(idx, count, (uint32_t)(n - 1));
    cudaResourceDesc rd{}; rd.resType = cudaResourceTypeLinear; rd.res.linear.devPtr = table;
    rd.res.linear.desc = cudaCreateChannelDesc<float>(); rd.res.linear.sizeInBytes = n * 4;
    cudaTextureDesc td{}; td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex; CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));
    printf("---- table %llu MiB (2^%d f32) ----\n", (unsigned long long)(n * 4 >> 20), log_n);
    for (int bps : {1, 2}) {
      run<0>("ldg", table, tex, idx, count, out, 1024, bps);
      run<1>("tex", table, tex, idx, count, out, 1024, bps);
      run<2>("ldg+tex", table, tex, idx, count, out, 1024, bps);
      run<3>("cp.async", table, tex, idx, count, out, 1024, bps);
    }
    run<0>("ldg", table, tex, idx, count, out, 512, 1);
    cudaDestroyTextureObject(tex); cudaFree(table);
  }
  return 0;
}
