// Random-access ceiling of HBM on this GPU: every thread issues U independent loads of `BYTES` bytes at hashed,
// BYTES-aligned offsets of a table of T bytes, over and over.  Prints effective GB/s (useful bytes) per configuration:
// the roofline of the hash-table look-ups of k_rows (one 64-byte bucket per off-diagonal term).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 tools/random_access.cu -o /tmp/random_access && /tmp/random_access
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t mix(uint64_t x) {
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

template <int BYTES, int U>
__global__ void k_random(const uint4 *__restrict__ table, uint64_t n_slots, int iters, uint64_t *sink) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t acc = 0, state = tid * 0x9E3779B97F4A7C15ull + 1;
  for (int it = 0; it < iters; ++it) {
    uint4 v[U][BYTES / 16];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      state = mix(state + u);
      const uint64_t slot = (uint64_t)(((state >> 32) * n_slots) >> 32);
#pragma unroll
      for (int c = 0; c < BYTES / 16; ++c) v[u][c] = __ldg(table + slot * (BYTES / 16) + c);
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int c = 0; c < BYTES / 16; ++c) acc += v[u][c].x ^ v[u][c].w;
  }
  if (acc == 0x1234567) *sink = acc;
}

template <int BYTES, int U>
void run(const uint4 *table, size_t table_bytes, int blocks_per_sm, uint64_t *sink) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int blocks = sms * blocks_per_sm, threads = 256, iters = 64;
  const uint64_t n_slots = table_bytes / BYTES;
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  k_random<BYTES, U><<<blocks, threads>>>(table, n_slots, 4, sink);
  cudaEventRecord(a);
  k_random<BYTES, U><<<blocks, threads>>>(table, n_slots, iters, sink);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  const double loads = (double)blocks * threads * iters * U;
  printf("table %6.0f MB  access %3d B  %d in flight/thread  %2d CTAs/SM : %7.1f G accesses/s  %7.1f GB/s useful\n",
         table_bytes / 1048576.0, BYTES, U, blocks_per_sm, loads / ms / 1e6, loads * BYTES / ms / 1e6);
}

int main() {
  uint64_t *sink;
  cudaMalloc(&sink, 8);
  for (size_t mb : {256ul, 1024ul, 4096ul, 16384ul}) {
    uint4 *table;
    if (cudaMalloc(&table, mb << 20) != cudaSuccess) { printf("alloc %zu MB failed\n", mb); continue; }
    cudaMemset(table, 1, mb << 20);
    run<16, 4>(table, mb << 20, 8, sink);
    run<32, 4>(table, mb << 20, 8, sink);
    run<64, 2>(table, mb << 20, 2, sink);
    run<64, 4>(table, mb << 20, 2, sink);
    run<64, 4>(table, mb << 20, 8, sink);
    run<64, 8>(table, mb << 20, 8, sink);
    run<128, 4>(table, mb << 20, 8, sink);
    cudaFree(table);
  }
  return 0;
}
