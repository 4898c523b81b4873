// Random-access ceiling of HBM and of the L2 on this GPU, in three parts.
//  1. every thread issues U independent loads of `BYTES` bytes at hashed, BYTES-aligned offsets of a table of T bytes,
//     over and over.  Prints effective GB/s (useful bytes) per configuration: the roofline of the hash-table look-ups
//     of k_rows (one 32-byte bucket per off-diagonal term) when they miss the L2.
//  2. the same at 32 bytes on tables that fit the L2 (8, 16, 32 MB): the rate of random sectors that HIT.
//  3. a model of k_rows on its ordered table: 2^24 rows walked like k_rows walks them (one row per lane, tiles of 32 rows
//     strided over the grid, two CTAs per SM), 36 look-ups per row into a 4 GB table of 8 sectors per row of which one is
//     occupied.  A look-up is NEAR with a given probability (the sector of a row within a window of W MB of table
//     around the lane's own row, so the window slides through the table as the rows advance) and FAR otherwise (the
//     sector of any row).  Each combination runs with four treatments of the loads: no hint; an evict_normal policy on
//     both (the hinted instruction, default behaviour); far evict_first, near evict_normal; far evict_first, near
//     evict_last.  Prints look-ups/s.  Per-instruction policies only (createpolicy + ld ... .L2::cache_hint): nothing
//     device-wide is set.
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
void run(const uint4 *table, size_t table_bytes, int blocks_per_sm, uint64_t *sink, int iters = 64) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int blocks = sms * blocks_per_sm, threads = 256;
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

// ---- part 3: the model of k_rows on its ordered table
enum Policy { kNormal = 0, kFirst = 1, kLast = 2 };
constexpr int kTerms = 36;          // look-ups per row
constexpr int kRowBits = 24;        // rows; the table has 8 sectors of 32 bytes per row (4 GB), one of them occupied

__device__ __forceinline__ uint64_t make_policy(int kind) {
  uint64_t p;
  if (kind == kFirst) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  else if (kind == kLast) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// one 32-byte sector as two 128-bit loads, not allocated in L1: the bucket load of k_rows, without and with a policy
__device__ __forceinline__ uint64_t load_sector(const unsigned char *q) {
  uint64_t a, b, c, d;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(q));
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2+16];" : "=l"(c), "=l"(d) : "l"(q));
  return a ^ b ^ c ^ d;
}
__device__ __forceinline__ uint64_t load_sector(const unsigned char *q, uint64_t policy) {
  uint64_t a, b, c, d;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;"
               : "=l"(a), "=l"(b) : "l"(q), "l"(policy));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2+16], %3;"
               : "=l"(c), "=l"(d) : "l"(q), "l"(policy));
  return a ^ b ^ c ^ d;
}

// near_per_256: look-ups out of 256 that are near; window_rows: width of the near window in rows (8 sectors each)
template <bool HINT>
__global__ void __launch_bounds__(256, 2) k_mixed(const unsigned char *__restrict__ table, uint32_t near_per_256,
                                                   int64_t window_rows, int far_kind, int near_kind, uint64_t *sink) {
  const int64_t n_rows = (int64_t)1 << kRowBits;
  const uint64_t far_policy = make_policy(far_kind), near_policy = make_policy(near_kind);
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const int64_t warps_total = (int64_t)gridDim.x * 8;
  uint64_t acc = 0;
  for (int64_t tile = (int64_t)blockIdx.x * 8 + warp; tile < n_rows / 32; tile += warps_total) {
    const int64_t row = tile * 32 + lane;
    int64_t lo = row - window_rows / 2;
    lo = lo < 0 ? 0 : (lo + window_rows > n_rows ? n_rows - window_rows : lo);
    uint64_t state = (uint64_t)row * 0x9E3779B97F4A7C15ull + 1;
#pragma unroll 4
    for (int t = 0; t < kTerms; ++t) {
      state = mix(state + t);
      const bool near = (state & 255u) < near_per_256;
      const uint64_t r = state >> 32;   // 32 random bits
      const int64_t target = near ? lo + (int64_t)((r * (uint64_t)window_rows) >> 32) : (int64_t)(r >> (32 - kRowBits));
      const unsigned char *q = table + ((size_t)target * 8 + (mix((uint64_t)target) & 7u)) * 32;
      // the policy of a load is one value per warp (it travels in a uniform register), so lanes that differ take
      // different instructions
      if constexpr (!HINT) acc += load_sector(q);
      else if (near) acc += load_sector(q, near_policy);
      else acc += load_sector(q, far_policy);
    }
  }
  if (acc == 0x1234567) *sink = acc;
}

void run_mixed(const unsigned char *table, int window_mb, uint32_t near_per_256, int treatment, uint64_t *sink) {
  static const char *names[] = {"no hint", "far normal / near normal", "far evict_first / near normal",
                                "far evict_first / near evict_last"};
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int blocks = sms * 2;
  const int64_t window_rows = (int64_t)window_mb * 1048576 / 256;
  const int far_kind = treatment >= 2 ? kFirst : kNormal, near_kind = treatment == 3 ? kLast : kNormal;
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e30f, worst = 0;
  for (int rep = 0; rep < 4; ++rep) {   // the first pass is the warm-up; each pass streams the whole table through L2
    cudaEventRecord(a);
    if (treatment == 0) k_mixed<false><<<blocks, 256>>>(table, near_per_256, window_rows, far_kind, near_kind, sink);
    else k_mixed<true><<<blocks, 256>>>(table, near_per_256, window_rows, far_kind, near_kind, sink);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    if (rep == 0) continue;
    best = ms < best ? ms : best;
    worst = ms > worst ? ms : worst;
  }
  const double loads = (double)((int64_t)1 << kRowBits) * kTerms;
  printf("mixed  window %2d MB  near %3u/256  %-34s : %6.1f G look-ups/s  (%.2f .. %.2f ms, 3 passes)\n", window_mb,
         near_per_256, names[treatment], loads / best / 1e6, best, worst);
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
    if (mb == 4096) {
      printf("# random 32-byte sectors of a table that fits the L2 (every access a hit after the warm-up pass)\n");
      for (size_t small : {8ul, 16ul, 32ul}) {
        run<32, 4>(table, small << 20, 8, sink, 256);
        run<32, 4>(table, small << 20, 2, sink, 1024);
      }
      printf("# model of k_rows on the ordered table: %d rows x %d look-ups, 4096 MB table\n", 1 << kRowBits, kTerms);
      run_mixed(reinterpret_cast<const unsigned char *>(table), 16, 0u, 0, sink);     // every look-up far
      run_mixed(reinterpret_cast<const unsigned char *>(table), 16, 256u, 0, sink);   // every look-up near
      for (int window_mb : {8, 16, 32})
        for (uint32_t near : {85u, 128u})
          for (int treatment = 0; treatment < 4; ++treatment)
            run_mixed(reinterpret_cast<const unsigned char *>(table), window_mb, near, treatment, sink);
    }
    cudaFree(table);
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}
