// dmv_solver.cu -- vector kernels of the device-resident Lanczos iteration (the consumer of the hot path; the reference
// drives its product from PRIMME's matvec callback, src/Diagonalize.chpl:134-225, src/PRIMME.chpl:267-373).
// Everything stays in HBM between products: y = H v, alpha = <v, y>, y -= alpha v + beta v_prev, beta' = |y|.
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>

#include "dmv_host.h"

namespace dmv {

void count_launch();

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// out[0..1] += sum_i conj(a_i) b_i   (real vectors: out[1] untouched)
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_dot(int64_t n, const double *__restrict__ a, const double *__restrict__ b,
                                                  double *out) {
  double re = 0.0, im = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (CE) {
      const double2 x = reinterpret_cast<const double2 *>(a)[i], y = reinterpret_cast<const double2 *>(b)[i];
      re += x.x * y.x + x.y * y.y;
      im += x.x * y.y - x.y * y.x;
    } else {
      re += a[i] * b[i];
    }
  }
  __shared__ double s_re[kThreads / 32], s_im[kThreads / 32];
  re = warp_sum(re);
  if (CE) im = warp_sum(im);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_re[warp] = re; s_im[warp] = im; }
  __syncthreads();
  if (warp == 0) {
    re = lane < kThreads / 32 ? s_re[lane] : 0.0;
    im = lane < kThreads / 32 ? s_im[lane] : 0.0;
    re = warp_sum(re);
    if (CE) im = warp_sum(im);
    if (lane == 0) {
      atomicAdd(out, re);
      if (CE) atomicAdd(out + 1, im);
    }
  }
}

// w -= alpha v + beta u (alpha, beta real: H is Hermitian);  out[0] += |w|^2 of the updated w
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_lanczos_update(int64_t n, double *w, const double *__restrict__ v,
                                                             const double *__restrict__ u, const double *coef,
                                                             double *out) {
  const double alpha = coef[0], beta = coef[1];
  double nrm = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t m = CE ? 2 * n : n;   // real and imaginary parts update alike
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    double t = w[i] - alpha * v[i];
    if (u) t -= beta * u[i];
    w[i] = t;
    nrm += t * t;
  }
  __shared__ double s[kThreads / 32];
  nrm = warp_sum(nrm);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) s[warp] = nrm;
  __syncthreads();
  if (warp == 0) {
    nrm = lane < kThreads / 32 ? s[lane] : 0.0;
    nrm = warp_sum(nrm);
    if (lane == 0) atomicAdd(out, nrm);
  }
}

// y = s * x (y may alias x);  or y += s * x
template <bool ACCUMULATE>
__global__ void __launch_bounds__(kThreads) k_scale(int64_t m, double s, const double *x, double *y) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride)
    y[i] = ACCUMULATE ? y[i] + s * x[i] : s * x[i];
}

// deterministic start vector: uniform(-0.5, 0.5) from the splitmix64 finaliser of (seed, global element index)
__global__ void __launch_bounds__(kThreads) k_fill(int64_t m, uint64_t seed, uint64_t offset, double *x) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    const uint64_t h = hash64_01(seed * 0x9e3779b97f4a7c15ull + offset + (uint64_t)i + 1);
    x[i] = (double)(h >> 11) * (1.0 / 9007199254740992.0) - 0.5;
  }
}

int blocks_for(int64_t n) {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  int64_t b = (n + kThreads - 1) / kThreads;
  if (b < 1) b = 1;
  if (b > (int64_t)sms * 8) b = (int64_t)sms * 8;
  return (int)b;
}

void check(const char *what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
  count_launch();
}

}  // namespace

void launch_dot(int64_t n, bool complex_elements, const double *a, const double *b, double *out2, cudaStream_t s) {
  if (n <= 0) return;
  if (complex_elements) k_dot<true><<<blocks_for(n), kThreads, 0, s>>>(n, a, b, out2);
  else k_dot<false><<<blocks_for(n), kThreads, 0, s>>>(n, a, b, out2);
  check("k_dot");
}

void launch_lanczos_update(int64_t n, bool complex_elements, double *w, const double *v, const double *u,
                           const double *coef2, double *out1, cudaStream_t s) {
  if (n <= 0) return;
  if (complex_elements) k_lanczos_update<true><<<blocks_for(2 * n), kThreads, 0, s>>>(n, w, v, u, coef2, out1);
  else k_lanczos_update<false><<<blocks_for(n), kThreads, 0, s>>>(n, w, v, u, coef2, out1);
  check("k_lanczos_update");
}

void launch_scale(int64_t words, double scale, const double *x, double *y, bool accumulate, cudaStream_t s) {
  if (words <= 0) return;
  if (accumulate) k_scale<true><<<blocks_for(words), kThreads, 0, s>>>(words, scale, x, y);
  else k_scale<false><<<blocks_for(words), kThreads, 0, s>>>(words, scale, x, y);
  check("k_scale");
}

void launch_fill(int64_t words, uint64_t seed, uint64_t offset, double *x, cudaStream_t s) {
  if (words <= 0) return;
  k_fill<<<blocks_for(words), kThreads, 0, s>>>(words, seed, offset, x);
  check("k_fill");
}

}  // namespace dmv
