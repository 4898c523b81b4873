// dmv_solver.cu -- vector kernels of the device-resident Lanczos iteration (the consumer of the hot path; the reference
// drives its product from PRIMME's matvec callback, src/Diagonalize.chpl:134-225, src/PRIMME.chpl:267-373).
// Everything stays in HBM between products: y = H v, alpha = <v, y>, y -= alpha v + beta v_prev, beta' = |y|.
// Also the block kernels of dmv_expm_multiply (dmv_krylov.cu): h = V^H w and out = a w - V c over many stored vectors,
// and those of dmv_eigsh (dmv_eigsh.cu): V^H W and W^H W, W -= V C for a block W of up to six vectors, and the in-place
// rotation V <- V S.
#include <cuda_runtime.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "dmv_context.h"

namespace dmv {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// The fixed-order epilogue of a CTA's reductions: value v of every thread (re[v], and im[v] when CX), summed inside the
// warp by the xor butterfly and then over warps 0 .. 7 in order, lands in out[(blockIdx * NV + v) * 2 + {0, 1}]
// (imaginary part 0 when !CX).  A repeated launch on the same grid writes the same bits.  The kernel declares `s` next
// to its other shared arrays.
template <int NV, bool CX>
using CtaSums = double[kThreads / 32][NV][CX ? 2 : 1];
template <int NV, bool CX>
__device__ __forceinline__ void cta_partials(CtaSums<NV, CX> &s, const double *re, const double *im,
                                             double *__restrict__ out) {
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const double r = warp_sum(re[v]);
    const double i = CX ? warp_sum(im[v]) : 0.0;
    if ((threadIdx.x & 31) == 0) {
      s[threadIdx.x >> 5][v][0] = r;
      if constexpr (CX) s[threadIdx.x >> 5][v][1] = i;
    }
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double tr = 0.0, ti = 0.0;
    for (int q = 0; q < kThreads / 32; ++q) {
      tr += s[q][threadIdx.x][0];
      if constexpr (CX) ti += s[q][threadIdx.x][1];
    }
    out[(blockIdx.x * NV + threadIdx.x) * 2] = tr;
    out[(blockIdx.x * NV + threadIdx.x) * 2 + 1] = ti;
  }
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

// ---- block kernels of dmv_expm_multiply (full reorthogonalisation against up to kMaxBlockVectors stored vectors).
// Every reduction is deterministic: each CTA sums its warps in a fixed order into its own slot of `partials`, and
// k_reduce_partials sums the CTAs in a fixed order -- no floating-point atomics, so a repeated call is bit-identical.

// elements per thread and tile of k_block_dot: 32 bytes of every vector per thread and tile
template <bool CE> __host__ __device__ constexpr int dot_elems() { return CE ? 2 : 4; }
constexpr int kDotChunk = 8;   // vectors whose accumulators are held in registers at once

// partials[(blockIdx * (J + 1) + k) * 2 + {0, 1}] = this CTA's share of <V_k, w> (k < J) and of |w|^2 (k == J)
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_block_dot(int64_t n, VecList V, int J, const double *__restrict__ w,
                                                        double *__restrict__ partials) {
  constexpr int E = dot_elems<CE>();
  __shared__ double s_acc[kThreads / 32][kMaxBlockVectors + 1][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = lane; k <= J; k += 32) s_acc[warp][k][0] = s_acc[warp][k][1] = 0.0;   // warp-private rows
  __syncwarp();
  const int64_t tile = (int64_t)kThreads * E;
  for (int64_t base = (int64_t)blockIdx.x * tile; base < n; base += (int64_t)gridDim.x * tile) {
    double wr[E], wi[E];
    unsigned in = 0;   // bit e: element e of this thread's tile exists
    double nrm = 0.0;
#pragma unroll
    for (int e = 0; e < E; ++e) {   // w is read once per tile; the vectors stream past it in chunks
      const int64_t i = base + (int64_t)e * kThreads + threadIdx.x;
      wr[e] = wi[e] = 0.0;
      if (i < n) {
        in |= 1u << e;
        if (CE) { const double2 t = reinterpret_cast<const double2 *>(w)[i]; wr[e] = t.x; wi[e] = t.y; }
        else wr[e] = w[i];
      }
      nrm += wr[e] * wr[e] + wi[e] * wi[e];
    }
    nrm = warp_sum(nrm);
    if (lane == 0) s_acc[warp][J][0] += nrm;
    for (int k0 = 0; k0 < J; k0 += kDotChunk) {
      double ar[kDotChunk], ai[kDotChunk];
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {
        ar[kk] = ai[kk] = 0.0;
        if (k0 + kk < J) {
          const double *v = V.p[k0 + kk];
#pragma unroll
          for (int e = 0; e < E; ++e) {
            if (!(in >> e & 1u)) continue;
            const int64_t i = base + (int64_t)e * kThreads + threadIdx.x;
            if (CE) {   // conj(v) * w
              const double2 t = __ldg(reinterpret_cast<const double2 *>(v) + i);
              ar[kk] += t.x * wr[e] + t.y * wi[e];
              ai[kk] += t.x * wi[e] - t.y * wr[e];
            } else {
              ar[kk] += __ldg(v + i) * wr[e];
            }
          }
        }
      }
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {
        if (k0 + kk >= J) break;
        const double r = warp_sum(ar[kk]);
        const double im = CE ? warp_sum(ai[kk]) : 0.0;
        if (lane == 0) { s_acc[warp][k0 + kk][0] += r; s_acc[warp][k0 + kk][1] += im; }
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k <= J; k += blockDim.x) {
    double re = 0.0, im = 0.0;
#pragma unroll
    for (int q = 0; q < kThreads / 32; ++q) { re += s_acc[q][k][0]; im += s_acc[q][k][1]; }
    partials[((int64_t)blockIdx.x * (J + 1) + k) * 2] = re;
    partials[((int64_t)blockIdx.x * (J + 1) + k) * 2 + 1] = im;
  }
}

// out = a w - sum_k c_k V_k (w may be null: a w = 0; out may alias w), c interleaved (re, im) in device memory (real
// vectors use the real parts); partials[blockIdx * 2] = this CTA's share of |out|^2
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_block_combine(int64_t n, double a, const double *w, VecList V, int J,
                                                            const double *__restrict__ coef, double *out,
                                                            double *__restrict__ partials) {
  __shared__ double s_c[kMaxBlockVectors][2];
  __shared__ CtaSums<1, false> s;
  for (int k = threadIdx.x; k < J; k += blockDim.x) { s_c[k][0] = coef[2 * k]; s_c[k][1] = coef[2 * k + 1]; }
  __syncthreads();
  double nrm = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double re = 0.0, im = 0.0;
    if (w) {
      if (CE) { const double2 t = reinterpret_cast<const double2 *>(w)[i]; re = a * t.x; im = a * t.y; }
      else re = a * w[i];
    }
    for (int k0 = 0; k0 < J; k0 += kDotChunk) {
      double vr[kDotChunk], vi[kDotChunk];
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {   // issue the chunk's loads before the first use
        vr[kk] = vi[kk] = 0.0;
        if (k0 + kk < J) {
          if (CE) { const double2 t = __ldg(reinterpret_cast<const double2 *>(V.p[k0 + kk]) + i); vr[kk] = t.x; vi[kk] = t.y; }
          else vr[kk] = __ldg(V.p[k0 + kk] + i);
        }
      }
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {
        if (k0 + kk >= J) break;
        const double cr = s_c[k0 + kk][0], ci = s_c[k0 + kk][1];
        if (CE) { re -= cr * vr[kk] - ci * vi[kk]; im -= cr * vi[kk] + ci * vr[kk]; }
        else re -= cr * vr[kk];
      }
    }
    if (CE) reinterpret_cast<double2 *>(out)[i] = make_double2(re, im);
    else out[i] = re;
    nrm += re * re + im * im;
  }
  cta_partials<1, false>(s, &nrm, nullptr, partials);
}

// out[2k + {0, 1}] = sum over the `blocks` CTAs of partials[(b * width + k) * 2 + {0, 1}], in a fixed order; one CTA per k
__global__ void __launch_bounds__(kThreads) k_reduce_partials(int blocks, int width, const double *__restrict__ partials,
                                                              double *__restrict__ out) {
  const int k = blockIdx.x;
  double re = 0.0, im = 0.0;
  for (int b = threadIdx.x; b < blocks; b += blockDim.x) {
    re += partials[((int64_t)b * width + k) * 2];
    im += partials[((int64_t)b * width + k) * 2 + 1];
  }
  __shared__ CtaSums<1, true> s;
  cta_partials<1, true>(s, &re, &im, out);
}

// ---- block kernels of dmv_eigsh (block Krylov-Schur): R <= 6 right-hand vectors W_0 .. W_{R-1}, w_stride elements apart
// (a block of the basis), against J stored vectors.  Deterministic like the kernels above.

// Sums each of the NV values of a[] over the warp (NV a power of two, <= 32) in a fixed order with NV - 1 + 5 - log2(NV)
// shuffles instead of 5 NV: each step hands half of the values to the partner lane.  On return, lane v << (5 - log2 NV)
// holds the total of value v (the other lanes hold copies or partial sums).
template <int N, int H, int OFF>
__device__ __forceinline__ void reduce_scatter_steps(double (&a)[N], int lane) {   // the first H values -> H / 2
  if constexpr (H > 1) {
    constexpr int h = H / 2;
    const bool hi = lane & OFF;
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const double send = hi ? a[i] : a[i + h];
      const double keep = hi ? a[i + h] : a[i];
      a[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
    reduce_scatter_steps<N, h, OFF / 2>(a, lane);
  }
}

template <int NV>
__device__ __forceinline__ double warp_reduce_scatter(double (&a)[NV]) {
  static_assert(NV >= 1 && NV <= 32 && (NV & (NV - 1)) == 0, "NV must be a power of two <= 32");
  reduce_scatter_steps<NV, NV, 16>(a, threadIdx.x & 31);
  double v = a[0];
#pragma unroll
  for (int off = 16 / NV; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

constexpr int log2_int(int v) { return v <= 1 ? 0 : 1 + log2_int(v / 2); }
constexpr int pow2_ceil(int v) { return v <= 1 ? 1 : 2 * pow2_ceil((v + 1) / 2); }

template <bool CE, int R> __host__ __device__ constexpr int gram_chunk() { return R >= 8 ? 1 : 8 / R; }
// elements per thread and tile of k_block_gram: about 24 doubles of W in registers
template <bool CE, int R> __host__ __device__ constexpr int gram_elems() {
  return CE ? (R <= 3 ? 4 : 2) : (R <= 3 ? 8 : 4);
}

// partials[(blockIdx * width + t) * 2 + {0, 1}], width = J R + R R: this CTA's share of <V_k, W_r> (t = k R + r) and of
// <W_r, W_s> (t = J R + r R + s).  Every warp accumulates into its own rows of dynamic shared memory.
template <bool CE, int R>
__global__ void __launch_bounds__(kThreads, 2) k_block_gram(int64_t n, VecList V, int J, const double *__restrict__ W,
                                                         int64_t w_stride, double *__restrict__ partials) {
  constexpr int E = gram_elems<CE, R>(), KC = gram_chunk<CE, R>(), C = CE ? 2 : 1;
  constexpr int NV = KC * R * C, NVP = pow2_ceil(NV), SH = 5 - log2_int(NVP);
  constexpr int NG = R * C, NGP = pow2_ceil(NG), SHG = 5 - log2_int(NGP);
  extern __shared__ double s_gram[];   // [warps][width][C]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int width = J * R + R * R;
  double *acc = s_gram + (size_t)warp * width * C;
  for (int t = lane; t < width * C; t += 32) acc[t] = 0.0;
  __syncwarp();
  const int64_t tile = (int64_t)kThreads * E;
  for (int64_t base = (int64_t)blockIdx.x * tile; base < n; base += (int64_t)gridDim.x * tile) {
    double wr[R][E], wi[R][E];
    unsigned in = 0;
#pragma unroll
    for (int e = 0; e < E; ++e) {   // W is read once per tile; the stored vectors stream past it KC at a time
      const int64_t i = base + (int64_t)e * kThreads + threadIdx.x;
      if (i < n) in |= 1u << e;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        wr[r][e] = wi[r][e] = 0.0;
        if (i < n) {
          if (CE) { const double2 t = reinterpret_cast<const double2 *>(W + 2 * r * w_stride)[i]; wr[r][e] = t.x; wi[r][e] = t.y; }
          else wr[r][e] = W[r * w_stride + i];
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {   // row r of the Gram matrix: conj(W_r) W_s
      double g[NGP];
#pragma unroll
      for (int v = 0; v < NGP; ++v) g[v] = 0.0;
#pragma unroll
      for (int s = 0; s < R; ++s)
#pragma unroll
        for (int e = 0; e < E; ++e) {
          g[s * C] += wr[r][e] * wr[s][e] + wi[r][e] * wi[s][e];
          if (CE) g[s * C + 1] += wr[r][e] * wi[s][e] - wi[r][e] * wr[s][e];
        }
      const double t = warp_reduce_scatter<NGP>(g);
      if ((lane & ((1 << SHG) - 1)) == 0 && (lane >> SHG) < NG) acc[(J * R + r * R) * C + (lane >> SHG)] += t;
    }
    for (int k0 = 0; k0 < J; k0 += KC) {
      double a[NVP];
#pragma unroll
      for (int v = 0; v < NVP; ++v) a[v] = 0.0;
#pragma unroll
      for (int kk = 0; kk < KC; ++kk) {
        if (k0 + kk < J) {
          const double *v = V.p[k0 + kk];
#pragma unroll
          for (int e = 0; e < E; ++e) {
            if (!(in >> e & 1u)) continue;
            const int64_t i = base + (int64_t)e * kThreads + threadIdx.x;
            if (CE) {   // conj(v) * w
              const double2 t = __ldg(reinterpret_cast<const double2 *>(v) + i);
#pragma unroll
              for (int r = 0; r < R; ++r) {
                a[(kk * R + r) * 2] += t.x * wr[r][e] + t.y * wi[r][e];
                a[(kk * R + r) * 2 + 1] += t.x * wi[r][e] - t.y * wr[r][e];
              }
            } else {
              const double t = __ldg(v + i);
#pragma unroll
              for (int r = 0; r < R; ++r) a[kk * R + r] += t * wr[r][e];
            }
          }
        }
      }
      const double t = warp_reduce_scatter<NVP>(a);
      const int v = lane >> SH;
      if ((lane & ((1 << SH) - 1)) == 0 && v < NV && k0 * R * C + v < J * R * C) acc[k0 * R * C + v] += t;
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < width; t += blockDim.x) {
    double re = 0.0, im = 0.0;
#pragma unroll
    for (int q = 0; q < kThreads / 32; ++q) {
      re += s_gram[((size_t)q * width + t) * C];
      if (CE) im += s_gram[((size_t)q * width + t) * C + 1];
    }
    partials[((int64_t)blockIdx.x * width + t) * 2] = re;
    partials[((int64_t)blockIdx.x * width + t) * 2 + 1] = im;
  }
}

// W_r -= sum_{k < J} c_{k r} V_k with c[2 (k R + r) + {0, 1}] in device memory (real vectors use the real parts);
// partials[(blockIdx * R + r) * 2] = this CTA's share of |W_r|^2 after the update
template <bool CE, int R>
__global__ void __launch_bounds__(kThreads) k_block_update(int64_t n, VecList V, int J, const double *__restrict__ coef,
                                                           double *W, int64_t w_stride, double *__restrict__ partials) {
  __shared__ double s_c[kMaxBlockVectors * R][2];
  __shared__ CtaSums<R, false> s;
  for (int k = threadIdx.x; k < J * R; k += blockDim.x) { s_c[k][0] = coef[2 * k]; s_c[k][1] = coef[2 * k + 1]; }
  __syncthreads();
  double nrm[R];
#pragma unroll
  for (int r = 0; r < R; ++r) nrm[r] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double re[R], im[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (CE) { const double2 t = reinterpret_cast<const double2 *>(W + 2 * r * w_stride)[i]; re[r] = t.x; im[r] = t.y; }
      else { re[r] = W[r * w_stride + i]; im[r] = 0.0; }
    }
    for (int k0 = 0; k0 < J; k0 += kDotChunk) {
      double vr[kDotChunk], vi[kDotChunk];
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {   // issue the chunk's loads before the first use
        vr[kk] = vi[kk] = 0.0;
        if (k0 + kk < J) {
          if (CE) { const double2 t = __ldg(reinterpret_cast<const double2 *>(V.p[k0 + kk]) + i); vr[kk] = t.x; vi[kk] = t.y; }
          else vr[kk] = __ldg(V.p[k0 + kk] + i);
        }
      }
#pragma unroll
      for (int kk = 0; kk < kDotChunk; ++kk) {
        if (k0 + kk >= J) break;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const double cr = s_c[(k0 + kk) * R + r][0], ci = s_c[(k0 + kk) * R + r][1];
          if (CE) { re[r] -= cr * vr[kk] - ci * vi[kk]; im[r] -= cr * vi[kk] + ci * vr[kk]; }
          else re[r] -= cr * vr[kk];
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (CE) reinterpret_cast<double2 *>(W + 2 * r * w_stride)[i] = make_double2(re[r], im[r]);
      else W[r * w_stride + i] = re[r];
      nrm[r] += re[r] * re[r] + im[r] * im[r];
    }
  }
  cta_partials<R, false>(s, nrm, nullptr, partials);
}

// In place V_j <- sum_{i < k} S_{ij} V_i for j < l <= k, S[2 (i l + j) + {0, 1}] in device memory (real vectors use the
// real parts).  A CTA stages a tile of every one of the k inputs in shared memory before it writes any output over them,
// so no second basis is needed; each output element is summed over i in ascending order.
constexpr int kRotWords = 64;   // 8-byte words of every vector in a tile: 64 real or 32 complex elements
constexpr int kRotOut = 4;      // outputs per thread and pass
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_block_rotate(int64_t n, VecList V, int k, int l,
                                                           const double *__restrict__ S) {
  constexpr int TE = CE ? kRotWords / 2 : kRotWords;   // elements per tile
  extern __shared__ double s_tile[];                   // [k][kRotWords]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double2 *S2 = reinterpret_cast<const double2 *>(S);
  for (int64_t base = (int64_t)blockIdx.x * TE; base < n; base += (int64_t)gridDim.x * TE) {
    const int words = (int)(std::min<int64_t>(TE, n - base) * (CE ? 2 : 1));
    const int64_t w0 = base * (CE ? 2 : 1);
    for (int t = threadIdx.x; t < k * kRotWords; t += kThreads) {
      const int i = t / kRotWords, e = t % kRotWords;
      s_tile[t] = e < words ? V.p[i][w0 + e] : 0.0;
    }
    __syncthreads();
    for (int j0 = warp * kRotOut; j0 < l; j0 += (kThreads / 32) * kRotOut) {
      double ar[kRotOut][2], ai[kRotOut][2];   // [output][element of the lane: lane, lane + 32 (real only)]
#pragma unroll
      for (int jj = 0; jj < kRotOut; ++jj) ar[jj][0] = ar[jj][1] = ai[jj][0] = ai[jj][1] = 0.0;
      for (int i = 0; i < k; ++i) {
        double xr0, xi0 = 0.0, xr1 = 0.0;
        if (CE) { const double2 t = reinterpret_cast<const double2 *>(s_tile + i * kRotWords)[lane]; xr0 = t.x; xi0 = t.y; }
        else { xr0 = s_tile[i * kRotWords + lane]; xr1 = s_tile[i * kRotWords + 32 + lane]; }
#pragma unroll
        for (int jj = 0; jj < kRotOut; ++jj) {
          if (j0 + jj < l) {
            const double2 c = __ldg(S2 + (size_t)i * l + j0 + jj);
            if (CE) { ar[jj][0] += xr0 * c.x - xi0 * c.y; ai[jj][0] += xr0 * c.y + xi0 * c.x; }
            else { ar[jj][0] += xr0 * c.x; ar[jj][1] += xr1 * c.x; }
          }
        }
      }
#pragma unroll
      for (int jj = 0; jj < kRotOut; ++jj) {
        if (j0 + jj >= l) break;
        double *out = const_cast<double *>(V.p[j0 + jj]) + w0;
        if (CE) { if (2 * lane < words) reinterpret_cast<double2 *>(out)[lane] = make_double2(ar[jj][0], ai[jj][0]); }
        else {
          if (lane < words) out[lane] = ar[jj][0];
          if (32 + lane < words) out[32 + lane] = ar[jj][1];
        }
      }
    }
    __syncthreads();   // the next tile overwrites s_tile
  }
}

// ---- kernels of dmv_lanczos_quadrature (dmv_thermal.cu): G <= 6 independent three-term recurrences without a stored
// basis, vector g of a group at offset g n elements.  Deterministic like the kernels above.

// Seeded start vectors: entry s of vector first + g depends only on (seed, first + g, reps[s]), so every rank count
// starts from the same vectors.  float64: +-1; complex128: e^{i phi}, phi uniform in [0, 2 pi).
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_quad_fill(int64_t n, const uint64_t *__restrict__ reps, uint64_t seed,
                                                        int first, int G, double *x) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int g = 0; g < G; ++g) {
    const uint64_t key = hash64_01(seed + 0x9e3779b97f4a7c15ull * (uint64_t)(first + g + 1));
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      const uint64_t h = hash64_01(reps[i] ^ key);
      if (CE) {
        double s, c;
        sincos(6.283185307179586 * ((double)(h >> 11) * 0x1p-53), &s, &c);
        reinterpret_cast<double2 *>(x)[(int64_t)g * n + i] = make_double2(c, s);
      } else {
        x[(int64_t)g * n + i] = (h >> 63) ? -1.0 : 1.0;
      }
    }
  }
}

// partials[(blockIdx * G + g) * 2 + {0, 1}] = this CTA's share of <A_g, B_g>; A and B are read once
template <bool CE, int G>
__global__ void __launch_bounds__(kThreads) k_quad_dot(int64_t n, const double *__restrict__ A,
                                                       const double *__restrict__ B, double *__restrict__ partials) {
  double re[G], im[G];
#pragma unroll
  for (int g = 0; g < G; ++g) re[g] = im[g] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (CE) {   // conj(a) * b
        const double2 a = __ldg(reinterpret_cast<const double2 *>(A) + (int64_t)g * n + i);
        const double2 b = __ldg(reinterpret_cast<const double2 *>(B) + (int64_t)g * n + i);
        re[g] += a.x * b.x + a.y * b.y;
        im[g] += a.x * b.y - a.y * b.x;
      } else {
        re[g] += __ldg(A + (int64_t)g * n + i) * __ldg(B + (int64_t)g * n + i);
      }
    }
  }
  __shared__ CtaSums<G, true> s;   // real vectors too: their imaginary sums are zeros, as they always were
  cta_partials<G, true>(s, re, im, partials);
}

// Step j of G recurrences r_{j+1} = W / beta_j - alpha_j r_j / beta_j - beta_j r_{j-1} / beta_{j-1}, written over
// P = r_{j-1}; Q = r_j, W = H r_j.  The coefficients come from device memory: dot[2 (t G + g)] = <r_t, H r_t> and
// b2[2 (t G + g)] = |r_t|^2 of step t.  A vector whose recurrence broke down at step j (quad_breakdown, or already zero)
// gets r_{j+1} = r_j = 0.  partials[(blockIdx * G + g) * 2] = this CTA's share of |r_{j+1}|^2.
template <bool CE, int G>
__global__ void __launch_bounds__(kThreads) k_quad_update(int64_t n, double *P, double *Q, const double *__restrict__ W,
                                                          const double *__restrict__ dot, const double *__restrict__ b2,
                                                          int j, double *__restrict__ partials) {
  __shared__ double s_c[G][3];   // 1 / beta_j, alpha_j / beta_j, beta_j / beta_{j-1}
  __shared__ int s_dead[G];
  __shared__ CtaSums<G, false> s;
  if (threadIdx.x < G) {
    const int g = threadIdx.x;
    const double bj2 = b2[2 * (j * G + g)];
    bool dead = !(bj2 > 0.0);
    double bp2 = 0.0;
    if (!dead && j > 0) {
      bp2 = b2[2 * ((j - 1) * G + g)];
      dead = !(bp2 > 0.0) || quad_breakdown(bj2, dot[2 * ((j - 1) * G + g)], bp2);
    }
    const double beta = sqrt(bj2);
    s_dead[g] = dead;
    s_c[g][0] = dead ? 0.0 : 1.0 / beta;
    s_c[g][1] = dead ? 0.0 : dot[2 * (j * G + g)] / bj2 / beta;
    s_c[g][2] = dead || j == 0 ? 0.0 : beta / sqrt(bp2);
  }
  __syncthreads();
  double nrm[G];
#pragma unroll
  for (int g = 0; g < G; ++g) nrm[g] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t e = (int64_t)g * n + i;
      if (s_dead[g]) {
        if (CE) { reinterpret_cast<double2 *>(P)[e] = make_double2(0.0, 0.0); reinterpret_cast<double2 *>(Q)[e] = make_double2(0.0, 0.0); }
        else { P[e] = 0.0; Q[e] = 0.0; }
        continue;
      }
      const double cw = s_c[g][0], cq = s_c[g][1], cp = s_c[g][2];
      if (CE) {
        const double2 w = __ldg(reinterpret_cast<const double2 *>(W) + e), q = reinterpret_cast<const double2 *>(Q)[e];
        const double2 p = j > 0 ? reinterpret_cast<const double2 *>(P)[e] : make_double2(0.0, 0.0);
        const double rx = cw * w.x - cq * q.x - cp * p.x, ry = cw * w.y - cq * q.y - cp * p.y;
        reinterpret_cast<double2 *>(P)[e] = make_double2(rx, ry);
        nrm[g] += rx * rx + ry * ry;
      } else {
        const double p = j > 0 ? P[e] : 0.0;
        const double r = cw * __ldg(W + e) - cq * Q[e] - cp * p;
        P[e] = r;
        nrm[g] += r * r;
      }
    }
  }
  cta_partials<G, false>(s, nrm, nullptr, partials);
}

}  // namespace

namespace {

constexpr int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// the vector kernels with atomic or no reductions: eight CTAs per SM at most
int blocks_for(int64_t n) { return capped_grid(ceil_div(n, kThreads), (int64_t)sm_count() * 8); }

// f(std::integral_constant<int, W>) for the W = 1 .. kMaxBlockRhs vectors of a block or a group
template <typename F>
auto with_width(int w, F &&f) {
  return with_choice<1, 2, 3, 4, 5, 6>(w, f);
}

}  // namespace

int launch_dot(int64_t n, bool complex_elements, const double *a, const double *b, double *out2, cudaStream_t s) {
  if (n <= 0) return 0;
  const int grid = blocks_for(n);
  with_bool(complex_elements, [&](auto ce) { k_dot<ce()><<<grid, kThreads, 0, s>>>(n, a, b, out2); });
  check_launch("k_dot");
  return grid;
}

int launch_lanczos_update(int64_t n, bool complex_elements, double *w, const double *v, const double *u,
                          const double *coef2, double *out1, cudaStream_t s) {
  if (n <= 0) return 0;
  const int grid = blocks_for(complex_elements ? 2 * n : n);
  with_bool(complex_elements, [&](auto ce) {
    k_lanczos_update<ce()><<<grid, kThreads, 0, s>>>(n, w, v, u, coef2, out1);
  });
  check_launch("k_lanczos_update");
  return grid;
}

int launch_scale(int64_t words, double scale, const double *x, double *y, bool accumulate, cudaStream_t s) {
  if (words <= 0) return 0;
  const int grid = blocks_for(words);
  with_bool(accumulate, [&](auto acc) { k_scale<acc()><<<grid, kThreads, 0, s>>>(words, scale, x, y); });
  check_launch("k_scale");
  return grid;
}

int launch_fill(int64_t words, uint64_t seed, uint64_t offset, double *x, cudaStream_t s) {
  if (words <= 0) return 0;
  const int grid = blocks_for(words);
  k_fill<<<grid, kThreads, 0, s>>>(words, seed, offset, x);
  check_launch("k_fill");
  return grid;
}

namespace {

// CTAs of a k_block_dot / k_block_combine launch over n elements
int block_dot_grid(int64_t n, bool complex_elements) {
  return with_bool(complex_elements, [&](auto ce) {
    return one_wave(k_block_dot<ce()>, ceil_div(ceil_div(std::max<int64_t>(n, 0), dot_elems<ce()>()), kThreads));
  });
}
int block_combine_grid(int64_t n, bool complex_elements) {
  return with_bool(complex_elements, [&](auto ce) { return one_wave(k_block_combine<ce()>, ceil_div(n, kThreads)); });
}

}  // namespace

int block_partials_grid(int64_t n, bool complex_elements) {
  return std::max(block_dot_grid(n, complex_elements), block_combine_grid(n, complex_elements));
}

int launch_block_dot(int64_t n, bool complex_elements, const VecList &V, int J, const double *w, double *partials,
                     double *h, cudaStream_t s) {
  if (J < 0 || J > kMaxBlockVectors) throw std::runtime_error("k_block_dot: bad number of vectors");
  const int grid = block_dot_grid(n, complex_elements);
  with_bool(complex_elements, [&](auto ce) { k_block_dot<ce()><<<grid, kThreads, 0, s>>>(n, V, J, w, partials); });
  check_launch("k_block_dot");
  launch_reduce_partials(grid, J + 1, partials, h, s);
  return grid;
}

int launch_block_combine(int64_t n, bool complex_elements, double a, const double *w, const VecList &V, int J,
                         const double *coef, double *out, double *partials, double *nrm2, cudaStream_t s) {
  if (J < 0 || J > kMaxBlockVectors) throw std::runtime_error("k_block_combine: bad number of vectors");
  const int grid = block_combine_grid(n, complex_elements);
  with_bool(complex_elements, [&](auto ce) {
    k_block_combine<ce()><<<grid, kThreads, 0, s>>>(n, a, w, V, J, coef, out, partials);
  });
  check_launch("k_block_combine");
  launch_reduce_partials(grid, 1, partials, nrm2, s);
  return grid;
}

size_t block_gram_partials() {
  // the most CTAs one wave can hold (8 of 256 threads per SM) times the widest output, J R + R R with J < 65, R = 6
  return (size_t)sm_count() * 8 * (kMaxBlockVectors * kMaxBlockRhs + kMaxBlockRhs * kMaxBlockRhs) * 2;
}

int launch_block_gram(int64_t n, bool complex_elements, const VecList &V, int J, const double *W, int64_t w_stride,
                      int R, double *partials, double *h, cudaStream_t s) {
  if (J < 0 || J > kMaxBlockVectors || R < 1 || R > kMaxBlockRhs)
    throw std::runtime_error("k_block_gram: bad number of vectors");
  const int width = J * R + R * R;
  return with_bool(complex_elements, [&](auto ce) {
    return with_width(R, [&](auto r) {
      constexpr bool CE = ce();
      constexpr int E = gram_elems<CE, r()>();
      const size_t smem = (size_t)(kThreads / 32) * width * (CE ? 2 : 1) * sizeof(double);
      const int grid = one_wave(k_block_gram<CE, r()>, ceil_div(std::max<int64_t>(n, 0), (int64_t)kThreads * E), smem);
      k_block_gram<CE, r()><<<grid, kThreads, smem, s>>>(n, V, J, W, w_stride, partials);
      check_launch("k_block_gram");
      launch_reduce_partials(grid, width, partials, h, s);
      return grid;
    });
  });
}

int launch_block_update(int64_t n, bool complex_elements, const VecList &V, int J, const double *coef, double *W,
                        int64_t w_stride, int R, double *partials, double *nrm2, cudaStream_t s) {
  if (J < 0 || J > kMaxBlockVectors || R < 1 || R > kMaxBlockRhs)
    throw std::runtime_error("k_block_update: bad number of vectors");
  return with_bool(complex_elements, [&](auto ce) {
    return with_width(R, [&](auto r) {
      const int grid = one_wave(k_block_update<ce(), r()>, ceil_div(std::max<int64_t>(n, 0), kThreads));
      k_block_update<ce(), r()><<<grid, kThreads, 0, s>>>(n, V, J, coef, W, w_stride, partials);
      check_launch("k_block_update");
      launch_reduce_partials(grid, R, partials, nrm2, s);
      return grid;
    });
  });
}

void launch_reduce_partials(int blocks, int width, const double *partials, double *out, cudaStream_t s) {
  k_reduce_partials<<<width, kThreads, 0, s>>>(blocks, width, partials, out);
  check_launch("k_reduce_partials");
}

int launch_block_rotate(int64_t n, bool complex_elements, const VecList &V, int k, int l, const double *S,
                        cudaStream_t s) {
  if (k < 1 || k > kMaxBlockVectors || l < 1 || l > k) throw std::runtime_error("k_block_rotate: bad shape");
  if (n <= 0) return 0;
  const size_t smem = (size_t)k * kRotWords * sizeof(double);
  const int grid = with_bool(complex_elements, [&](auto ce) {
    const int g = one_wave(k_block_rotate<ce()>, ceil_div(n, ce() ? kRotWords / 2 : kRotWords), smem);
    k_block_rotate<ce()><<<g, kThreads, smem, s>>>(n, V, k, l, S);
    return g;
  });
  check_launch("k_block_rotate");
  return grid;
}

size_t quad_partials(int G) {
  // the most CTAs one wave can hold (8 of 256 threads per SM) times G (re, im) pairs
  return (size_t)sm_count() * 8 * G * 2;
}

int launch_quad_fill(int64_t n, bool complex_elements, const uint64_t *reps, uint64_t seed, int first, int G,
                     double *x, cudaStream_t s) {
  if (n <= 0) return 0;
  const int grid = blocks_for(n);
  with_bool(complex_elements, [&](auto ce) {
    k_quad_fill<ce()><<<grid, kThreads, 0, s>>>(n, reps, seed, first, G, x);
  });
  check_launch("k_quad_fill");
  return grid;
}

int launch_quad_dot(int64_t n, bool complex_elements, int G, const double *A, const double *B, double *partials,
                    double *out, cudaStream_t s) {
  if (G < 1 || G > kMaxBlockRhs) throw std::runtime_error("k_quad_dot: bad number of vectors");
  return with_bool(complex_elements, [&](auto ce) {
    return with_width(G, [&](auto g) {
      const int grid = one_wave(k_quad_dot<ce(), g()>, ceil_div(n, kThreads));
      k_quad_dot<ce(), g()><<<grid, kThreads, 0, s>>>(n, A, B, partials);
      check_launch("k_quad_dot");
      launch_reduce_partials(grid, G, partials, out, s);
      return grid;
    });
  });
}

int launch_quad_update(int64_t n, bool complex_elements, int G, double *P, double *Q, const double *W,
                       const double *dot, const double *b2, int j, double *partials, double *nrm2, cudaStream_t s) {
  if (G < 1 || G > kMaxBlockRhs) throw std::runtime_error("k_quad_update: bad number of vectors");
  return with_bool(complex_elements, [&](auto ce) {
    return with_width(G, [&](auto g) {
      const int grid = one_wave(k_quad_update<ce(), g()>, ceil_div(n, kThreads));
      k_quad_update<ce(), g()><<<grid, kThreads, 0, s>>>(n, P, Q, W, dot, b2, j, partials);
      check_launch("k_quad_update");
      launch_reduce_partials(grid, G, partials, nrm2, s);
      return grid;
    });
  });
}

}  // namespace dmv

// ---- dmv_debug_solver_kernel (include/dmv_b200.h): one launcher above on host data, for the tests -------------------

namespace {

struct PrivateStream {
  cudaStream_t s = nullptr;
  PrivateStream() { CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~PrivateStream() {
    cudaStreamSynchronize(s);
    cudaStreamDestroy(s);
  }
};

}  // namespace

extern "C" int dmv_debug_solver_kernel(const char *kernel, int elt, int64_t n, const int64_t *args, int n_args,
                                       double scalar, double *arena, int64_t arena_words, const double *coef,
                                       int64_t coef_words, double *out, int64_t out_words, int *grid) {
  API_BEGIN
  if (grid) *grid = 0;
  if (!kernel) throw std::runtime_error("kernel must not be null");
  const std::string k = kernel;
  if (elt != DMV_F64 && elt != DMV_C128) throw std::runtime_error("elt must be DMV_F64 or DMV_C128");
  if (n < 0) throw std::runtime_error(k + ": n must be >= 0");
  if (n_args < 0 || (n_args > 0 && !args) || arena_words < 0 || (arena_words > 0 && !arena) || coef_words < 0 ||
      (coef_words > 0 && !coef) || out_words < 0 || (out_words > 0 && !out))
    throw std::runtime_error(k + ": bad array");
  const bool ce = elt == DMV_C128;
  const int64_t vec = ce ? 2 * n : n;   // words of one vector
  auto arg = [&](int i) {
    if (i >= n_args) throw std::runtime_error(k + ": too few arguments");
    return args[i];
  };
  auto count = [&](int i) {   // a number of vectors or a step: the launchers take int
    const int64_t v = arg(i);
    if (v < -(1 << 20) || v > (1 << 20)) throw std::runtime_error(k + ": argument " + std::to_string(i) + " out of range");
    return (int)v;
  };
  // a vector argument of `words` words at a word offset into the arena (-1: null, where the launcher takes null);
  // complex elements load as double2, so their offsets must be even
  auto vector = [&](int64_t off, int64_t words, bool nullable, bool pairs) {
    if (off == -1 && nullable) return;
    if (off < 0 || off > arena_words || words > arena_words - off)
      throw std::runtime_error(k + ": a vector argument lies past the arena");
    if (pairs && ce && (off & 1)) throw std::runtime_error(k + ": odd word offset for complex elements");
  };
  // fixed arguments, then `listed` stored-vector offsets
  auto shape = [&](int fixed, int listed) {
    if (n_args != fixed + std::max(listed, 0))
      throw std::runtime_error(k + ": expects " + std::to_string(fixed) + " arguments and " +
                               std::to_string(std::max(listed, 0)) + " vector offsets");
    for (int i = 0; i < listed; ++i) vector(args[fixed + i], vec, false, true);
  };
  int64_t need_coef = 0, need_out = 0;
  int list_at = 0, listed = 0;
  if (k == "dot") {
    shape(2, 0);
    vector(arg(0), vec, false, true);
    vector(arg(1), vec, false, true);
    need_out = 2;
  } else if (k == "lanczos_update") {
    shape(3, 0);
    vector(arg(0), vec, false, true);
    vector(arg(1), vec, false, true);
    vector(arg(2), vec, true, true);
    need_coef = 2;
    need_out = 1;
  } else if (k == "scale" || k == "fill") {   // word kernels: n is in words
    shape(3, 0);
    vector(arg(0), n, false, false);
    if (k == "scale") vector(arg(1), n, false, false);
  } else if (k == "block_dot" || k == "block_combine") {
    const int J = count(0), fixed = k == "block_dot" ? 2 : 3;
    shape(fixed, J);
    list_at = fixed, listed = J;
    vector(arg(1), vec, k == "block_combine", true);
    if (k == "block_combine") {
      vector(arg(2), vec, false, true);
      need_coef = 2 * (int64_t)std::max(J, 0);
      need_out = 2;
    } else {
      need_out = 2 * ((int64_t)std::max(J, 0) + 1);
    }
  } else if (k == "block_gram" || k == "block_update") {
    const int J = count(0), R = count(1);
    shape(4, J);
    list_at = 4, listed = J;
    const int64_t w_stride = arg(3);
    if (w_stride < n) throw std::runtime_error(k + ": w_stride must be at least n");
    const int64_t Rv = std::max(R, 1), Jv = std::max(J, 0);
    if (w_stride > (int64_t(1) << 40)) throw std::runtime_error(k + ": w_stride out of range");
    vector(arg(2), ((Rv - 1) * w_stride + n) * (ce ? 2 : 1), false, true);
    if (k == "block_gram") {
      need_out = 2 * (Jv * Rv + Rv * Rv);
    } else {
      need_coef = 2 * Jv * Rv;
      need_out = 2 * Rv;
    }
  } else if (k == "block_rotate") {
    const int kk = count(0), l = count(1);
    shape(2, kk);
    list_at = 2, listed = kk;
    need_coef = 2 * (int64_t)std::max(kk, 0) * std::max(l, 0);
  } else if (k == "quad_fill") {
    shape(4, 0);
    const int G = count(3);
    vector(arg(0), std::max(G, 0) * vec, false, true);
    need_coef = n;   // the representatives, as uint64 bit patterns
  } else if (k == "quad_dot" || k == "quad_update") {
    const bool update = k == "quad_update";
    shape(update ? 6 : 3, 0);
    const int G = count(0);
    const int64_t Gv = std::max(G, 0);
    for (int i = 1; i < (update ? 4 : 3); ++i) vector(arg(i), Gv * vec, false, true);
    if (update) {
      const int j = count(4);
      const int64_t b2_at = arg(5);
      if (j < 0) throw std::runtime_error(k + ": j must be >= 0");
      const int64_t steps = 2 * ((int64_t)j + 1) * Gv;   // dot and b2 of steps 0 .. j
      if (b2_at < 0 || b2_at > coef_words) throw std::runtime_error(k + ": too few coefficients");
      need_coef = std::max(steps, b2_at + steps);
    }
    need_out = 2 * Gv;
  } else {
    throw std::runtime_error("unknown kernel " + k);
  }
  if (coef_words < need_coef) throw std::runtime_error(k + ": too few coefficients");
  if (out_words < need_out) throw std::runtime_error(k + ": too few outputs");
  // the partials buffer, sized as the solvers size it (after the checks above: the sizes query the device)
  int64_t partial_words = 0;
  if (k == "block_dot" || k == "block_combine")
    partial_words = (int64_t)block_partials_grid(n, ce) * (std::max((int)args[0], 0) + 1) * 2;
  else if (k == "block_gram" || k == "block_update")
    partial_words = (int64_t)block_gram_partials();
  else if (k == "quad_dot" || k == "quad_update")
    partial_words = (int64_t)quad_partials(std::max((int)args[0], 1));

  PrivateStream ps;   // declared first: the buffers are freed before the stream goes
  const cudaStream_t st = ps.s;
  host::DevBuf<double> d_arena, d_coef, d_out, d_partials;
  d_arena.alloc(arena_words);
  d_coef.alloc(coef_words);
  d_out.alloc(need_out);
  d_partials.alloc(partial_words);
  if (arena_words)
    CUDA_CHECK(cudaMemcpyAsync(d_arena.ptr, arena, arena_words * 8, cudaMemcpyHostToDevice, st));
  if (coef_words) CUDA_CHECK(cudaMemcpyAsync(d_coef.ptr, coef, coef_words * 8, cudaMemcpyHostToDevice, st));
  // k_dot and k_lanczos_update add to their output; every other output and the partials start as NaN bytes, so a
  // slot no CTA writes shows
  if (k == "dot" || k == "lanczos_update")
    CUDA_CHECK(cudaMemcpyAsync(d_out.ptr, out, need_out * 8, cudaMemcpyHostToDevice, st));
  else if (need_out)
    CUDA_CHECK(cudaMemsetAsync(d_out.ptr, 0xff, need_out * 8, st));
  if (partial_words) CUDA_CHECK(cudaMemsetAsync(d_partials.ptr, 0xff, partial_words * 8, st));
  auto at = [&](int64_t off) { return off == -1 ? nullptr : d_arena.ptr + off; };
  VecList V{};
  for (int i = 0; i < std::min(listed, kMaxBlockVectors); ++i) V.p[i] = at(args[list_at + i]);
  double *const c = d_coef.ptr, *const o = d_out.ptr, *const pt = d_partials.ptr;
  int g = 0;
  if (k == "dot") g = launch_dot(n, ce, at(args[0]), at(args[1]), o, st);
  else if (k == "lanczos_update") g = launch_lanczos_update(n, ce, at(args[0]), at(args[1]), at(args[2]), c, o, st);
  else if (k == "scale") g = launch_scale(n, scalar, at(args[0]), at(args[1]), args[2] != 0, st);
  else if (k == "fill") g = launch_fill(n, (uint64_t)args[1], (uint64_t)args[2], at(args[0]), st);
  else if (k == "block_dot") g = launch_block_dot(n, ce, V, (int)args[0], at(args[1]), pt, o, st);
  else if (k == "block_combine")
    g = launch_block_combine(n, ce, scalar, at(args[1]), V, (int)args[0], c, at(args[2]), pt, o, st);
  else if (k == "block_gram") g = launch_block_gram(n, ce, V, (int)args[0], at(args[2]), args[3], (int)args[1], pt, o, st);
  else if (k == "block_update")
    g = launch_block_update(n, ce, V, (int)args[0], c, at(args[2]), args[3], (int)args[1], pt, o, st);
  else if (k == "block_rotate") g = launch_block_rotate(n, ce, V, (int)args[0], (int)args[1], c, st);
  else if (k == "quad_fill")
    g = launch_quad_fill(n, ce, reinterpret_cast<const uint64_t *>(c), (uint64_t)args[1], (int)args[2], (int)args[3],
                         at(args[0]), st);
  else if (k == "quad_dot") g = launch_quad_dot(n, ce, (int)args[0], at(args[1]), at(args[2]), pt, o, st);
  else g = launch_quad_update(n, ce, (int)args[0], at(args[1]), at(args[2]), at(args[3]), c, c + args[5], (int)args[4],
                              pt, o, st);
  if (arena_words) CUDA_CHECK(cudaMemcpyAsync(arena, d_arena.ptr, arena_words * 8, cudaMemcpyDeviceToHost, st));
  if (need_out) CUDA_CHECK(cudaMemcpyAsync(out, d_out.ptr, need_out * 8, cudaMemcpyDeviceToHost, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  if (grid) *grid = g;
  API_END
}
