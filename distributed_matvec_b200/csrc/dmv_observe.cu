// dmv_observe.cu -- dmv_zz_correlations: the spin-spin correlations <x|σᶻᵢσᶻⱼ|x> / <x|x> and the magnetisation
// <x|σᶻᵢ> / <x|x> of vectors in the symmetry-adapted basis, in one pass over x and the representatives.
//
// For a diagonal observable O invariant under the group G of the basis, <x|O|x> = sum_b |x_b|^2 O(r_b): O takes the
// same value on every state of the orbit of r_b.  σᶻᵢσᶻⱼ is not invariant, but x lies in a one-dimensional irrep, so
// its expectation value equals that of its G-average.  With s_i(r) = +1 / -1 for bit i of r set / clear (σᶻ |1> = |1>):
//     M_ij = sum_b |x_b|^2 s_i(r_b) s_j(r_b),   W = sum_b |x_b|^2,
//     C_ij = 1 / (|G| W) sum_g M[p_g(i), p_g(j)],   m_i = 1 / (|G| W) sum_g (-1)^{f_g} sum_b |x_b|^2 s_{p_g(i)}(r_b)
// (g.s) bit i = s bit p_g(i) followed by a global flip when f_g != 0 (dmv_basis_desc).  The device computes the
// (N + 1) x N block G = sum_b w_b a(r_b) s(r_b)^T with a(r) = (s(r), 1) on the FP64 tensor cores (k_zz_gram); its
// diagonal is W and its last row the one-point sums.  The group average is O(|G| N^2) on the host.
#include <cuda_runtime.h>

#include "dmv_solve.h"

namespace dmv {

int sm_count();                       // dmv_solver.cu
void check_launch(const char *what);

namespace {

constexpr int kZzStates = 512;     // states staged in shared memory per tile

// row tiles of 16 (N sites + the constant row), column tiles of 8 (N sites)
int zz_row_tiles(int n_sites) { return (n_sites + 1 + 15) / 16; }
int zz_col_tiles(int n_sites) { return (n_sites + 7) / 8; }
// warps of a CTA: one row tile each, repeated over `slices` interleaved quarters of the staged states (about 8 warps)
int zz_slices(int n_sites) { return std::max(1, 8 / zz_row_tiles(n_sites)); }

constexpr uint64_t kOne = 0x3FF0000000000000ull;   // 1.0
constexpr uint64_t kSign = 0x8000000000000000ull;

// d += a b for the m16n8k4 FP64 tile (row-major A 16 x 4, column-major B 4 x 8): lane l holds A[l/4][l%4] and
// A[l/4 + 8][l%4], B[l%4][l/4], and D[l/4][2 (l%4) + {0, 1}], D[l/4 + 8][2 (l%4) + {0, 1}]
__device__ __forceinline__ void dmma_16x8x4(double (&d)[4], double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a0), "d"(a1), "d"(b));
}

// partials[blockIdx * RP * CP + i * CP + j] = this CTA's share of G[i][j] = sum_b w_b a_i(r_b) s_j(r_b), padded to
// RP = 16 row_tiles rows and CP = 8 col_tiles columns (zero outside i <= N, j < N).  The k dimension of the mma is
// states: a lane takes state l % 4 of every group of four, builds its A entries (+-1, or 1 in the constant row) and its
// B entries (+-w) from the state word, and the products are exact; the sums run in FP64 in a fixed order.  Warp w owns
// row tile w % row_tiles and every column tile, and walks the groups of four states w / row_tiles, + slices, ...; the
// slices are summed in shared memory in slice order, so a repeated call is bit-identical.
template <bool CE, int CT>
__global__ void __launch_bounds__(256, 1) k_zz_gram(int64_t n, int n_sites, int row_tiles, int slices,
                                                 const uint64_t *__restrict__ reps, const double *__restrict__ x,
                                                 double *__restrict__ partials) {
  extern __shared__ double s_block[];   // [RP][CP]
  __shared__ uint64_t s_rep[kZzStates];
  __shared__ double s_w[kZzStates];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rt = warp % row_tiles, slice = warp / row_tiles;
  constexpr int CP = 8 * CT;
  const int g = lane >> 2, q = lane & 3;
  // the two rows of A this lane holds: a site (sign from the state), the constant row N (1.0) or padding (0.0)
  const int row0 = rt * 16 + g, row1 = row0 + 8;
  const bool site0 = row0 < n_sites, site1 = row1 < n_sites;
  const int sh0 = site0 ? row0 : 0, sh1 = site1 ? row1 : 0;
  const double fixed0 = row0 == n_sites ? 1.0 : 0.0, fixed1 = row1 == n_sites ? 1.0 : 0.0;
  unsigned col_ok = 0;   // bit ct: column ct * 8 + g is a site
#pragma unroll
  for (int ct = 0; ct < CT; ++ct) col_ok |= (ct * 8 + g < n_sites ? 1u : 0u) << ct;
  double acc[CT][4];
#pragma unroll
  for (int ct = 0; ct < CT; ++ct) acc[ct][0] = acc[ct][1] = acc[ct][2] = acc[ct][3] = 0.0;

  for (int64_t base = (int64_t)blockIdx.x * kZzStates; base < n; base += (int64_t)gridDim.x * kZzStates) {
    __syncthreads();   // the previous tile has been consumed
    for (int t = threadIdx.x; t < kZzStates; t += blockDim.x) {
      const int64_t i = base + t;
      uint64_t r = 0;
      double w = 0.0;   // states past the end weigh nothing
      if (i < n) {
        r = reps[i];
        if (CE) { const double2 v = reinterpret_cast<const double2 *>(x)[i]; w = v.x * v.x + v.y * v.y; }
        else { const double v = x[i]; w = v * v; }
      }
      s_rep[t] = r;
      s_w[t] = w;
    }
    __syncthreads();
    for (int k = 4 * slice; k < kZzStates; k += 4 * slices) {
      const uint64_t nr = ~s_rep[k + q];   // bit i of nr set: s_i = -1
      const uint64_t wb = (uint64_t)__double_as_longlong(s_w[k + q]);   // w >= 0: sign bit clear
      const double a0 = site0 ? __longlong_as_double((long long)(kOne | ((nr >> sh0) << 63))) : fixed0;
      const double a1 = site1 ? __longlong_as_double((long long)(kOne | ((nr >> sh1) << 63))) : fixed1;
      const uint64_t u = nr >> g;   // bit 8 ct: the sign of column ct * 8 + g
      double b[CT];
#pragma unroll
      for (int ct = 0; ct < CT; ++ct)
        b[ct] = (col_ok >> ct & 1u) ? __longlong_as_double((long long)(wb | ((u << (63 - 8 * ct)) & kSign))) : 0.0;
#pragma unroll
      for (int ct = 0; ct < CT; ++ct) dmma_16x8x4(acc[ct], a0, a1, b[ct]);
    }
  }
  __syncthreads();
  for (int s = 0; s < slices; ++s) {   // the slices of a row tile, in order
    if (slice == s) {
#pragma unroll
      for (int ct = 0; ct < CT; ++ct) {
        double *p = s_block + (size_t)row0 * CP + ct * 8 + 2 * q;
        if (s == 0) { p[0] = acc[ct][0]; p[1] = acc[ct][1]; p[8 * CP] = acc[ct][2]; p[8 * CP + 1] = acc[ct][3]; }
        else { p[0] += acc[ct][0]; p[1] += acc[ct][1]; p[8 * CP] += acc[ct][2]; p[8 * CP + 1] += acc[ct][3]; }
      }
    }
    __syncthreads();
  }
  const int size = 16 * row_tiles * CP;
  for (int t = threadIdx.x; t < size; t += blockDim.x) partials[(int64_t)blockIdx.x * size + t] = s_block[t];
}

// one wave of resident CTAs over the tiles of states (at least one, so that an empty block still writes its partials);
// launch == true also launches
template <bool CE, int CT>
int zz_run(bool launch, int64_t n, int n_sites, const uint64_t *reps, const double *x, double *partials,
           cudaStream_t s) {
  const int rows = zz_row_tiles(n_sites), slices = zz_slices(n_sites), threads = 32 * rows * slices;
  const size_t smem = (size_t)16 * rows * 8 * CT * sizeof(double);
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_zz_gram<CE, CT>, threads, smem);
  const int64_t tiles = (std::max<int64_t>(n, 0) + kZzStates - 1) / kZzStates;
  const int grid = (int)std::min<int64_t>(std::max<int64_t>(tiles, 1), (int64_t)sm_count() * std::max(per_sm, 1));
  if (launch) k_zz_gram<CE, CT><<<grid, threads, smem, s>>>(n, n_sites, rows, slices, reps, x, partials);
  return grid;
}

template <bool CE>
int zz_dispatch(bool launch, int64_t n, int n_sites, const uint64_t *reps, const double *x, double *partials,
                cudaStream_t s) {
  switch (zz_col_tiles(n_sites)) {
    case 1: return zz_run<CE, 1>(launch, n, n_sites, reps, x, partials, s);
    case 2: return zz_run<CE, 2>(launch, n, n_sites, reps, x, partials, s);
    case 3: return zz_run<CE, 3>(launch, n, n_sites, reps, x, partials, s);
    case 4: return zz_run<CE, 4>(launch, n, n_sites, reps, x, partials, s);
    case 5: return zz_run<CE, 5>(launch, n, n_sites, reps, x, partials, s);
    case 6: return zz_run<CE, 6>(launch, n, n_sites, reps, x, partials, s);
    case 7: return zz_run<CE, 7>(launch, n, n_sites, reps, x, partials, s);
    default: return zz_run<CE, 8>(launch, n, n_sites, reps, x, partials, s);
  }
}

}  // namespace

int zz_gram_columns(int n_sites) { return 8 * zz_col_tiles(n_sites); }
size_t zz_gram_size(int n_sites) { return (size_t)16 * zz_row_tiles(n_sites) * zz_gram_columns(n_sites); }

size_t zz_gram_partials(int64_t n, int n_sites) {
  const int grid = std::max(zz_dispatch<false>(false, n, n_sites, nullptr, nullptr, nullptr, nullptr),
                            zz_dispatch<true>(false, n, n_sites, nullptr, nullptr, nullptr, nullptr));
  return (size_t)grid * zz_gram_size(n_sites);
}

void launch_zz_gram(int64_t n, bool complex_elements, int n_sites, const uint64_t *reps, const double *x,
                    double *partials, double *gram, cudaStream_t s) {
  if (n_sites < 1 || n_sites > 64) throw std::runtime_error("k_zz_gram: 1 to 64 sites");
  const int grid = complex_elements ? zz_dispatch<true>(true, n, n_sites, reps, x, partials, s)
                                    : zz_dispatch<false>(true, n, n_sites, reps, x, partials, s);
  check_launch("k_zz_gram");
  launch_reduce_partials(grid, (int)(zz_gram_size(n_sites) / 2), partials, gram, s);
}

}  // namespace dmv

namespace {

// The group the correlations are averaged over: the permutations and flips of the basis, {1, flip} for spin inversion
// without permutations, {1} without symmetries.
struct ZzGroup {
  int64_t order = 1;
  std::vector<int32_t> perms;   // [order][N]
  std::vector<uint8_t> flips;   // [order]
};

ZzGroup zz_group(int n_sites, bool has_permutations, int64_t group_order, const int32_t *perms, const uint8_t *flips,
                 int spin_inversion) {
  ZzGroup G;
  if (has_permutations) {
    if (group_order < 1 || !perms || !flips) throw std::runtime_error("the basis has permutations but no group tables");
    G.order = group_order;
    G.perms.assign(perms, perms + group_order * n_sites);
    G.flips.assign(flips, flips + group_order);
    return G;
  }
  G.order = spin_inversion != 0 ? 2 : 1;
  for (int64_t e = 0; e < G.order; ++e)
    for (int i = 0; i < n_sites; ++i) G.perms.push_back(i);
  G.flips = spin_inversion != 0 ? std::vector<uint8_t>{0, 1} : std::vector<uint8_t>{0};
  return G;
}

// gram: (N + 1) x N, row-major; correlations N x N, magnetization N (may be null)
void zz_symmetrize(int N, const ZzGroup &G, const double *gram, double *correlations, double *magnetization) {
  const double W = gram[0];   // G[0][0] = sum_b |x_b|^2 s_0^2
  if (!(W > 0.0)) throw std::runtime_error("x is a zero vector: <x|x> = 0");
  std::vector<double> C((size_t)N * N, 0.0), m((size_t)N, 0.0);
  for (int64_t e = 0; e < G.order; ++e) {
    const int32_t *p = G.perms.data() + e * N;
    for (int i = 0; i < N; ++i) {
      const double *row = gram + (size_t)p[i] * N;
      double *out = C.data() + (size_t)i * N;
      for (int j = 0; j < N; ++j) out[j] += row[p[j]];
      m[i] += (G.flips[e] ? -1.0 : 1.0) * gram[(size_t)N * N + p[i]];
    }
  }
  const double scale = 1.0 / ((double)G.order * W);
  for (size_t t = 0; t < C.size(); ++t) correlations[t] = C[t] * scale;
  if (magnetization)
    for (int i = 0; i < N; ++i) magnetization[i] = m[i] * scale;
}

}  // namespace

extern "C" {

// ---- spin-spin correlations (DESIGN.md section 3, "dmv_zz_correlations"): one k_zz_gram pass per vector, the
// (N + 1) x N block all-reduced over the ranks, the group average on the host.
int dmv_zz_correlations(dmv_context *ctx, int elt, int num_vectors, const void *x, double *correlations,
                        double *magnetization) {
  API_BEGIN
  SolverRun run(ctx, elt, "dmv_zz_correlations", false);
  if (num_vectors < 1) throw std::runtime_error("num_vectors must be positive");
  if (!x) throw std::runtime_error("x must not be null");
  if (!correlations) throw std::runtime_error("correlations must not be null");
  const int N = ctx->n_sites;
  const ZzGroup G = zz_group(N, ctx->has_permutations, ctx->k_group_order, ctx->k_perms.data(), ctx->k_flips.data(),
                             ctx->spin_inversion);
  const int64_t n = run.n;
  const size_t words = run.words;
  cudaStream_t st = run.st;
  const size_t size = zz_gram_size(N);
  double *partials = run.partials(zz_gram_partials(n, N)), *d_gram = run.scalars(size);
  const InArg<double> xin(static_cast<const double *>(x), (size_t)num_vectors * words, st);
  std::vector<double> padded(size), gram((size_t)(N + 1) * N);
  std::vector<double> C((size_t)num_vectors * N * N), m((size_t)num_vectors * N);
  for (int v = 0; v < num_vectors; ++v) {
    // d_reps holds the states of every basis, the identity-index one included (dmv_basis_build enumerates them all)
    launch_zz_gram(n, run.ce, N, ctx->d_reps.ptr, xin.ptr + (size_t)v * words, partials, d_gram, st);
    run.all_reduce(d_gram, size);
    CUDA_CHECK(cudaMemcpyAsync(padded.data(), d_gram, size * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    const int CP = zz_gram_columns(N);
    for (int i = 0; i <= N; ++i)
      for (int j = 0; j < N; ++j) gram[(size_t)i * N + j] = padded[(size_t)i * CP + j];
    zz_symmetrize(N, G, gram.data(), C.data() + (size_t)v * N * N, m.data() + (size_t)v * N);
  }
  CUDA_CHECK(cudaMemcpyAsync(correlations, C.data(), C.size() * sizeof(double), cudaMemcpyDefault, st));
  if (magnetization)
    CUDA_CHECK(cudaMemcpyAsync(magnetization, m.data(), m.size() * sizeof(double), cudaMemcpyDefault, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  API_END
}

// host-only self-check entry for the group average behind dmv_zz_correlations (no device needed)
int dmv_debug_zz_symmetrize(const dmv_basis_desc *basis, const double *gram, double *correlations,
                            double *magnetization) {
  API_BEGIN
  if (!basis || !gram || !correlations) throw std::runtime_error("basis, gram and correlations must not be null");
  const int N = basis->number_sites;
  if (N < 1 || N > 64) throw std::runtime_error("number_sites must be between 1 and 64");
  const ZzGroup G = zz_group(N, basis->has_permutations != 0, basis->group_order, basis->perms, basis->flips,
                             basis->spin_inversion);
  zz_symmetrize(N, G, gram, correlations, magnetization);
  API_END
}

}  // extern "C"
