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

namespace {

constexpr int kZzStates = 512;     // states staged in shared memory per tile

// row tiles of 32 of a reduced density matrix block of dimension d (dmv_reduced_density_matrix, below)
__host__ __device__ __forceinline__ int rdm_macro_dev(int d) { return (d + 31) / 32; }

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

// a k_zz_gram CTA: a warp per row tile and slice, the CTA's block of the Gram matrix in shared memory
int zz_threads(int n_sites) { return 32 * zz_row_tiles(n_sites) * zz_slices(n_sites); }
size_t zz_smem(int n_sites) { return (size_t)16 * zz_row_tiles(n_sites) * 8 * zz_col_tiles(n_sites) * sizeof(double); }

// one wave of resident CTAs of `kernel` over the tiles of n states (at least one, so that an empty block still writes
// its partials)
template <typename K>
int zz_grid(K kernel, int64_t n, int n_sites) {
  return one_wave(kernel, (std::max<int64_t>(n, 0) + kZzStates - 1) / kZzStates, zz_smem(n_sites), zz_threads(n_sites));
}

// f(k_zz_gram<CE, CT>) for the column tiles CT of n_sites
template <typename F>
auto with_zz_gram(bool complex_elements, int n_sites, F &&f) {
  return with_bool(complex_elements, [&](auto ce) {
    return with_choice<1, 2, 3, 4, 5, 6, 7, 8>(zz_col_tiles(n_sites), [&](auto ct) { return f(k_zz_gram<ce(), ct()>); });
  });
}

// ---- the look-up of the observables (k_pm_*, k_spin_rows, k_rdm_fill): chi (n x)[rep(a)] at any state a of a basis's
// sector, through StateLookup::at.  The host half (ObservableLookup, below) picks the build and fills the struct.
enum LookupKind {
  LOOK_NONE = 0,        // no symmetry: the index of the basis
  LOOK_INVERSION = 1,   // spin inversion alone: min(a, flip a), the character when flipped
  LOOK_GROUP = 2,       // permutations: orbit minimum (orbit_scan and its character when they are not trivial), the index
  LOOK_TABLE = 3,       // permutations, trivial characters: orbit minimum, then k_rows' hash table (x n in the slot)
};

template <bool CE>
__device__ __forceinline__ double2 pm_load(const double *x, int64_t i) {
  if constexpr (CE) return __ldg(reinterpret_cast<const double2 *>(x) + i);
  else return make_double2(__ldg(x + i), 0.0);
}

struct StateLookup {
  StateIndex index;          // the basis the states are looked up in: this rank's, or the whole basis on several ranks
  OrbitProgram orbit;
  const double *norms;       // of index's states
  const uint32_t *pos;       // several ranks: global index g lives at x[pos[g]]; null on one rank
  const double *x;           // the vector (the gathered one on several ranks)
  uint64_t site_mask;        // the basis's sites, all flipped by spin inversion
  double inversion_character;
  const unsigned char *table;   // LOOK_TABLE: k_rows' table (table_slot / ordered layout), filled from x
  uint32_t table_slots;
  OrderedDir table_dir;
  DenseOrder dord;              // ... or the dense ordered table (blocks not null), its slots in `dense`
  const unsigned char *dense;
  unsigned long long *status;

  // chi (n x)[rep(a)]; a state outside the basis is counted in bad / bad_state unless its projection vanishes (a
  // stabiliser sum of zero under non-trivial characters), which contributes nothing
  template <int LOOK, int TK, bool CE>
  __device__ __forceinline__ double2 at(uint64_t a, unsigned long long &bad, uint64_t &bad_state) const {
    double2 chi = make_double2(1.0, 0.0);
    uint64_t key = a;
    if constexpr (LOOK == LOOK_INVERSION) {
      const uint64_t inv = a ^ site_mask;
      if (inv < a) { key = inv; chi.x = inversion_character; }
    } else if constexpr (LOOK == LOOK_GROUP || LOOK == LOOK_TABLE) {
      if (LOOK == LOOK_TABLE || orbit.trivial_characters) {
        if constexpr (TK > 0) key = orbit_min_torus_sq<TK>(orbit, a);
        else key = orbit_representative(orbit, a);
      } else {
        const OrbitResult r = orbit_scan<false, false>(orbit, a);
        key = r.rep;
        chi = __ldg(orbit.characters + r.arg);   // chi(g), not conjugated: the convention of k_pull
      }
    }
    if constexpr (LOOK == LOOK_TABLE) {
      if (dord.blocks != nullptr) {   // dense ordered table: the rank block, then the slot (or the block's leftovers)
        const uint64_t h = dord_hash(key);
        const uint32_t p = ordered_block(key, table_dir.k_lo, table_dir.shift, table_dir.last);
        const uint64_t *w = dord.blocks + 4 * (size_t)dord_block(h, __ldg(table_dir.dir + p), __ldg(table_dir.dir + p + 1));
        uint32_t end = 0;
        for (uint32_t s = dord_slot(__ldg(w), __ldg(w + 1), __ldg(w + 2), __ldg(w + 3), dord_bits(h), end); s < end; ++s) {
          const size_t width = CE ? 32 : 16;
          const ulonglong2 kv = __ldg(reinterpret_cast<const ulonglong2 *>(dense + s * width));
          if (kv.x != key) continue;
          if (CE) return __ldg(reinterpret_cast<const double2 *>(dense + s * width + 16));
          return make_double2(__longlong_as_double((long long)kv.y), 0.0);
        }
        ++bad; bad_state = key;
        return make_double2(0.0, 0.0);
      }
      uint32_t bk = table_home(key, table_slots, table_dir);
      for (;;) {
        const ulonglong2 k = __ldg(reinterpret_cast<const ulonglong2 *>(table + (size_t)bk * 32));
        const double2 v = __ldg(reinterpret_cast<const double2 *>(table + (size_t)bk * 32 + 16));
        if (CE) {   // { key, spare, re, im }
          if (k.x == key) return v;
          if (k.x == kEmptyKey) break;
        } else {    // { key0, key1, value0, value1 }
          if (k.x == key) return make_double2(v.x, 0.0);
          if (k.y == key) return make_double2(v.y, 0.0);
          if (k.x == kEmptyKey || k.y == kEmptyKey) break;
        }
        bk = bk + 1 == table_slots ? 0 : bk + 1;
      }
      ++bad; bad_state = key;
      return make_double2(0.0, 0.0);
    } else {
      const int64_t idx = locate(index, key);
      if (idx < 0) {
        if (LOOK != LOOK_GROUP || orbit.trivial_characters ||
            orbit_stabiliser_sum(orbit, key) > 1e-12 * (double)orbit.group_order) { ++bad; bad_state = key; }
        return make_double2(0.0, 0.0);
      }
      double2 v = pm_load<CE>(x, pos ? (int64_t)__ldg(pos + idx) : idx);
      if constexpr (LOOK == LOOK_GROUP) {
        const double nrm = __ldg(norms + idx);
        v = make_double2(v.x * nrm, v.y * nrm);
      }
      return make_double2(chi.x * v.x - chi.y * v.y, chi.x * v.y + chi.y * v.x);
    }
  }
};

// the states a kernel found outside the basis: status[0] counts them, status[1] holds one of them
__device__ __forceinline__ void report_bad(unsigned long long *status, unsigned long long bad, uint64_t bad_state) {
  if (bad && atomicAdd(status, bad) == 0) status[1] = bad_state;
}

// f(lk, tk, ce): the look-up builds (LOOK, TK, CE) as compile-time constants.  TK, the square-torus orbit minimum
// (rows_torus_k: 6, 4 or 0), exists only for the orbit look-ups, LOOK >= LOOK_GROUP.
template <typename F>
void with_lookup(const char *kernel, int look, int tk, bool ce, F &&f) {
  with_choice<LOOK_NONE, LOOK_INVERSION, LOOK_GROUP, LOOK_TABLE>(look, [&](auto lk) {
    with_bool(ce, [&](auto e) {
      with_choice<6, 4, 0>(tk, [&](auto t) {
        if constexpr (lk() >= LOOK_GROUP || t() == 0) f(lk, t, e);
        else throw std::logic_error(std::string(kernel) + " has no square-torus build without a group");
      });
    });
  });
}

// ---- flip-flop correlations (dmv_pm_correlations).  A row b and an antiparallel pair (i, j) with bit i of b set and
// bit j clear give the term conj(x_b) / n_b chi (n x)[rep(b ^ (1 << i | 1 << j))] of the class of the ordered pair
// (i, j); the host turns the class sums into <σ⁺ᵢσ⁻ⱼ>.  The rows are the looked-up basis's own (this rank's share).
struct PmArgs {
  StateLookup look;
  const uint64_t *rows;      // this rank's representatives and their norms
  const double *row_norms;
  int64_t n_rows, x_row_offset;
  const int16_t *class_of;   // [N * N]: class of the ordered pair (i, j), -1 on the diagonal
  const uint16_t *pairs;     // pair-major walk: the unordered pairs i | j << 8
  int n_sites, n_pairs, c_lo, c_hi;   // classes [c_lo, c_hi) of this pass
  double *partials;          // [grid][c_hi - c_lo][2]
};

// conj(x_b) / n_b of row i
template <int LOOK, bool CE>
__device__ __forceinline__ double2 pm_row_factor(const PmArgs &A, int64_t i) {
  const double2 v = pm_load<CE>(A.look.x, A.x_row_offset + i);
  const double s = LOOK >= LOOK_GROUP ? 1.0 / __ldg(A.row_norms + i) : 1.0;
  return make_double2(v.x * s, -v.y * s);
}

// Lane-major walk (bases with permutations: few classes).  One lane owns one row and walks all its antiparallel pairs
// (w (N - w) at a fixed Hamming weight, the same for every lane).  Lane-private class slots in shared memory,
// [class][thread] (real parts, then imaginary parts when CPLX), are summed in thread order = lane order, then warp order.
template <int LOOK, int TK, bool CE, bool CPLX>
__global__ void __launch_bounds__(256, 2) k_pm_rows(const PmArgs A) {
  extern __shared__ double s_slot[];
  const int T = blockDim.x, t = threadIdx.x, C = A.c_hi - A.c_lo, N = A.n_sites;
  for (int c = 0; c < C * (CPLX ? 2 : 1); ++c) s_slot[c * T + t] = 0.0;
  unsigned long long bad = 0;
  uint64_t bad_state = 0;
  for (int64_t i = (int64_t)blockIdx.x * T + t; i < A.n_rows; i += (int64_t)gridDim.x * T) {
    const uint64_t b = __ldg(A.rows + i);
    const double2 xb = pm_row_factor<LOOK, CE>(A, i);
    for (uint64_t up = b & A.look.site_mask; up; up &= up - 1) {
      const int si = __ffsll((long long)up) - 1;
      const int16_t *cls = A.class_of + si * N;
      for (uint64_t dn = ~b & A.look.site_mask; dn; dn &= dn - 1) {
        const int sj = __ffsll((long long)dn) - 1;
        const int c = (int)__ldg(cls + sj) - A.c_lo;
        if ((unsigned)c >= (unsigned)C) continue;
        const double2 v = A.look.at<LOOK, TK, CE>(b ^ (1ull << si) ^ (1ull << sj), bad, bad_state);
        s_slot[c * T + t] += xb.x * v.x - xb.y * v.y;
        if constexpr (CPLX) s_slot[(C + c) * T + t] += xb.x * v.y + xb.y * v.x;
      }
    }
  }
  __syncthreads();
  for (int c = t; c < C; c += T) {
    double re = 0.0, im = 0.0;
    for (int u = 0; u < T; ++u) {
      re += s_slot[c * T + u];
      if constexpr (CPLX) im += s_slot[(C + c) * T + u];
    }
    A.partials[((int64_t)blockIdx.x * C + c) * 2] = re;
    A.partials[((int64_t)blockIdx.x * C + c) * 2 + 1] = im;
  }
  report_bad(A.look.status, bad, bad_state);
}

// Pair-major walk (bases without permutations: a class per ordered pair, or per {(i, j), (j, i)} with spin inversion).
// The CTA's warps share a tile of 32 rows, one per lane; warp w takes the unordered pairs w, w + warps, ..., every lane
// adds its row's term and the warp sums them by shuffles in a fixed order, one sum per direction of the pair.  The
// classes of an unordered pair belong to one warp only, so lane 0 owns their slots in shared memory.
// JW (fermionic bases, LOOK_NONE only): the term of c†ᵢcⱼ carries the Jordan-Wigner sign (-1)^popc(b & between(i, j)),
// the bits strictly between the two modes; b and its target agree there, so both directions of a pair take one sign.
template <int LOOK, bool CE, bool JW>
__global__ void __launch_bounds__(256) k_pm_pairs(const PmArgs A) {
  extern __shared__ double s_cls[];   // [classes] real parts, then imaginary parts
  const int C = A.c_hi, N = A.n_sites, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) s_cls[c] = 0.0;
  __syncthreads();
  unsigned long long bad = 0;
  uint64_t bad_state = 0;
  for (int64_t tile = blockIdx.x; tile * 32 < A.n_rows; tile += gridDim.x) {
    const int64_t i = tile * 32 + lane;
    const bool valid = i < A.n_rows;
    const uint64_t b = valid ? __ldg(A.rows + i) : 0ull;
    const double2 xb = valid ? pm_row_factor<LOOK, CE>(A, i) : make_double2(0.0, 0.0);
    for (int p = warp; p < A.n_pairs; p += warps) {
      const unsigned pr = __ldg(A.pairs + p), si = pr & 0xffu, sj = pr >> 8;
      const bool bi = (b >> si) & 1ull, bj = (b >> sj) & 1ull;
      double2 c = make_double2(0.0, 0.0);
      if (valid && bi != bj) {
        const double2 v = A.look.at<LOOK, 0, CE>(b ^ (1ull << si) ^ (1ull << sj), bad, bad_state);
        c = make_double2(xb.x * v.x - xb.y * v.y, xb.x * v.y + xb.y * v.x);
        if constexpr (JW) {   // pairs are stored with si < sj
          const uint64_t between = ((1ull << sj) - 1) & ~((2ull << si) - 1);
          if (__popcll(b & between) & 1) c = make_double2(-c.x, -c.y);
        }
      }
      double s[4] = {bi ? c.x : 0.0, bi ? c.y : 0.0, bi ? 0.0 : c.x, bi ? 0.0 : c.y};   // (i, j), then (j, i)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int k = 0; k < 4; ++k) s[k] += __shfl_xor_sync(0xffffffffu, s[k], off);
      if (lane == 0) {
        const int cij = __ldg(A.class_of + si * N + sj), cji = __ldg(A.class_of + sj * N + si);
        s_cls[cij] += s[0]; s_cls[C + cij] += s[1];
        s_cls[cji] += s[2]; s_cls[C + cji] += s[3];
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    A.partials[((int64_t)blockIdx.x * C + c) * 2] = s_cls[c];
    A.partials[((int64_t)blockIdx.x * C + c) * 2 + 1] = s_cls[C + c];
  }
  report_bad(A.look.status, bad, bad_state);
}

constexpr size_t kPmSmem = 96 * 1024;   // shared memory of one CTA: two CTAs per SM
constexpr int kPmThreads = 256;

// f(kernel) for the walk the basis asks for: k_pm_pairs<LOOK, CE, JW> without permutations, else k_pm_rows<LOOK, TK,
// CE, CPLX>.  The class sums are complex (CPLX) with complex vectors or characters; LOOK_TABLE runs on trivial
// characters only, so there CPLX == CE.  JW (fermionic bases) only with LOOK_NONE.
template <typename F>
void with_pm_kernel(int look, int tk, bool ce, bool cplx, bool jw, F &&f) {
  with_lookup("k_pm_rows", look, tk, ce, [&](auto lk, auto t, auto e) {
    if (jw && lk() != LOOK_NONE) throw std::logic_error("k_pm_pairs has Jordan-Wigner builds only without symmetries");
    if constexpr (lk() == LOOK_NONE) {
      with_bool(jw, [&](auto j) { f(k_pm_pairs<LOOK_NONE, e(), j()>); });
    } else if constexpr (lk() == LOOK_INVERSION) {
      f(k_pm_pairs<LOOK_INVERSION, e(), false>);
    } else {
      with_bool(cplx, [&](auto cx) {
        if constexpr (lk() == LOOK_TABLE ? cx() == e() : cx() || !e()) f(k_pm_rows<lk(), t(), e(), cx()>);
        else throw std::logic_error("k_pm_rows has no build for these sums");
      });
    }
  });
}

// ---- one-site operators between two bases (dmv_apply_spin).  Row r of the target basis is
//     y_r = 1 / n_t(r) sum_k K_k <r| o_k |psi>,   psi = B_s x,
// with o_k = σ⁺_k on the set bits of r and σ⁻_k on its clear bits (the source state r ^ (1 << k)), or the diagonal
// factor sum_k K_k s_k(r) (σᶻ) or sum_k K_k (1).  StateLookup::at gives psi at any state of the source's sector: chi
// (n x)[rep] with the orbit minimum and character of the source (LOOK_GROUP, LOOK_TABLE), x[index] without a group
// (LOOK_NONE), chi x[index] with spin inversion alone, whose norm sqrt(1/2) is src_scale.  The host forms K
// (spin_weights below).
enum SpinWalk {
  SPIN_SELF = 0,    // σᶻ / 1: the row's own state, times c0 + sum over its set bits of k_set + over its clear bits of k_clear
  SPIN_CLEAR = 1,   // σ⁻: the clear bits of the row (k_clear)
  SPIN_SET = 2,     // σ⁺: the set bits (k_set)
  SPIN_BOTH = 3,    // σ^± with spin inversion in the target group at free weight: both, each with its own coefficients
};

struct SpinArgs {
  StateLookup src;            // the source's look-up
  const uint64_t *rows;       // this rank's rows of the target basis and their norms (null: row_norm for every row)
  const double *row_norms;
  double row_norm, src_scale;
  const double *k;            // [2][N] complex: k_set, then k_clear
  double2 c0;
  uint64_t walk_mask;         // SPIN_SET / SPIN_CLEAR / SPIN_BOTH: the sites (modes) the walk visits
  uint64_t diag_mask;         // SPIN_SELF: the sites whose k_set / k_clear enter the row factor (0 for the identity)
  int64_t n_rows;
  int n_sites;
  double *y;
};

// One lane owns one row of the target basis and walks its sites; one store of y per row, no atomics.
// JW (dmv_apply_fermion, LOOK_NONE with SPIN_SET / SPIN_CLEAR only): the walk is c†_k on the set bits or c_k on the
// clear bits of the row, each term with the Jordan-Wigner sign (-1)^popc(r & ((1 << k) - 1)); walk_mask holds the modes
// the walk visits (one spin half of a spinful basis).
template <int LOOK, int TK, int WALK, bool CE, bool JW>
__global__ void __launch_bounds__(256, 2) k_spin_rows(const SpinArgs A) {
  __shared__ double2 s_k[128];   // k_set [0, N), k_clear [N, 2 N)
  const int N = A.n_sites;
  for (int t = threadIdx.x; t < 2 * N; t += blockDim.x) s_k[t] = __ldg(reinterpret_cast<const double2 *>(A.k) + t);
  __syncthreads();
  unsigned long long bad = 0;
  uint64_t bad_state = 0;
  const uint64_t mask = A.walk_mask;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n_rows; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t r = __ldg(A.rows + i);
    double2 acc = make_double2(0.0, 0.0);
    auto add = [&](double2 k, double2 v) {
      acc.x += k.x * v.x - (CE ? k.y * v.y : 0.0);
      if constexpr (CE) acc.y += k.x * v.y + k.y * v.x;
    };
    auto string_sign = [&](double2 k, int mode) {   // k times the Jordan-Wigner sign of `mode` on r
      if constexpr (JW)
        if (__popcll(r & ((1ull << mode) - 1)) & 1) return make_double2(-k.x, -k.y);
      return k;
    };
    if constexpr (WALK == SPIN_SELF) {
      double2 c = A.c0;
      for (uint64_t m = r & A.diag_mask; m; m &= m - 1) {
        const double2 k = s_k[__ffsll((long long)m) - 1];
        c.x += k.x; c.y += k.y;
      }
      for (uint64_t m = ~r & A.diag_mask; m; m &= m - 1) {
        const double2 k = s_k[N + __ffsll((long long)m) - 1];
        c.x += k.x; c.y += k.y;
      }
      add(c, A.src.at<LOOK, TK, CE>(r, bad, bad_state));
    } else {
      if constexpr (WALK & SPIN_SET)
        for (uint64_t m = r & mask; m; m &= m - 1) {
          const int k = __ffsll((long long)m) - 1;
          add(string_sign(s_k[k], k), A.src.at<LOOK, TK, CE>(r ^ (1ull << k), bad, bad_state));
        }
      if constexpr (WALK & SPIN_CLEAR)
        for (uint64_t m = ~r & mask; m; m &= m - 1) {
          const int k = __ffsll((long long)m) - 1;
          add(string_sign(s_k[N + k], k), A.src.at<LOOK, TK, CE>(r ^ (1ull << k), bad, bad_state));
        }
    }
    const double s = A.src_scale / (A.row_norms ? __ldg(A.row_norms + i) : A.row_norm);
    if constexpr (CE) reinterpret_cast<double2 *>(A.y)[i] = make_double2(acc.x * s, acc.y * s);
    else A.y[i] = acc.x * s;
  }
  report_bad(A.src.status, bad, bad_state);
}

constexpr int kSpinThreads = 256;

// f(k_spin_rows<LOOK, TK, WALK, CE, JW>); JW only for LOOK_NONE with the set-bit or clear-bit walk
template <typename F>
void with_spin_kernel(int look, int tk, int walk, bool ce, bool jw, F &&f) {
  with_lookup("k_spin_rows", look, tk, ce, [&](auto lk, auto t, auto e) {
    with_choice<SPIN_SELF, SPIN_CLEAR, SPIN_SET, SPIN_BOTH>(walk, [&](auto wk) {
      if constexpr (lk() == LOOK_NONE && (wk() == SPIN_SET || wk() == SPIN_CLEAR))
        with_bool(jw, [&](auto j) { f(k_spin_rows<lk(), t(), wk(), e(), j()>); });
      else if (jw)
        throw std::logic_error("k_spin_rows has Jordan-Wigner builds only for the set-bit and clear-bit walks "
                               "without symmetries");
      else
        f(k_spin_rows<lk(), t(), wk(), e(), false>);
    });
  });
}

// ---- reduced density matrices (dmv_reduced_density_matrix).  At a fixed Hamming weight W, ρ_A = Tr_B |ψ><ψ| is block
// diagonal in the weight w of A; block w is Ψ Ψᴴ with Ψ[a, b] = ψ(embed_A(a) | embed_B(b)) over the configurations a of A
// of weight w and b of B of weight W - w.  The columns b are cut into chunks; k_rdm_fill writes the amplitudes of a
// chunk, row-major with `ld` columns (zeros past the chunk's last column), and k_rdm_gram adds Ψ Ψᴴ on the FP64 tensor
// cores.
struct RdmArgs {
  StateLookup src;             // the basis's look-up
  const uint64_t *embed_a;     // [d]: the states of A's rows, deposited on A's sites
  const uint64_t *binom;       // [64][65]: C(n, k) (B's columns at a fixed weight)
  uint64_t sites_b[64];        // site of bit j of a B configuration, as a one-bit mask
  double scale;                // the source's src_scale (spin inversion alone: sqrt(1/2))
  int64_t col0, cols, ld;      // first column (rank of b) of the chunk, its columns, row stride of psi
  int d, n_b, k_b;             // rows, sites of B, ones of B (-1: free weight, b = the column itself)
  double *psi;
};

constexpr int kRdmRowGroup = 16;   // rows of one column a lane fills (the column's configuration is unranked once)

// b of column r: the r-th configuration of k ones on n_b sites in ascending numeric order (combinadic), on B's sites
__device__ __forceinline__ uint64_t rdm_column_state(const RdmArgs &A, uint64_t r) {
  uint64_t s = 0;
  if (A.k_b < 0) {
    for (uint64_t m = r; m; m &= m - 1) s |= A.sites_b[__ffsll((long long)m) - 1];
    return s;
  }
  int k = A.k_b;
  for (int pos = A.n_b - 1; pos >= 0 && k > 0; --pos) {
    const uint64_t c = __ldg(A.binom + pos * 65 + k);
    if (c <= r) { s |= A.sites_b[pos]; r -= c; --k; }
  }
  return s;
}

// psi[a * ld + c] = scale chi (n x)[rep(embed_A(a) | b_c)] for c < cols, 0 for cols <= c < ld.  A lane owns a column and
// a group of kRdmRowGroup rows; a state outside the basis whose projection does not vanish goes to status.
template <int LOOK, int TK, bool CE>
__global__ void __launch_bounds__(256, 2) k_rdm_fill(const RdmArgs A) {
  unsigned long long bad = 0;
  uint64_t bad_state = 0;
  const int64_t groups = (A.d + kRdmRowGroup - 1) / kRdmRowGroup, work = groups * A.ld;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < work; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = t % A.ld;
    const int a0 = (int)(t / A.ld) * kRdmRowGroup, a1 = min(A.d, a0 + kRdmRowGroup);
    const bool live = c < A.cols;
    const uint64_t b = live ? rdm_column_state(A, (uint64_t)(A.col0 + c)) : 0;
    for (int a = a0; a < a1; ++a) {
      double2 v = make_double2(0.0, 0.0);
      if (live) v = A.src.at<LOOK, TK, CE>(__ldg(A.embed_a + a) | b, bad, bad_state);
      if constexpr (CE) reinterpret_cast<double2 *>(A.psi)[a * A.ld + c] = make_double2(v.x * A.scale, v.y * A.scale);
      else A.psi[a * A.ld + c] = v.x * A.scale;
    }
  }
  report_bad(A.src.status, bad, bad_state);
}

constexpr int kRdmThreads = 256;

template <typename F>
void with_rdm_fill(int look, int tk, bool ce, F &&f) {
  with_lookup("k_rdm_fill", look, tk, ce, [&](auto lk, auto t, auto e) { f(k_rdm_fill<lk(), t(), e()>); });
}

// Block tiles of 32 x 32 of ρ: a CTA per tile on or above the diagonal (I <= J) and per slice of the chunk's columns.
constexpr int kRdmTile = 32;
constexpr int kRdmTarget = 1024;   // CTAs a chunk is split into at most (tiles x slices), fixed so that sums never move

int64_t rdm_tiles(int d) { const int64_t M = rdm_macro_dev(d); return M * (M + 1) / 2; }
// slices of a chunk of `ld` columns, and the columns of one (a multiple of 32: the eight warps take four each)
int rdm_slices(int d, int64_t ld) {
  const int64_t by_tiles = (kRdmTarget + rdm_tiles(d) - 1) / rdm_tiles(d), by_cols = std::max<int64_t>(1, ld / 256);
  return (int)std::max<int64_t>(1, std::min(by_tiles, by_cols));
}
int64_t rdm_slice_cols(int d, int64_t ld) {
  const int S = rdm_slices(d, ld);
  return (ld + 32 * S - 1) / (32 * S) * 32;
}

// partials[(s * tiles + t) * 1024 * (CE ? 2 : 1) + ...] = slice s's share of tile t = (I, J) of Ψ Ψᴴ: real parts
// [32][32], then (CE) imaginary parts.  Warp w walks the groups of four columns w, w + 8, ... of the slice and holds
// the 2 x 4 mma tiles of 16 x 8 in registers; the warps are summed in shared memory in warp order.  With Ψ = R + i I,
// Re = R Rᵀ + I Iᵀ and Im = I Rᵀ - R Iᵀ (four real products per element); real elements take R Rᵀ alone.
template <bool CE>
__global__ void __launch_bounds__(256, 1) k_rdm_gram(const double *__restrict__ psi, int64_t ld, int d, int64_t cols,
                                                   int64_t slice_cols, double *__restrict__ partials) {
  __shared__ double s_blk[(CE ? 2 : 1) * kRdmTile * kRdmTile];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
  const int M = rdm_macro_dev(d);
  int t = blockIdx.x, I = 0;
  while (t >= M - I) { t -= M - I; ++I; }
  const int J = I + t;
  // rows of A (tile I) and of B (tile J) this lane reads: row tile rt rows rt * 16 + g, + 8; column tile ct row ct * 8 + g
  int64_t ra[4], rb[4];
  bool oka[4], okb[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int r = I * kRdmTile + (u >> 1) * 16 + (u & 1) * 8 + g, c = J * kRdmTile + u * 8 + g;
    oka[u] = r < d; okb[u] = c < d;
    ra[u] = (int64_t)(oka[u] ? r : 0) * ld; rb[u] = (int64_t)(okb[u] ? c : 0) * ld;
  }
  double re[2][4][4], im[2][4][4];
#pragma unroll
  for (int rt = 0; rt < 2; ++rt)
#pragma unroll
    for (int ct = 0; ct < 4; ++ct)
#pragma unroll
      for (int e = 0; e < 4; ++e) re[rt][ct][e] = im[rt][ct][e] = 0.0;
  const int64_t k0 = (int64_t)blockIdx.y * slice_cols, k1 = min(cols, k0 + slice_cols);
#pragma unroll(CE ? 1 : 2)   // complex: 64 accumulators, no room for a second group's fragments
  for (int64_t kw = k0 + 4 * warp; kw < k1; kw += 32) {   // warp-uniform: k1 - k0 is a multiple of 32
    const int64_t k = kw + q;
    double ar[4], ai[4], br[4], bi[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if constexpr (CE) {
        const double2 va = oka[u] ? __ldg(reinterpret_cast<const double2 *>(psi) + ra[u] + k) : make_double2(0.0, 0.0);
        const double2 vb = okb[u] ? __ldg(reinterpret_cast<const double2 *>(psi) + rb[u] + k) : make_double2(0.0, 0.0);
        ar[u] = va.x; ai[u] = va.y; br[u] = vb.x; bi[u] = vb.y;
      } else {
        ar[u] = oka[u] ? __ldg(psi + ra[u] + k) : 0.0;
        br[u] = okb[u] ? __ldg(psi + rb[u] + k) : 0.0;
        ai[u] = bi[u] = 0.0;
      }
    }
#pragma unroll
    for (int rt = 0; rt < 2; ++rt)
#pragma unroll
      for (int ct = 0; ct < 4; ++ct) {
        dmma_16x8x4(re[rt][ct], ar[2 * rt], ar[2 * rt + 1], br[ct]);
        if constexpr (CE) {
          dmma_16x8x4(re[rt][ct], ai[2 * rt], ai[2 * rt + 1], bi[ct]);
          dmma_16x8x4(im[rt][ct], ai[2 * rt], ai[2 * rt + 1], br[ct]);
          dmma_16x8x4(im[rt][ct], -ar[2 * rt], -ar[2 * rt + 1], bi[ct]);
        }
      }
  }
  for (int w = 0; w < 8; ++w) {   // the warps, in order
    if (warp == w) {
#pragma unroll
      for (int rt = 0; rt < 2; ++rt)
#pragma unroll
        for (int ct = 0; ct < 4; ++ct)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = rt * 16 + g + (e >> 1) * 8, j = ct * 8 + 2 * q + (e & 1);
            double *p = s_blk + i * kRdmTile + j;
            if (w == 0) { p[0] = re[rt][ct][e]; if (CE) p[kRdmTile * kRdmTile] = im[rt][ct][e]; }
            else { p[0] += re[rt][ct][e]; if (CE) p[kRdmTile * kRdmTile] += im[rt][ct][e]; }
          }
    }
    __syncthreads();
  }
  constexpr int size = (CE ? 2 : 1) * kRdmTile * kRdmTile;
  double *out = partials + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * size;
  for (int e = threadIdx.x; e < size; e += blockDim.x) out[e] = s_blk[e];
}

// acc[2 (i d + j) + {0, 1}] += sum over the slices s in order of partials (i <= j's tile, i, j < d): one thread per
// element of the computed tiles
template <bool CE>
__global__ void __launch_bounds__(256) k_rdm_reduce(const double *__restrict__ partials, int slices, int64_t tiles,
                                                    int d, double *__restrict__ acc) {
  constexpr int size = (CE ? 2 : 1) * kRdmTile * kRdmTile;
  const int M = rdm_macro_dev(d);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tiles * kRdmTile * kRdmTile;
       e += (int64_t)gridDim.x * blockDim.x) {
    int t = (int)(e / (kRdmTile * kRdmTile)), I = 0;
    const int f = (int)(e % (kRdmTile * kRdmTile));
    while (t >= M - I) { t -= M - I; ++I; }
    const int i = I * kRdmTile + f / kRdmTile, j = (I + t) * kRdmTile + f % kRdmTile;
    if (i >= d || j >= d) continue;
    const int64_t base = (e / (kRdmTile * kRdmTile)) * size + f;
    double re = 0.0, im = 0.0;
    for (int s = 0; s < slices; ++s) {
      re += partials[(int64_t)s * tiles * size + base];
      if (CE) im += partials[(int64_t)s * tiles * size + base + kRdmTile * kRdmTile];
    }
    acc[2 * ((int64_t)i * d + j)] += re;
    if (CE) acc[2 * ((int64_t)i * d + j) + 1] += im;
  }
}

// out = scale ρ with the lower triangle mirrored from the upper one (conj) and a real diagonal
__global__ void __launch_bounds__(256) k_rdm_finish(const double *__restrict__ acc, int d, double scale,
                                                    double *__restrict__ out) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)d * d;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / d), j = (int)(e % d);
    const double *p = acc + 2 * (i <= j ? e : (int64_t)j * d + i);
    out[2 * e] = p[0] * scale;
    out[2 * e + 1] = i == j ? 0.0 : (i < j ? p[1] : -p[1]) * scale;
  }
}

}  // namespace

int zz_gram_columns(int n_sites) { return 8 * zz_col_tiles(n_sites); }
size_t zz_gram_size(int n_sites) { return (size_t)16 * zz_row_tiles(n_sites) * zz_gram_columns(n_sites); }

size_t zz_gram_partials(int64_t n, int n_sites) {
  auto grid = [&](bool ce) { return with_zz_gram(ce, n_sites, [&](auto kernel) { return zz_grid(kernel, n, n_sites); }); };
  return (size_t)std::max(grid(false), grid(true)) * zz_gram_size(n_sites);
}

void launch_zz_gram(int64_t n, bool complex_elements, int n_sites, const uint64_t *reps, const double *x,
                    double *partials, double *gram, cudaStream_t s) {
  if (n_sites < 1 || n_sites > 64) throw std::runtime_error("k_zz_gram: 1 to 64 sites");
  with_zz_gram(complex_elements, n_sites, [&](auto kernel) {
    const int grid = zz_grid(kernel, n, n_sites);
    kernel<<<grid, zz_threads(n_sites), zz_smem(n_sites), s>>>(n, n_sites, zz_row_tiles(n_sites), zz_slices(n_sites),
                                                                reps, x, partials);
    check_launch("k_zz_gram");
    launch_reduce_partials(grid, (int)(zz_gram_size(n_sites) / 2), partials, gram, s);
  });
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

// W = <x|x> (the return value), C and m of one vector of this rank: k_zz_gram over this rank's rows, the block
// all-reduced over the ranks, the group average on the host.  partials: zz_gram_partials doubles, d_gram: zz_gram_size.
double zz_moments(SolverRun &run, const ZzGroup &G, const double *xv, double *partials, double *d_gram, double *C,
                  double *m) {
  const int N = run.ctx->n_sites;
  const size_t size = zz_gram_size(N);
  std::vector<double> padded(size), gram((size_t)(N + 1) * N);
  // d_reps holds the states of every basis, the identity-index one included (dmv_basis_build enumerates them all)
  launch_zz_gram(run.n, run.ce, N, run.ctx->d_reps.ptr, xv, partials, d_gram, run.st);
  run.all_reduce(d_gram, size);
  CUDA_CHECK(cudaMemcpyAsync(padded.data(), d_gram, size * sizeof(double), cudaMemcpyDeviceToHost, run.st));
  CUDA_CHECK(cudaStreamSynchronize(run.st));
  const int CP = zz_gram_columns(N);
  for (int i = 0; i <= N; ++i)
    for (int j = 0; j < N; ++j) gram[(size_t)i * N + j] = padded[(size_t)i * CP + j];
  zz_symmetrize(N, G, gram.data(), C, m);
  return gram[0];
}

// Classes of the ordered site pairs under the group: (p, no flip) sends (i, j) to (p(i), p(j)), (p, flip) to
// (p(j), p(i)) (a global spin flip turns σ⁺σ⁻ into σ⁻σ⁺).  Numbered in the order of their first pair, row-major.
struct PmClasses {
  std::vector<int32_t> of;     // [N * N]: class of (i, j), -1 on the diagonal
  std::vector<int32_t> size;   // [count]: pairs in the class
};

PmClasses pm_classes(int N, const ZzGroup &G) {
  PmClasses K;
  K.of.assign((size_t)N * N, -1);
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      if (i == j || K.of[(size_t)i * N + j] >= 0) continue;
      const int32_t id = (int32_t)K.size.size();
      int32_t count = 0;
      for (int64_t e = 0; e < G.order; ++e) {
        const int32_t *p = G.perms.data() + e * N;
        const int k = G.flips[e] ? p[j] : p[i], l = G.flips[e] ? p[i] : p[j];
        if (K.of[(size_t)k * N + l] < 0) { K.of[(size_t)k * N + l] = id; ++count; }
      }
      K.size.push_back(count);
    }
  return K;
}

// pm[2 (i N + j) + {0, 1}] = <σ⁺ᵢσ⁻ⱼ> from the class sums (2 per class) for i != j, (1 + m_i) / 2 on the diagonal
void pm_finish(int N, const PmClasses &K, const double *sums, double W, const double *m, double *pm) {
  if (!(W > 0.0)) throw std::runtime_error("x is a zero vector: <x|x> = 0");
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      double *out = pm + 2 * ((size_t)i * N + j);
      if (i == j) { out[0] = 0.5 * (1.0 + m[i]); out[1] = 0.0; continue; }
      const int32_t c = K.of[(size_t)i * N + j];
      const double scale = 1.0 / (W * (double)K.size[c]);
      out[0] = sums[2 * c] * scale;
      out[1] = sums[2 * c + 1] * scale;
    }
}

// sums[2 c + {0, 1}] = class sum c of the vector A.x over this rank's rows (classes < count).  The lane-major walk runs
// once per group of classes whose slots fit in shared memory.  jw: the Jordan-Wigner walk of fermionic bases.
void pm_sums(SolverRun &run, PmArgs A, int count, int look, int tk, bool cplx, bool jw, double *sums) {
  const bool pairs = look <= LOOK_INVERSION;
  const int per_pass = pairs ? count : (int)(kPmSmem / ((size_t)kPmThreads * (cplx ? 16 : 8)));
  for (int c0 = 0; c0 < count; c0 += per_pass) {
    A.c_lo = c0;
    A.c_hi = std::min(count, c0 + per_pass);
    // k_pm_pairs: a tile of 32 rows per CTA and a slot per class; k_pm_rows: a row per thread and a slot per class and
    // thread
    const size_t smem = pairs ? (size_t)A.c_hi * 16 : (size_t)kPmThreads * (A.c_hi - A.c_lo) * (cplx ? 16 : 8);
    const int64_t work = pairs ? (A.n_rows + 31) / 32 : (A.n_rows + kPmThreads - 1) / kPmThreads;
    with_pm_kernel(look, tk, run.ce, cplx, jw, [&](auto kernel) {
      const int grid = one_wave(kernel, work, smem, kPmThreads);
      A.partials = run.partials((size_t)grid * (A.c_hi - A.c_lo) * 2);
      kernel<<<grid, kPmThreads, smem, run.st>>>(A);
      check_launch(pairs ? "k_pm_pairs" : "k_pm_rows");
      launch_reduce_partials(grid, A.c_hi - A.c_lo, A.partials, sums + 2 * c0, run.st);
    });
  }
}

// ---- host half of dmv_apply_spin: the checks and the per-site coefficients K.  With psi = B_s x in the source's irrep,
// the target projector P_t = 1 / |G_t| sum_g conj chi_t(g) U_g turns O = sum_j w_j o_j into
//     P_t O psi = sum_k K_k o'_k psi,   K_k = 1 / |G_t| sum_{g in G_t} chi_t(g) conj chi_s(g) w_{p_g^-1(k)},
// where o'_k = o_k for an element without a flip, and with a flip -σᶻ_k for σᶻ_k and σ∓_k for σ±_k (a global spin flip
// swaps raising and lowering).  The direction of p_g and the characters are pinned against the dense construction
// (tests/test_spin_operators.py).
struct SpinBasis {
  int n_sites, hamming_weight;
  ZzGroup G;
  std::vector<double> chars;   // [order] interleaved (re, im)
};

SpinBasis spin_basis(int n_sites, int hamming_weight, bool has_permutations, int64_t group_order, const int32_t *perms,
                     const uint8_t *flips, const double *characters, int spin_inversion) {
  SpinBasis B{n_sites, hamming_weight, zz_group(n_sites, has_permutations, group_order, perms, flips, spin_inversion), {}};
  if (has_permutations) {
    if (!characters) throw std::runtime_error("the basis has permutations but no characters");
    B.chars.assign(characters, characters + 2 * group_order);
  } else {
    B.chars = {1.0, 0.0};
    if (spin_inversion != 0) B.chars.insert(B.chars.end(), {(double)spin_inversion, 0.0});
  }
  return B;
}

SpinBasis spin_basis(const dmv_context *c) {
  return spin_basis(c->n_sites, c->hamming_weight, c->has_permutations, c->k_group_order, c->k_perms.data(),
                    c->k_flips.data(), c->k_chars.data(), c->spin_inversion);
}

struct SpinPlan {
  int walk = SPIN_SELF;
  std::vector<double> k;        // [2][N] complex: k_set, then k_clear
  double c0[2] = {0.0, 0.0};
  bool diag_sites = false;      // SPIN_SELF: the row factor sums k_set / k_clear over the sites (σᶻ)
};

const char *const kSpinKinds[4] = {"DMV_SPIN_ONE", "DMV_SPIN_Z", "DMV_SPIN_PLUS", "DMV_SPIN_MINUS"};

SpinPlan spin_plan(const SpinBasis &src, const SpinBasis &tgt, int elt, int kind, const double *w) {
  if (kind < DMV_SPIN_ONE || kind > DMV_SPIN_MINUS)
    throw std::runtime_error("kind must be DMV_SPIN_ONE, DMV_SPIN_Z, DMV_SPIN_PLUS or DMV_SPIN_MINUS (got " +
                             std::to_string(kind) + ")");
  if (!w) throw std::runtime_error("weights must not be null");
  if (elt != DMV_F64 && elt != DMV_C128) throw std::runtime_error("elt must be DMV_F64 or DMV_C128");
  const int N = src.n_sites;
  if (tgt.n_sites != N)
    throw std::runtime_error("the target has " + std::to_string(tgt.n_sites) + " sites and the source " +
                             std::to_string(N) + ": both bases need the same number of sites");
  const int delta = kind == DMV_SPIN_PLUS ? 1 : kind == DMV_SPIN_MINUS ? -1 : 0;
  const bool both_free = src.hamming_weight < 0 && tgt.hamming_weight < 0;
  if (!both_free && (src.hamming_weight < 0 || tgt.hamming_weight != src.hamming_weight + delta))
    throw std::runtime_error(std::string("Hamming weights: ") + kSpinKinds[kind] + " needs target = source" +
                             (delta > 0 ? " + 1" : delta < 0 ? " - 1" : "") + " or both free, got source " +
                             std::to_string(src.hamming_weight) + " and target " + std::to_string(tgt.hamming_weight));
  // the source element of every target element, compared as (permutation, flip)
  std::map<std::pair<std::vector<int32_t>, int>, int64_t> where;
  for (int64_t e = 0; e < src.G.order; ++e)
    where.emplace(std::make_pair(std::vector<int32_t>(src.G.perms.begin() + e * N, src.G.perms.begin() + (e + 1) * N),
                                 src.G.flips[e] ? 1 : 0), e);
  if (elt == DMV_F64) {
    bool real = true;
    for (int j = 0; j < N; ++j) real &= w[2 * j + 1] == 0.0;
    for (size_t e = 1; e < src.chars.size(); e += 2) real &= src.chars[e] == 0.0;
    for (size_t e = 1; e < tgt.chars.size(); e += 2) real &= tgt.chars[e] == 0.0;
    if (!real)
      throw std::runtime_error("DMV_F64 needs real weights and real characters in both bases: use DMV_C128");
  }
  SpinPlan S;
  S.k.assign(4 * (size_t)N, 0.0);
  double *k_set = S.k.data(), *k_clear = S.k.data() + 2 * N;
  bool any_flip = false;
  std::vector<int32_t> inv(N);
  for (int64_t e = 0; e < tgt.G.order; ++e) {
    const int32_t *p = tgt.G.perms.data() + e * N;
    const int f = tgt.G.flips[e] ? 1 : 0;
    const auto it = where.find(std::make_pair(std::vector<int32_t>(p, p + N), f));
    if (it == where.end()) {
      std::string perm;
      for (int i = 0; i < N && i < 12; ++i) perm += (i ? " " : "") + std::to_string(p[i]);
      throw std::runtime_error("the target group is not a subgroup of the source group: its element " +
                               std::to_string(e) + " (permutation " + perm + (N > 12 ? " ..." : "") + ", flip " +
                               std::to_string(f) + ") is not in the source group");
    }
    any_flip |= f != 0;
    const double ct_re = tgt.chars[2 * e], ct_im = tgt.chars[2 * e + 1];
    const double cs_re = src.chars[2 * it->second], cs_im = src.chars[2 * it->second + 1];
    double chi_re = ct_re * cs_re + ct_im * cs_im, chi_im = ct_im * cs_re - ct_re * cs_im;   // chi_t conj(chi_s)
    if (kind == DMV_SPIN_Z && f) { chi_re = -chi_re; chi_im = -chi_im; }
    for (int i = 0; i < N; ++i) inv[p[i]] = i;
    // σ⁺ terms walk the set bits of the row, σ⁻ terms its clear bits; a flip swaps them
    const bool to_set = kind == DMV_SPIN_Z || kind == DMV_SPIN_ONE || ((kind == DMV_SPIN_PLUS) != (f != 0));
    double *dst = to_set ? k_set : k_clear;
    for (int k = 0; k < N; ++k) {
      const double wr = w[2 * inv[k]], wi = w[2 * inv[k] + 1];
      dst[2 * k] += chi_re * wr - chi_im * wi;
      dst[2 * k + 1] += chi_re * wi + chi_im * wr;
    }
  }
  const double scale = 1.0 / (double)tgt.G.order;
  for (double &v : S.k) v *= scale;
  if (kind == DMV_SPIN_ONE) {   // a constant: sum_k K_k
    for (int k = 0; k < N; ++k) { S.c0[0] += k_set[2 * k]; S.c0[1] += k_set[2 * k + 1]; }
    std::fill(S.k.begin(), S.k.end(), 0.0);
  } else if (kind == DMV_SPIN_Z) {   // s_k = +1 on a set bit, -1 on a clear one
    for (int t = 0; t < 2 * N; ++t) k_clear[t] = -k_set[t];
    S.diag_sites = true;
  }
  S.walk = kind <= DMV_SPIN_Z ? SPIN_SELF
           : any_flip         ? SPIN_BOTH
           : kind == DMV_SPIN_PLUS ? SPIN_SET
                                   : SPIN_CLEAR;
  return S;
}

// ---- host half of dmv_apply_fermion: the particle numbers of the two bases.  Returns the modes the walk visits: every
// mode of a spinless basis; for a spinful one the spin half the non-zero weights lie in (number_up is fixed, so the
// other half's neighbours of a row are outside the source basis).  The weights themselves go through spin_plan.
uint64_t fermion_walk(const dmv_context *src, const dmv_context *tgt, int kind, const double *w) {
  if (kind != DMV_FERMION_CREATE && kind != DMV_FERMION_ANNIHILATE)
    throw std::runtime_error("kind must be DMV_FERMION_CREATE or DMV_FERMION_ANNIHILATE (got " + std::to_string(kind) +
                             ")");
  if (!w) throw std::runtime_error("weights must not be null");
  if (tgt->particle_type != src->particle_type)
    throw std::runtime_error(std::string("the target is a ") + particle_name(tgt->particle_type) +
                             " basis and the source a " + particle_name(src->particle_type) +
                             " basis: both need the same particle type");
  const int M = src->n_sites;
  if (tgt->n_sites != M)
    throw std::runtime_error("the target has " + std::to_string(tgt->n_sites) + " modes and the source " +
                             std::to_string(M) + ": both bases need the same number of modes");
  const int d = kind == DMV_FERMION_CREATE ? 1 : -1;
  const std::string op = kind == DMV_FERMION_CREATE ? "c†" : "c", sd = d > 0 ? " + 1" : " - 1";
  if (src->particle_type == DMV_SPINLESS_FERMION) {
    const int ns = src->number_particles, nt = tgt->number_particles;
    if (!((ns < 0 && nt < 0) || (ns >= 0 && nt == ns + d)))
      throw std::runtime_error("particle numbers: " + op + " needs target = source" + sd + " or both free, got source " +
                               std::to_string(ns) + " and target " + std::to_string(nt));
    return src->site_mask;
  }
  const int N = M / 2;
  const uint64_t up = (1ull << N) - 1;   // N <= 32
  bool w_up = false, w_down = false;
  for (int j = 0; j < M; ++j)
    if (w[2 * j] != 0.0 || w[2 * j + 1] != 0.0) (j < N ? w_up : w_down) = true;
  const int su = src->number_up, sdn = src->number_particles - su;
  const int tu = tgt->number_up, tdn = tgt->number_particles - tu;
  auto sector = [](int u, int dn) {
    return "(number_up " + std::to_string(u) + ", number_down " + std::to_string(dn) + ")";
  };
  if (w_up && w_down)
    throw std::runtime_error("the weights are non-zero in both spin halves: " + op + " would reach the sectors " +
                             sector(su + d, sdn) + " and " + sector(su, sdn + d) +
                             " at once; apply the up and the down modes separately");
  const bool to_up = tu == su + d && tdn == sdn, to_down = tu == su && tdn == sdn + d;
  if (w_up ? !to_up : w_down ? !to_down : !(to_up || to_down))
    throw std::runtime_error("particle numbers: " + op + " on the " +
                             (w_up ? "up modes needs the target " + sector(su + d, sdn)
                              : w_down ? "down modes needs the target " + sector(su, sdn + d)
                                       : "up or down modes needs the target " + sector(su + d, sdn) + " or " +
                                             sector(su, sdn + d)) +
                             " from the source " + sector(su, sdn) + ", got " + sector(tu, tdn));
  return w_up || (!w_down && to_up) ? up : up << N;
}

// ---- host half of dmv_reduced_density_matrix: the blocks of ρ_A and the checks of A
struct RdmLayout {
  int w_first = -1;           // weight of A of the first block; -1 at free weight (one block, every configuration)
  std::vector<int> dims;      // d_w of the blocks, in ascending w
  std::vector<int> ones_b;    // ones of B of the blocks (-1 at free weight)
  size_t entries = 0;         // sum of d_w^2
};

RdmLayout rdm_layout(int n_sites, int hamming_weight, int n_a) {
  if (n_sites < 1 || n_sites > 64) throw std::runtime_error("number_sites must be between 1 and 64");
  if (hamming_weight < -1 || hamming_weight > n_sites)
    throw std::runtime_error("hamming_weight must be -1 (free) or between 0 and " + std::to_string(n_sites) +
                             " (got " + std::to_string(hamming_weight) + ")");
  if (n_a < 1 || n_a > 16) throw std::runtime_error("n_a must be between 1 and 16 (got " + std::to_string(n_a) + ")");
  if (n_a > n_sites)
    throw std::runtime_error("n_a = " + std::to_string(n_a) + " exceeds the " + std::to_string(n_sites) + " sites");
  RdmLayout L;
  if (hamming_weight < 0) {
    L.dims = {1 << n_a};
    L.ones_b = {-1};
  } else {
    L.w_first = std::max(0, hamming_weight - (n_sites - n_a));
    for (int w = L.w_first; w <= std::min(n_a, hamming_weight); ++w) {
      L.dims.push_back((int)binom().c[n_a][w]);
      L.ones_b.push_back(hamming_weight - w);
    }
  }
  for (int d : L.dims) L.entries += (size_t)d * d;
  return L;
}

// A's sites as one-bit masks (bit k of a configuration of A is sites[k]); B's sites ascending
void rdm_sites(int n_sites, int n_a, const int32_t *sites, std::vector<uint64_t> &a, std::vector<uint64_t> &b) {
  if (!sites) throw std::runtime_error("sites_a must not be null");
  uint64_t seen = 0;
  for (int k = 0; k < n_a; ++k) {
    const int32_t s = sites[k];
    if (s < 0 || s >= n_sites)
      throw std::runtime_error("site " + std::to_string(s) + " of sites_a is outside [0, " + std::to_string(n_sites) + ")");
    if (seen >> s & 1ull) throw std::runtime_error("site " + std::to_string(s) + " appears twice in sites_a");
    seen |= 1ull << s;
    a.push_back(1ull << s);
  }
  for (int s = 0; s < n_sites; ++s)
    if (!(seen >> s & 1ull)) b.push_back(1ull << s);
}

// embed_A of the rows of the block of weight w (w < 0: every configuration), ascending in the local configuration
std::vector<uint64_t> rdm_rows(const std::vector<uint64_t> &a, int w) {
  std::vector<uint64_t> rows;
  const int n_a = (int)a.size();
  for (uint32_t l = 0; l < (1u << n_a); ++l) {
    if (w >= 0 && __builtin_popcount(l) != w) continue;
    uint64_t s = 0;
    for (int k = 0; k < n_a; ++k)
      if (l >> k & 1u) s |= a[k];
    rows.push_back(s);
  }
  return rows;
}

// The column chunks of a block: at most kRdmChunk amplitudes, the columns a multiple of 32 (a function of d_w and K
// alone, so neither the sums nor their order depend on free memory)
constexpr int64_t kRdmChunk = int64_t(1) << 24;
int64_t rdm_chunk_cols(int d, uint64_t K) {
  const int64_t by_size = std::max<int64_t>(32, kRdmChunk / d / 32 * 32);
  return std::min<int64_t>(by_size, (int64_t)((K + 31) / 32 * 32));
}

// The look-up of the observables in the basis of `ctx`: on several ranks in its whole-basis twin (the replicated-x form)
// against the gathered x.  The build follows the product's: k_rows' table where k_rows looks up with it, the square-torus
// orbit minimum where k_rows takes it.  whose ("" or "source's "): for the refusal on several ranks.
struct ObservableLookup {
  dmv_context *ctx, *basis;   // the context searched, and where its states are looked up (ctx or its twin)
  int elt, look, tk;
  cudaStream_t st;
  StateLookup dev{};          // everything but x

  ObservableLookup(dmv_context *c, int elt_, cudaStream_t st_, const char *entry, const char *whose = "")
      : ctx(c), basis(c), elt(elt_), st(st_) {
    const bool several = ctx->num_ranks > 1;
    if (several) {
      if (!ctx->exchange_decided) decide_exchange(ctx);   // collective: every rank reaches the same decision
      if (!ctx->replicated)
        throw std::runtime_error(std::string(entry) + " on several ranks needs the " + whose + "whole basis on every "
                                 "rank (the replicated-x form), and it is switched off by the exchange / mode options "
                                 "or does not fit in device memory");
      basis = ctx->global;
    }
    const bool trivial = ctx->proj != PROJ_GROUP || ctx->orbit.trivial_characters;
    look = ctx->proj == PROJ_NONE        ? LOOK_NONE
           : ctx->proj == PROJ_INVERSION ? LOOK_INVERSION
           : (use_rows(basis) && basis->opt.rows_index != 1) ? LOOK_TABLE
                                                             : LOOK_GROUP;
    tk = look >= LOOK_GROUP && trivial ? rows_torus_k(basis->orbit, basis->opt.rows_index == 1, basis->opt.rows_ctas)
                                       : 0;
    dev.index = base_params(basis).index;
    dev.orbit = basis->orbit;
    dev.norms = basis->d_norms.ptr;
    dev.pos = several ? ctx->d_pos.ptr : nullptr;
    dev.site_mask = ctx->site_mask;
    dev.inversion_character = (double)ctx->spin_inversion;
    dev.status = ctx->d_status.ptr;
    if (look == LOOK_TABLE) {   // k_rows' table over `basis`, its values refilled per vector (as every product does)
      ensure_table(basis, elt, st);
      dev.table = basis->d_table.ptr;
      dev.table_slots = basis->table_slots;
      dev.table_dir = basis->table_dir;
      dev.dord = basis->dord;
      dev.dense = basis->dense_order ? basis->d_dense.ptr : nullptr;
    }
  }

  // the look-up of xv, a vector of this rank's states: gathered from every rank on several, the table refilled from it
  StateLookup vector(const double *xv) const {
    StateLookup L = dev;
    L.x = ctx->num_ranks > 1 ? gather_x(ctx, elt, xv) : xv;
    if (look == LOOK_TABLE) fill_table(basis, elt, L.x, L.pos, st);
    return L;
  }
};

// The walk of dmv_pm_correlations (spin bases: <σ⁺ᵢσ⁻ⱼ>) and dmv_one_body_density_matrix (fermionic bases: <c†ᵢcⱼ>,
// with the Jordan-Wigner sign).  A spinful basis fixes number_up, so a pair with one mode in each spin half leaves the
// basis: such pairs are not walked, and their entries stay exactly 0.  entry / out_name: for the messages.
void pair_correlations(dmv_context *ctx, int elt, int num_vectors, const void *x, double *pm, const char *entry,
                       const char *out_name) {
  SolverRun run(ctx, elt, entry, false);
  if (num_vectors < 1) throw std::runtime_error("num_vectors must be positive");
  if (!x) throw std::runtime_error("x must not be null");
  if (!pm) throw std::runtime_error(std::string(out_name) + " must not be null");
  const int N = ctx->n_sites;
  const bool jw = ctx->particle_type != DMV_SPIN;
  const ZzGroup G = zz_group(N, ctx->has_permutations, ctx->k_group_order, ctx->k_perms.data(), ctx->k_flips.data(),
                             ctx->spin_inversion);
  const PmClasses K = pm_classes(N, G);
  const int count = (int)K.size.size();
  cudaStream_t st = run.st;
  const ObservableLookup lookup(ctx, elt, st, entry);
  const bool cplx = run.ce || (ctx->proj == PROJ_GROUP && !ctx->orbit.trivial_characters);
  std::vector<int16_t> class_of(K.of.begin(), K.of.end());
  std::vector<uint16_t> pairs;
  for (int i = 0; i < N; ++i)
    for (int j = i + 1; j < N; ++j)
      if (ctx->particle_type != DMV_SPINFUL_FERMION || (i < N / 2) == (j < N / 2)) pairs.push_back((uint16_t)(i | j << 8));
  DevBuf<int16_t> d_class_of;
  DevBuf<uint16_t> d_pairs;
  d_class_of.upload(class_of, st);
  d_pairs.upload(pairs, st);
  PmArgs A{};
  A.rows = ctx->d_reps.ptr;
  A.row_norms = ctx->d_norms.ptr;
  A.n_rows = run.n;
  A.x_row_offset = run.P > 1 ? (int64_t)ctx->rank * ctx->repl_block : 0;
  A.class_of = d_class_of.ptr;
  A.pairs = d_pairs.ptr;
  A.n_sites = N;
  A.n_pairs = (int)pairs.size();
  const size_t gram_size = zz_gram_size(N);
  double *d_gram = run.scalars(gram_size + 2 * (size_t)count), *d_sums = d_gram + gram_size;
  const InArg<double> xin(static_cast<const double *>(x), (size_t)num_vectors * run.words, st);
  std::vector<double> out((size_t)num_vectors * N * N * 2), C((size_t)N * N), m((size_t)N), sums(2 * (size_t)count);
  for (int v = 0; v < num_vectors; ++v) {
    const double *xv = xin.ptr + (size_t)v * run.words;
    const double W = zz_moments(run, G, xv, run.partials(zz_gram_partials(run.n, N)), d_gram, C.data(), m.data());
    A.look = lookup.vector(xv);
    pm_sums(run, A, count, lookup.look, lookup.tk, cplx, jw, d_sums);
    run.all_reduce(d_sums, 2 * (size_t)count);
    CUDA_CHECK(cudaMemcpyAsync(sums.data(), d_sums, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    check_status(ctx);   // synchronises
    pm_finish(N, K, sums.data(), W, m.data(), out.data() + (size_t)v * N * N * 2);
  }
  CUDA_CHECK(cudaMemcpyAsync(pm, out.data(), out.size() * sizeof(double), cudaMemcpyDefault, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
}

// The entry checks of dmv_apply_spin and dmv_apply_fermion: `require` (spin or fermionic bases) of both contexts, and a
// target on the source's device with the source's rank and number of ranks.  The run is the source's.
SolverRun one_site_run(dmv_context *target, dmv_context *source, int elt, const char *entry,
                       void (*require)(const dmv_context *, const char *)) {
  if (!target || !source) throw std::runtime_error("target and source must not be null");
  require(source, entry);
  require(target, entry);
  SolverRun run(source, elt, entry, false);
  require_states(target);
  if (target->device != source->device) throw std::runtime_error("target and source must be on the same device");
  if (target->rank != source->rank || target->num_ranks != source->num_ranks)
    throw std::runtime_error("target and source must have the same rank and number of ranks");
  return run;
}

// The launch half of dmv_apply_spin and dmv_apply_fermion: per vector one k_spin_rows pass over the target's rows of
// this rank, with Jordan-Wigner signs on fermionic bases.  walk_mask: the modes the set-bit / clear-bit walks visit.
void apply_one_site(SolverRun &run, dmv_context *target, const SpinPlan &S, uint64_t walk_mask, int num_vectors,
                    const void *x, void *y) {
  if (num_vectors < 1) throw std::runtime_error("num_vectors must be positive");
  if (!x) throw std::runtime_error("x must not be null");
  if (!y) throw std::runtime_error("y must not be null");
  dmv_context *source = run.ctx;
  cudaStream_t st = run.st;
  const ObservableLookup lookup(source, run.elt, st, run.name, "source's ");
  const bool jw = source->particle_type != DMV_SPIN;
  DevBuf<double> d_k;
  d_k.upload(S.k, st);
  SpinArgs A{};
  A.rows = target->d_reps.ptr;
  A.row_norms = target->proj == PROJ_GROUP ? target->d_norms.ptr : nullptr;
  A.row_norm = target->proj == PROJ_INVERSION ? std::sqrt(0.5) : 1.0;
  A.src_scale = source->proj == PROJ_INVERSION ? std::sqrt(0.5) : 1.0;
  A.k = d_k.ptr;
  A.c0 = make_double2(S.c0[0], S.c0[1]);
  A.walk_mask = walk_mask;
  A.diag_mask = S.diag_sites ? source->site_mask : 0;
  A.n_rows = target->n_states;
  A.n_sites = source->n_sites;
  const size_t out_words = (size_t)target->n_states * run.elt;
  const InArg<double> xin(static_cast<const double *>(x), (size_t)num_vectors * run.words, st);
  OutArg<double> yout(static_cast<double *>(y), (size_t)num_vectors * out_words);
  for (int v = 0; v < num_vectors; ++v) {
    A.src = lookup.vector(xin.ptr + (size_t)v * run.words);
    A.y = yout.ptr + (size_t)v * out_words;
    if (A.n_rows > 0)
      with_spin_kernel(lookup.look, lookup.tk, S.walk, run.ce, jw, [&](auto kernel) {
        const int grid = one_wave(kernel, (A.n_rows + kSpinThreads - 1) / kSpinThreads, 0, kSpinThreads);
        kernel<<<grid, kSpinThreads, 0, st>>>(A);
        check_launch("k_spin_rows");
      });
  }
  yout.finish(st);
  check_status(source);   // synchronises
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
  const size_t words = run.words;
  cudaStream_t st = run.st;
  double *partials = run.partials(zz_gram_partials(run.n, N)), *d_gram = run.scalars(zz_gram_size(N));
  const InArg<double> xin(static_cast<const double *>(x), (size_t)num_vectors * words, st);
  std::vector<double> C((size_t)num_vectors * N * N), m((size_t)num_vectors * N);
  for (int v = 0; v < num_vectors; ++v)
    zz_moments(run, G, xin.ptr + (size_t)v * words, partials, d_gram, C.data() + (size_t)v * N * N,
               m.data() + (size_t)v * N);
  CUDA_CHECK(cudaMemcpyAsync(correlations, C.data(), C.size() * sizeof(double), cudaMemcpyDefault, st));
  if (magnetization)
    CUDA_CHECK(cudaMemcpyAsync(magnetization, m.data(), m.size() * sizeof(double), cudaMemcpyDefault, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  API_END
}

// ---- flip-flop correlations (DESIGN.md section 3, "dmv_pm_correlations"): per vector one k_zz_gram pass (W and the
// magnetisation for the diagonal), one walk over this rank's rows and their antiparallel pairs (k_pm_rows with
// permutations, k_pm_pairs without) into one sum per class of site pairs, all-reduced over the ranks, finished on the
// host.  On several ranks the targets are looked up in the whole basis of the replicated-x form, against the gathered x.
int dmv_pm_correlations(dmv_context *ctx, int elt, int num_vectors, const void *x, double *pm) {
  API_BEGIN
  require_spin(ctx, "dmv_pm_correlations");
  pair_correlations(ctx, elt, num_vectors, x, pm, "dmv_pm_correlations", "pm");
  API_END
}

// ---- the one-body density matrix of a fermionic basis (DESIGN.md section 3, "dmv_one_body_density_matrix"): the walk
// of dmv_pm_correlations with a Jordan-Wigner sign on each term, over the pairs of modes that stay in the basis.
int dmv_one_body_density_matrix(dmv_context *ctx, int elt, int num_vectors, const void *x, double *out) {
  API_BEGIN
  require_fermion(ctx, "dmv_one_body_density_matrix");
  pair_correlations(ctx, elt, num_vectors, x, out, "dmv_one_body_density_matrix", "out");
  API_END
}

// ---- one-site operators between bases (DESIGN.md section 3, "dmv_apply_spin"): per vector one k_spin_rows pass over
// the target's rows of this rank, the source's states found as dmv_pm_correlations finds its targets.  On several ranks
// in the source's whole-basis twin against the gathered x.
int dmv_apply_spin(dmv_context *target, dmv_context *source, int elt, int kind, const double *weights, int num_vectors,
                   const void *x, void *y) {
  API_BEGIN
  SolverRun run = one_site_run(target, source, elt, "dmv_apply_spin", require_spin);
  const SpinPlan S = spin_plan(spin_basis(source), spin_basis(target), elt, kind, weights);
  apply_one_site(run, target, S, source->site_mask, num_vectors, x, y);
  API_END
}

// ---- c† and c between particle sectors (DESIGN.md section 3, "dmv_apply_fermion"): the walk of dmv_apply_spin with a
// Jordan-Wigner sign on each term, over the modes of the spin half the weights live in.
int dmv_apply_fermion(dmv_context *target, dmv_context *source, int elt, int kind, const double *weights,
                      int num_vectors, const void *x, void *y) {
  API_BEGIN
  SolverRun run = one_site_run(target, source, elt, "dmv_apply_fermion", require_fermion);
  const uint64_t walk_mask = fermion_walk(source, target, kind, weights);
  const SpinPlan S = spin_plan(spin_basis(source), spin_basis(target), elt,
                               kind == DMV_FERMION_CREATE ? DMV_SPIN_PLUS : DMV_SPIN_MINUS, weights);
  apply_one_site(run, target, S, walk_mask, num_vectors, x, y);
  API_END
}

// ---- reduced density matrices (DESIGN.md section 3, "dmv_reduced_density_matrix"): per vector and block w of ρ_A, the
// columns of B are cut into chunks (every P-th chunk on each rank); per chunk one k_rdm_fill pass writes its amplitudes
// through the observables' look-up, k_rdm_gram adds Ψ Ψᴴ per slice of columns and k_rdm_reduce adds the slices,
// in order, to the block.  The blocks are all-reduced over the ranks, mirrored and divided by <x|x>.
int dmv_reduced_density_matrix(dmv_context *ctx, int elt, int num_vectors, const void *x, int n_a,
                               const int32_t *sites_a, double *rho) {
  API_BEGIN
  require_spin(ctx, "dmv_reduced_density_matrix");
  SolverRun run(ctx, elt, "dmv_reduced_density_matrix", true);
  if (num_vectors < 1) throw std::runtime_error("num_vectors must be positive");
  if (!x) throw std::runtime_error("x must not be null");
  if (!rho) throw std::runtime_error("rho must not be null");
  const int N = ctx->n_sites, P = run.P;
  const RdmLayout L = rdm_layout(N, ctx->hamming_weight, n_a);
  std::vector<uint64_t> site_a, site_b;
  rdm_sites(N, n_a, sites_a, site_a, site_b);
  const int n_b = (int)site_b.size();
  const size_t cw = run.ce ? 2 : 1;
  // every size follows from the layout alone: the blocks, the largest chunk, its slices' partials, a host staging copy
  std::vector<uint64_t> cols_total(L.dims.size());
  size_t psi_words = 0, part_words = 0;
  int max_d = 0;
  for (size_t i = 0; i < L.dims.size(); ++i) {
    const int d = L.dims[i];
    cols_total[i] = L.ones_b[i] < 0 ? 1ull << n_b : binom().c[n_b][L.ones_b[i]];
    const int64_t ld = rdm_chunk_cols(d, cols_total[i]);
    psi_words = std::max(psi_words, (size_t)d * ld * cw);
    part_words = std::max(part_words, (size_t)rdm_slices(d, ld) * rdm_tiles(d) * kRdmTile * kRdmTile * cw);
    max_d = std::max(max_d, d);
  }
  const size_t acc_words = 2 * L.entries;
  const bool host_out = !is_device_pointer(rho);
  {
    size_t free_b = 0, total_b = 0;
    CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    const double need = 8.0 * ((double)acc_words * (host_out ? 1.0 + num_vectors : 1.0) + (double)psi_words +
                               (double)part_words);
    if (need > (double)free_b)
      throw std::runtime_error("dmv_reduced_density_matrix: ρ of " + std::to_string(n_a) + " sites (" +
                               std::to_string(L.entries) + " entries per vector) with its work space needs " +
                               std::to_string((uint64_t)need) + " bytes, but only " + std::to_string(free_b) +
                               " bytes are free on the device");
  }
  cudaStream_t st = run.st;
  const ObservableLookup lookup(ctx, elt, st, "dmv_reduced_density_matrix");
  // <x|x> of every vector first: a zero vector is refused before anything is written
  const InArg<double> xin(static_cast<const double *>(x), (size_t)num_vectors * run.words, st);
  double *d_norm2 = run.scalars(2 * (size_t)num_vectors), *q_part = run.partials(quad_partials(1));
  for (int v = 0; v < num_vectors; ++v)
    launch_quad_dot(run.n, run.ce, 1, xin.ptr + (size_t)v * run.words, xin.ptr + (size_t)v * run.words, q_part,
                    d_norm2 + 2 * v, st);
  run.all_reduce(d_norm2, 2 * (size_t)num_vectors);
  std::vector<double> norm2(2 * (size_t)num_vectors);
  CUDA_CHECK(cudaMemcpyAsync(norm2.data(), d_norm2, norm2.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  for (int v = 0; v < num_vectors; ++v)
    if (!(norm2[2 * v] > 0.0))
      throw std::runtime_error("x is a zero vector: <x|x> = 0 (vector " + std::to_string(v) + ")");

  RdmArgs A{};
  A.scale = ctx->proj == PROJ_INVERSION ? std::sqrt(0.5) : 1.0;
  A.n_b = n_b;
  std::copy(site_b.begin(), site_b.end(), A.sites_b);
  std::vector<uint64_t> h_binom(64 * 65);
  for (int n = 0; n < 64; ++n)
    for (int k = 0; k <= 64; ++k) h_binom[n * 65 + k] = binom().c[n][k];
  DevBuf<uint64_t> d_binom, d_rows;
  DevBuf<double> d_acc, d_psi, d_part;
  d_binom.upload(h_binom, st);
  d_rows.alloc(max_d);
  d_acc.alloc(acc_words);
  d_psi.alloc(psi_words);
  d_part.alloc(part_words);
  A.binom = d_binom.ptr;
  A.embed_a = d_rows.ptr;
  A.psi = d_psi.ptr;
  OutArg<double> out(rho, (size_t)num_vectors * acc_words);
  int64_t amplitudes = 0, flops = 0;
  for (int v = 0; v < num_vectors; ++v) {
    A.src = lookup.vector(xin.ptr + (size_t)v * run.words);
    CUDA_CHECK(cudaMemsetAsync(d_acc.ptr, 0, acc_words * sizeof(double), st));
    size_t off = 0;
    for (size_t bi = 0; bi < L.dims.size(); ++bi) {
      const int d = L.dims[bi];
      const uint64_t K = cols_total[bi];
      const int64_t ld = rdm_chunk_cols(d, K), tiles = rdm_tiles(d), slice_cols = rdm_slice_cols(d, ld);
      const int slices = rdm_slices(d, ld);
      const std::vector<uint64_t> rows = rdm_rows(site_a, L.ones_b[bi] < 0 ? -1 : L.w_first + (int)bi);
      CUDA_CHECK(cudaMemcpyAsync(d_rows.ptr, rows.data(), rows.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
      A.d = d;
      A.k_b = L.ones_b[bi];
      A.ld = ld;
      const uint64_t n_chunks = (K + ld - 1) / ld;
      for (uint64_t c = P > 1 ? (uint64_t)ctx->rank : 0; c < n_chunks; c += P) {   // every P-th chunk
        A.col0 = (int64_t)(c * ld);
        A.cols = (int64_t)std::min<uint64_t>(ld, K - c * ld);
        with_rdm_fill(lookup.look, lookup.tk, run.ce, [&](auto kernel) {
          const int64_t work = (d + kRdmRowGroup - 1) / kRdmRowGroup * ld;
          kernel<<<one_wave(kernel, (work + kRdmThreads - 1) / kRdmThreads, 0, kRdmThreads), kRdmThreads, 0, st>>>(A);
          check_launch("k_rdm_fill");
        });
        with_bool(run.ce, [&](auto ce) {
          k_rdm_gram<ce()><<<dim3((unsigned)tiles, (unsigned)slices), 256, 0, st>>>(d_psi.ptr, ld, d, ld, slice_cols,
                                                                                   d_part.ptr);
          check_launch("k_rdm_gram");
          const int grid = one_wave(k_rdm_reduce<ce()>, (tiles * kRdmTile * kRdmTile + 255) / 256, 0, 256);
          k_rdm_reduce<ce()><<<grid, 256, 0, st>>>(d_part.ptr, slices, tiles, d, d_acc.ptr + off);
          check_launch("k_rdm_reduce");
        });
        amplitudes += (int64_t)d * A.cols;
        flops += tiles * kRdmTile * kRdmTile * ld * (run.ce ? 4 : 1);
      }
      off += 2 * (size_t)d * d;
    }
    run.all_reduce(d_acc.ptr, acc_words);
    off = 0;
    for (const int d : L.dims) {
      const int grid = one_wave(k_rdm_finish, ((int64_t)d * d + 255) / 256, 0, 256);
      k_rdm_finish<<<grid, 256, 0, st>>>(d_acc.ptr + off, d, 1.0 / norm2[2 * v], out.ptr + (size_t)v * acc_words + off);
      check_launch("k_rdm_finish");
      off += 2 * (size_t)d * d;
    }
  }
  out.finish(st);
  check_status(ctx);   // synchronises
  ctx->rdm_amplitudes = amplitudes;
  ctx->rdm_gram_flops = flops;
  API_END
}

// host-only layout of dmv_reduced_density_matrix (no device needed)
int dmv_rdm_layout(int n_sites, int hamming_weight, int n_a, const int32_t *sites_a, int *num_blocks, int *w_first,
                   int32_t *dims) {
  API_BEGIN
  if (!num_blocks) throw std::runtime_error("num_blocks must not be null");
  const RdmLayout L = rdm_layout(n_sites, hamming_weight, n_a);
  if (sites_a) {
    std::vector<uint64_t> a, b;
    rdm_sites(n_sites, n_a, sites_a, a, b);
  }
  *num_blocks = (int)L.dims.size();
  if (w_first) *w_first = L.w_first;
  if (dims) std::copy(L.dims.begin(), L.dims.end(), dims);
  API_END
}

// host-only self-check entry for the host half of dmv_apply_spin (no device needed)
int dmv_debug_spin_weights(const dmv_basis_desc *source, const dmv_basis_desc *target, int elt, int kind,
                           const double *weights, double *k, double *c0, int *walk) {
  API_BEGIN
  if (!source || !target) throw std::runtime_error("source and target must not be null");
  for (const dmv_basis_desc *b : {source, target})
    if (b->number_sites < 1 || b->number_sites > 64) throw std::runtime_error("number_sites must be between 1 and 64");
  auto basis = [](const dmv_basis_desc *b) {
    return spin_basis(b->number_sites, b->hamming_weight, b->has_permutations != 0, b->group_order, b->perms, b->flips,
                      b->characters, b->spin_inversion);
  };
  const SpinPlan S = spin_plan(basis(source), basis(target), elt, kind, weights);
  if (k) std::copy(S.k.begin(), S.k.end(), k);
  if (c0) { c0[0] = S.c0[0]; c0[1] = S.c0[1]; }
  if (walk) *walk = S.walk;
  API_END
}

// host-only self-check entry for the host half of dmv_pm_correlations (no device needed)
int dmv_debug_pm_classes(const dmv_basis_desc *basis, int32_t *class_of, int32_t *class_size, int32_t *num_classes,
                         const double *sums, double W, const double *magnetization, double *pm) {
  API_BEGIN
  if (!basis || !class_of || !class_size || !num_classes)
    throw std::runtime_error("basis, class_of, class_size and num_classes must not be null");
  const int N = basis->number_sites;
  if (N < 1 || N > 64) throw std::runtime_error("number_sites must be between 1 and 64");
  const ZzGroup G = zz_group(N, basis->has_permutations != 0, basis->group_order, basis->perms, basis->flips,
                             basis->spin_inversion);
  const PmClasses K = pm_classes(N, G);
  std::copy(K.of.begin(), K.of.end(), class_of);
  std::copy(K.size.begin(), K.size.end(), class_size);
  *num_classes = (int32_t)K.size.size();
  if (sums) {
    if (!magnetization || !pm) throw std::runtime_error("the finish needs magnetization and pm");
    pm_finish(N, K, sums, W, magnetization, pm);
  }
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
