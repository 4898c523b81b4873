// dmv_gather.cu -- k_gather: the single-rank product traversed by ROWS, specialised for operators whose
// flip-mask groups all pass the bit-parallel emit test (every two-body spin Hamiltonian) on bases without
// permutation symmetries (BatchedOperator branches a and b, reference src/BatchedOperator.chpl:89-161).
//
//   y[b] = D(b) x[b] + sum_{g emits on row b} c_g(b) x[index(b ^ x_g)]
//
// The same arithmetic as localDiagonal + computeOffDiag + localProcess (reference
// src/DistributedMatrixVector.chpl:36-127), but every y element is produced by ONE lane and stored once:
// no (beta, c) records, no shared-memory queue, no FP64 atomics (the L2 atomic unit is the busiest unit of
// the scatter form), and the result is bit-reproducible.
// One lane owns one row: 8/16-byte coalesced loads of sigma_b and x_b, the emit mask of all groups from a few
// masked shifts (BpWord), then a walk over the set bits two at a time -- two index look-ups and two x gathers
// in flight per lane.  With <= 32 sites and <= 32 groups the whole row runs in 32-bit registers (NARROW).
// Only used when one rank owns the basis (the distributed product needs the scatter form: the owner of a
// row does not hold the x of its neighbours).
#include <cuda_runtime.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "dmv_host.h"

namespace dmv {

namespace {

constexpr int kThreads = 256;

template <bool C> struct Val { using type = double; };
template <> struct Val<true> { using type = double2; };

__device__ __forceinline__ int popc_w(uint32_t v) { return __popc(v); }
__device__ __forceinline__ int popc_w(uint64_t v) { return __popcll(v); }
__device__ __forceinline__ int ffs_w(uint32_t v) { return __ffs((int)v); }
__device__ __forceinline__ int ffs_w(uint64_t v) { return __ffsll((long long)v); }
__device__ __forceinline__ int top_w(uint32_t v) { return 31 - __clz((int)v); }
__device__ __forceinline__ int top_w(uint64_t v) { return 63 - __clzll((long long)v); }

// acc += c * s * x for the four (coefficient, element) type combinations
__device__ __forceinline__ void fma_to(double &acc, double c, double x) { acc = fma(c, x, acc); }
__device__ __forceinline__ void fma_to(double2 &acc, double c, double2 x) {
  acc.x = fma(c, x.x, acc.x); acc.y = fma(c, x.y, acc.y);
}
__device__ __forceinline__ void fma_to(double2 &acc, double2 c, double2 x) {
  acc.x = fma(c.x, x.x, fma(-c.y, x.y, acc.x));
  acc.y = fma(c.x, x.y, fma(c.y, x.x, acc.y));
}
__device__ __forceinline__ void fma_to(double2 &acc, double2 c, double x) {
  acc.x = fma(c.x, x, acc.x); acc.y = fma(c.y, x, acc.y);
}
__device__ __forceinline__ double scale(double c, double s) { return c * s; }
__device__ __forceinline__ double2 scale(double2 c, double s) { return make_double2(c.x * s, c.y * s); }
__device__ __forceinline__ bool nonzero(double c) { return c != 0.0; }
__device__ __forceinline__ bool nonzero(double2 c) { return c.x != 0.0 || c.y != 0.0; }
__device__ __forceinline__ double ldx(const double *x, uint32_t i) { return __ldg(x + i); }
__device__ __forceinline__ double2 ldx(const double2 *x, uint32_t i) { return __ldg(x + i); }
__device__ __forceinline__ double make_v(double re, double, double *) { return re; }
__device__ __forceinline__ double2 make_v(double re, double im, double2 *) { return make_double2(re, im); }
__device__ __forceinline__ double zero_of(double *) { return 0.0; }
__device__ __forceinline__ double2 zero_of(double2 *) { return make_double2(0.0, 0.0); }
__device__ __forceinline__ double shfl_xor_v(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ double2 shfl_xor_v(double2 v, int m) {
  return make_double2(__shfl_xor_sync(0xffffffffu, v.x, m), __shfl_xor_sync(0xffffffffu, v.y, m));
}
__device__ __forceinline__ void add_to(double &a, double b) { a += b; }
__device__ __forceinline__ void add_to(double2 &a, double2 b) { a.x += b.x; a.y += b.y; }

struct GatherLayout { size_t bp, dclass, diag, lut, gx, total; };
__host__ __device__ inline GatherLayout gather_layout(const KernelParams &p, size_t word_bytes, size_t val_bytes,
                                                      bool uniform) {
  GatherLayout L;
  size_t off = 0;
  L.bp = off; off += sizeof(BpWord) * (size_t)p.n_bp;
  L.dclass = off; off += sizeof(DiagClass) * (size_t)p.n_diag_classes;
  L.diag = off; off += sizeof(DiagTerm) * (size_t)p.n_diag_rest;
  off = (off + 15) / 16 * 16;
  L.lut = off; off += uniform ? 0 : val_bytes * (size_t)p.n_lut;
  L.gx = off; off += word_bytes * (size_t)p.n_groups;
  L.total = (off + 15) / 16 * 16;
  return L;
}

// masked-shift gather of one support bit of every group (see BpWord)
template <typename W>
__device__ __forceinline__ W bp_gather(const BpPair *pairs, int n, W a) {
  W out = 0;
#pragma unroll 1
  for (int k = 0; k < n; ++k) {
    const BpPair q = pairs[k];
    out |= (W)((a << q.l) >> q.r) & (W)q.m;
  }
  return out;
}

// state -> index for a full fixed-Hamming-weight block: Lin tables (see StateIndex).  kNone = not a basis state.
// Blocks hold fewer than 2^32 states (dmv_set_representatives / dmv_basis_build enforce it).
constexpr uint32_t kNone = 0xffffffffu;
template <typename W>
__device__ __forceinline__ uint32_t lin_index(const uint32_t *__restrict__ lin_a, const uint32_t *__restrict__ lin_b,
                                              int lin_bits, W lo_mask, int weight, uint32_t n, W key) {
  // key = (row state) ^ (flip mask): always inside the site mask, only the weight can be wrong
  if (popc_w(key) != weight) return kNone;
  const uint32_t r = __ldg(lin_a + (uint32_t)(key >> lin_bits)) + __ldg(lin_b + (uint32_t)(key & lo_mask));
  return r < n ? r : kNone;   // with spin inversion only the first half are representatives
}

template <bool INV, bool CV, bool CE, bool NARROW, bool LIN, bool UNI, int KB>
__global__ void __launch_bounds__(kThreads) k_gather(const KernelParams p) {
  using V = typename Val<CV>::type;            // coefficient type
  using E = typename Val<CE>::type;            // vector element type
  using A = typename Val<CV || CE>::type;      // row accumulator
  using W = typename std::conditional<NARROW, uint32_t, uint64_t>::type;
  extern __shared__ __align__(16) unsigned char smem[];
  const GatherLayout L = gather_layout(p, sizeof(W), sizeof(V), UNI);
  BpWord *s_bp = reinterpret_cast<BpWord *>(smem + L.bp);
  DiagClass *s_dclass = reinterpret_cast<DiagClass *>(smem + L.dclass);
  DiagTerm *s_diag = reinterpret_cast<DiagTerm *>(smem + L.diag);
  V *s_lut = reinterpret_cast<V *>(smem + L.lut);
  W *s_gx = reinterpret_cast<W *>(smem + L.gx);
  {
    const uint64_t *src = reinterpret_cast<const uint64_t *>(p.bp);
    uint64_t *dst = reinterpret_cast<uint64_t *>(s_bp);
    for (int i = threadIdx.x; i < p.n_bp * (int)(sizeof(BpWord) / 8); i += blockDim.x) dst[i] = src[i];
    src = reinterpret_cast<const uint64_t *>(p.diag_classes);
    dst = reinterpret_cast<uint64_t *>(s_dclass);
    for (int i = threadIdx.x; i < p.n_diag_classes * (int)(sizeof(DiagClass) / 8); i += blockDim.x) dst[i] = src[i];
    for (int i = threadIdx.x; i < p.n_diag_rest; i += blockDim.x) s_diag[i] = p.diag[i];
    if (!UNI)
      for (int i = threadIdx.x; i < p.n_lut; i += blockDim.x) s_lut[i] = reinterpret_cast<const V *>(p.lut)[i];
    for (int i = threadIdx.x; i < p.n_groups; i += blockDim.x) s_gx[i] = (W)p.groups[i].x;
  }
  __syncthreads();

  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  const int warps_per_cta = kThreads / 32;
  const W site = (W)p.site_mask;
  const E *xv = reinterpret_cast<const E *>(p.x);
  const V uni = make_v(p.uni_re, p.uni_im, (V *)nullptr);
  const uint32_t *__restrict__ lin_a = p.index.lin_a, *__restrict__ lin_b = p.index.lin_b;
  const int lin_bits = p.index.lin_bits, weight = p.index.weight;
  const W lo_mask = (W)((1ull << lin_bits) - 1);
  const uint32_t n_states = (uint32_t)p.index.n;
  const uint64_t *__restrict__ row_states = p.row_states ? p.row_states : p.index.reps;
  const uint32_t *__restrict__ pos = p.pos;   // replicated-x product: global index -> slot of the gathered x

  // row_split = S lanes share one row (each walks every S-th group), combined with S-1 shuffles: small bases
  const int S = p.row_split > 1 ? p.row_split : 1;
  const int rows_per_tile = 32 / S;
  const unsigned slice = lane & (unsigned)(S - 1);
  W slice_mask = ~(W)0;
  if (S > 1) {
    slice_mask = 0;
    for (int g = (int)slice; g < (int)(8 * sizeof(W)); g += S) slice_mask |= (W)1 << g;
  }
  const int64_t n_rows = p.row_end - p.row_begin;
  const int64_t n_tiles = (n_rows + rows_per_tile - 1) / rows_per_tile;
  const int64_t warps_total = (int64_t)gridDim.x * warps_per_cta;
  unsigned long long bad = 0, bad_state = 0;

  for (int64_t tile = (int64_t)blockIdx.x * warps_per_cta + warp; tile < n_tiles; tile += warps_total) {
    const int64_t i = p.row_begin + tile * rows_per_tile + lane / S;
    const bool valid = i < p.row_end;
    const W b = valid ? (W)__ldg(row_states + i) : (W)0;
    // KB vectors at once (x, y: KB arrays of p.batch_stride elements apart): one walk over the terms and one index
    // look-up per term serve all of them
    A acc[KB];
#pragma unroll
    for (int k = 0; k < KB; ++k) acc[k] = zero_of((A *)nullptr);

    for (int w = 0; w < p.n_bp; ++w) {
      const BpWord &Wd = s_bp[w];
      const W a0 = bp_gather<W>(Wd.p0, Wd.n0, b), a1 = bp_gather<W>(Wd.p1, Wd.n1, b);
      W mask = (~a0 & ~a1 & (W)Wd.tt[0]) | (a0 & ~a1 & (W)Wd.tt[1]) | (~a0 & a1 & (W)Wd.tt[2]) |
               (a0 & a1 & (W)Wd.tt[3]);
      mask &= slice_mask;
      if (!valid) mask = 0;
      const int g_base = 64 * w;
      // NB terms per trip (groups g[j] of this word; on[j]: this lane emits them): all index look-ups, then all
      // gathers, are in flight together
      auto batch = [&](auto nb, const int *g, const bool *on) {
        constexpr int NB = decltype(nb)::value;
        W key[NB];
        double sg[NB];
        uint32_t idx[NB];
        V c[NB];
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          key[j] = b ^ s_gx[g_base + g[j]];
          sg[j] = 1.0;
          if (INV) {   // reference src/BatchedOperator.chpl:145-152
            const W f = key[j] ^ site;
            if (f < key[j]) { key[j] = f; sg[j] = p.inversion_character; }
          }
        }
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          idx[j] = kNone;
          if (on[j]) {
            if (LIN) idx[j] = lin_index<W>(lin_a, lin_b, lin_bits, lo_mask, weight, n_states, key[j]);
            else idx[j] = (uint32_t)locate(p.index, (uint64_t)key[j]);   // -1 -> kNone
          }
        }
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          if (UNI) c[j] = uni;
          else c[j] = s_lut[4 * (g_base + g[j]) + ((unsigned)((a0 >> g[j]) & 1) | ((unsigned)((a1 >> g[j]) & 1) << 1))];
          if (pos && idx[j] != kNone) idx[j] = __ldg(pos + idx[j]);
        }
        E xs[NB][KB];
#pragma unroll
        for (int j = 0; j < NB; ++j)
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            xs[j][k] = zero_of((E *)nullptr);
            if (idx[j] != kNone) xs[j][k] = ldx(xv + (int64_t)k * p.batch_stride, idx[j]);
          }
        bool miss = false;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          if (INV) c[j] = scale(c[j], sg[j]);
#pragma unroll
          for (int k = 0; k < KB; ++k)
            if (on[j]) fma_to(acc[k], c[j], xs[j][k]);
          miss |= on[j] & (idx[j] == kNone);
        }
        if (miss) {   // DMV:115-118 (rare)
#pragma unroll
          for (int j = 0; j < NB; ++j)
            if (on[j] && idx[j] == kNone && nonzero(c[j])) { ++bad; bad_state = (unsigned long long)key[j]; }
        }
      };
      if (S == 1 && p.gather_walk == 1) {
        // GROUP-MAJOR walk (option "gather_walk" = 1), warp-uniform, four groups per trip: all 32 lanes handle the same
        // group at the same time.  For a fixed flip mask consecutive rows map to (nearly) consecutive indices, so the 32
        // gathers of a group fall into a few 128-byte lines instead of 32.  But every
        // lane now walks all emitting groups of the warp (24 instead of its own ~12.5 on chain_24): 35 % more
        // instructions, which cost more than the fewer L1 wavefronts save.  Kept for reference; the per-lane walk below is the default.
        W any;
        if constexpr (sizeof(W) == 4) any = __reduce_or_sync(0xffffffffu, mask);
        else {
          const uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)mask);
          const uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)((uint64_t)mask >> 32));
          any = (W)(((uint64_t)hi << 32) | lo);
        }
        while (any) {
          int g[4];
          bool on[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const bool more = any != 0;
            g[j] = more ? ffs_w(any) - 1 : g[0];
            any &= any - 1;   // no-op when already empty
            on[j] = more && ((mask >> g[j]) & 1);
          }
          batch(std::integral_constant<int, 4>{}, g, on);
        }
      } else {
        // every lane walks its own bits (S > 1: its own slice of the groups), two per trip -- from the TOP: the 32
        // consecutive rows of a warp share their high bits, hence the emit bits of the groups acting there, so the lanes
        // walk those groups in step and their gathers fall into the same few lines; only the groups touching the low,
        // varying bits come out of step, and those move the index by little ("gather_walk" = 2: from the bottom, round 1)
        const bool from_top = p.gather_walk != 2;
        while (mask) {
          int g[2];
          bool on[2];
          g[0] = from_top ? top_w(mask) : ffs_w(mask) - 1;
          mask &= ~((W)1 << g[0]);
          on[0] = true;
          on[1] = mask != 0;
          g[1] = on[1] ? (from_top ? top_w(mask) : ffs_w(mask) - 1) : g[0];
          if (on[1]) mask &= ~((W)1 << g[1]);
          batch(std::integral_constant<int, 2>{}, g, on);
        }
      }
    }
    if (S > 1)
      for (int m = 1; m < S; m <<= 1) {
#pragma unroll
        for (int k = 0; k < KB; ++k) add_to(acc[k], shfl_xor_v(acc[k], m));
      }

    if (valid && slice == 0) {
      // diagonal (DMV:36-53) and the single store of y[i]; without diagonal terms y is accumulated into.  A class
      // holds up to 64 zz terms whatever the row width (NARROW counts sites and flip-mask groups, not zz terms): one of
      // more than 32 terms is evaluated in 64 bits, else terms 32-63 would drop out of the mask and count as parallel
      double dre = 0.0, dim = 0.0;
      if (p.n_diag > 0) {
        for (int c = 0; c < p.n_diag_classes; ++c) {
          const DiagClass &D = s_dclass[c];
          int anti;
          if (sizeof(W) == 8 || (D.mask >> 32) == 0) {
            const W d0 = bp_gather<W>(D.p0, D.n0, b), d1 = bp_gather<W>(D.p1, D.n1, b);
            anti = popc_w((W)((d0 ^ d1) & (W)D.mask));
          } else {
            const uint64_t d0 = bp_gather<uint64_t>(D.p0, D.n0, (uint64_t)b);
            const uint64_t d1 = bp_gather<uint64_t>(D.p1, D.n1, (uint64_t)b);
            anti = __popcll((d0 ^ d1) & D.mask);
          }
          const double wgt = (double)(D.count - 2 * anti);
          dre += wgt * D.v_re;
          dim += wgt * D.v_im;
        }
        for (int t = 0; t < p.n_diag_rest; ++t) {
          const DiagTerm d = s_diag[t];
          if (((uint64_t)b & d.m) == d.r) {
            const double sg = (__popcll((uint64_t)b & d.s) & 1) ? -1.0 : 1.0;
            dre += sg * d.v_re;
            dim += sg * d.v_im;
          }
        }
      }
#pragma unroll
      for (int k = 0; k < KB; ++k) {
        E *yk = reinterpret_cast<E *>(p.y) + (int64_t)k * p.batch_stride;
        E out;
        if (p.n_diag > 0) {
          const E xi = ldx(xv + (int64_t)k * p.batch_stride, (uint32_t)(p.x_row_offset + i));
          if constexpr (CE) out = make_double2(dre * xi.x - dim * xi.y, dre * xi.y + dim * xi.x);
          else out = dre * xi;   // real vectors take the real part of the diagonal
        } else {
          out = yk[i];
        }
        if constexpr (CE) { out.x += acc[k].x; out.y += acc[k].y; }
        else if constexpr (CV) out += acc[k].x;
        else out += acc[k];
        yk[i] = out;
      }
    }
  }
  if (bad) {
    if (atomicAdd(p.status, bad) == 0) p.status[1] = bad_state;
  }
}

// one thread per chunk of consecutive global states (set-up only)
template <bool WRITE>
__global__ void k_owner_positions(const uint64_t *__restrict__ states, const uint8_t *__restrict__ masks, int64_t n,
                                  int num_ranks, int64_t chunk, unsigned long long *chunk_counts,
                                  const unsigned long long *__restrict__ chunk_base, int64_t block, uint32_t *pos) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t first = c * chunk;
  if (first >= n) return;
  const int64_t last = min(n, first + chunk);
  uint32_t cnt[32];
#pragma unroll
  for (int r = 0; r < 32; ++r) cnt[r] = 0;
  for (int64_t g = first; g < last; ++g) {
    const int r = masks ? (int)masks[g] : locale_idx_of(states[g], num_ranks);
    uint32_t k = 0;
#pragma unroll
    for (int q = 0; q < 32; ++q)   // register-resident counters: no dynamic indexing
      if (q == r) { k = cnt[q]; cnt[q] = k + 1; }
    if (WRITE) pos[g] = (uint32_t)((int64_t)r * block + (int64_t)chunk_base[c * num_ranks + r] + k);
  }
  if (!WRITE)
    for (int r = 0; r < num_ranks; ++r) {
      uint32_t k = 0;
#pragma unroll
      for (int q = 0; q < 32; ++q) if (q == r) k = cnt[q];
      chunk_counts[c * num_ranks + r] = k;
    }
}

// out[pos[i]] = in[i] (scatter) or out[i] = in[pos[i]] (gather) for 8- or 16-byte elements
template <typename T, bool GATHER>
__global__ void k_permute(int64_t n, const uint32_t *__restrict__ pos, const T *__restrict__ in, T *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (GATHER) out[i] = in[pos[i]];
    else out[pos[i]] = in[i];
  }
}

}  // namespace

void launch_permute(int64_t n, int elt, const uint32_t *pos, const void *in, void *out, bool gather, cudaStream_t stream) {
  if (n <= 0) return;
  const int blocks = capped_grid((n + 255) / 256, (int64_t)sm_count() * 16);
  with_bool(elt != 1, [&](auto wide) {
    using T = std::conditional_t<wide(), double2, double>;
    with_bool(gather, [&](auto g) {
      k_permute<T, g()><<<blocks, 256, 0, stream>>>(n, pos, (const T *)in, (T *)out);
    });
  });
  check_launch("k_permute");
}

void launch_owner_positions(const uint64_t *states, const uint8_t *masks, int64_t n, int num_ranks, int64_t chunk,
                            bool write_pass, unsigned long long *chunk_counts, const unsigned long long *chunk_base,
                            int64_t block, uint32_t *pos, cudaStream_t stream) {
  if (n <= 0) return;
  if (num_ranks > 32) throw std::runtime_error("replicated-x product supports at most 32 ranks");
  const int64_t n_chunks = (n + chunk - 1) / chunk;
  const unsigned blocks = (unsigned)((n_chunks + 127) / 128);
  with_bool(write_pass, [&](auto write) {
    k_owner_positions<write()><<<blocks, 128, 0, stream>>>(states, masks, n, num_ranks, chunk, chunk_counts, chunk_base,
                                                           block, pos);
  });
  check_launch("k_owner_positions");
}

// -------------------------------------------------------------------------------------------------
// Peer-direct all-gather of x for the replicated-x product: every rank stores its block straight into slot `rank` of
// the gathered vector of EVERY rank (its own included) over NVLink -- one kernel, 8- or 16-byte coalesced stores to the
// CUDA-IPC-mapped buffers of the peers -- and then raises its flag in every peer with a system-scope release store; the
// consumer waits for all flags of the epoch with acquire loads (k_wait_flags).  Replaces the reference's
// PUT + `isEmpty` flag handshake (DMV:361-410) for the one exchange this form of the product has, and the NCCL
// all-gather whose latency dominated small blocks.
// -------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_push_block(const T *__restrict__ x, int64_t n_words, int num_ranks,
                                                    T *const *__restrict__ peer_slot, unsigned *done,
                                                    unsigned *const *__restrict__ peer_flags, int rank, unsigned epoch) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
    const T v = x[i];
    for (int q = 0; q < num_ranks; ++q) peer_slot[q][i] = v;
  }
  // one system-scope fence per CTA, after the CTA barrier (cumulative: it covers the stores of the whole CTA); a fence in
  // every warp serialises every warp of the CTA behind a system-scope fence
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {     // last CTA: every block of the grid has fenced its stores
      __threadfence_system();
      *done = 0;
      for (int q = 0; q < num_ranks; ++q) {
        unsigned *f = peer_flags[q] + rank;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(epoch) : "memory");
      }
    }
  }
}

// wait until every rank has raised flag[q] to `epoch`; gives up after ~4 s (a dead peer must not hang the box)
__global__ void k_wait_flags(const unsigned *flags, int num_ranks, unsigned epoch, unsigned long long *status) {
  const int q = threadIdx.x;
  if (q < num_ranks) {
    const long long t0 = clock64();
    for (;;) {
      unsigned v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + q) : "memory");
      if ((int)(v - epoch) >= 0) break;
      if (clock64() - t0 > 8000000000ll) { atomicAdd(status + 3, 1ull); break; }
      __nanosleep(200);
    }
  }
}

// raise my flag in every rank to `value` (after everything this stream has stored into the peers before)
__global__ void k_raise_flags(unsigned *const *__restrict__ peer_flags, int num_ranks, int rank, unsigned value) {
  const int q = threadIdx.x;
  if (q < num_ranks) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_flags[q] + rank), "r"(value) : "memory");
  }
}

void launch_raise_flags(unsigned *const *peer_flags, int num_ranks, int rank, unsigned value, cudaStream_t stream) {
  k_raise_flags<<<1, 32, 0, stream>>>(peer_flags, num_ranks, rank, value);
  check_launch("k_raise_flags");
}

void launch_push_block(const void *x, int64_t n_doubles, int num_ranks, void *const *peer_slot, unsigned *done,
                       unsigned *const *peer_flags, int rank, unsigned epoch, bool wide, cudaStream_t stream) {
  // wide: 16-byte words (x and every slot 16-byte aligned, even number of doubles)
  const int64_t words = wide ? n_doubles / 2 : n_doubles;
  // a few words per thread: fewer CTAs to fence and count
  const int blocks = capped_grid((words + 4 * 256 - 1) / (4 * 256), (int64_t)sm_count() * 4);
  with_bool(wide, [&](auto w) {
    using T = std::conditional_t<w(), double2, double>;
    k_push_block<T><<<blocks, 256, 0, stream>>>(reinterpret_cast<const T *>(x), words, num_ranks,
                                                reinterpret_cast<T *const *>(peer_slot), done, peer_flags, rank, epoch);
  });
  check_launch("k_push_block");
}

void launch_wait_flags(const unsigned *flags, int num_ranks, unsigned epoch, unsigned long long *status,
                       cudaStream_t stream) {
  k_wait_flags<<<1, 32, 0, stream>>>(flags, num_ranks, epoch, status);
  check_launch("k_wait_flags");
}

// p.groups / p.lut / p.bp must point at the ROW-traversal tables (see k_pull); complex_values says whether the
// LUT is the interleaved complex one.
void launch_gather(const KernelParams &p, bool inversion, bool complex_values, bool complex_elements,
                   bool narrow, bool lin, bool uniform, cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return;
  if (p.batch > 1 && p.batch != 4) throw std::runtime_error("k_gather: vectors come one or four at a time");
  const int rpt = 32 / (p.row_split > 1 ? p.row_split : 1);
  const int64_t tiles = (p.row_end - p.row_begin + rpt - 1) / rpt;
  with_bool(inversion, [&](auto inv) {
  with_bool(complex_values, [&](auto cv) {
  with_bool(complex_elements, [&](auto ce) {
  with_bool(narrow, [&](auto nw) {
  with_bool(lin, [&](auto ln) {
  with_bool(uniform, [&](auto uni) {
  with_choice<1, 4>(p.batch == 4 ? 4 : 1, [&](auto kb) {
    auto kernel = k_gather<inv(), cv(), ce(), nw(), ln(), uni(), kb()>;
    const size_t smem = gather_layout(p, nw() ? 4 : 8, sizeof(typename Val<cv()>::type), uni()).total;
    // whole waves of resident CTAs, grid-stride over the tiles
    const int grid = one_wave(kernel, (tiles + kThreads / 32 - 1) / (kThreads / 32), smem);
    kernel<<<grid, kThreads, smem, stream>>>(p);
    check_launch("k_gather");
  }); }); }); }); }); }); });
}

}  // namespace dmv
