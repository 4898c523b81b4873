// dmv_kernels.cu -- hand-written sm_90a kernels of the distributed matrix-free H.x product.
//
//   k_generate   : diagonal + off-diagonal term generation (BatchedOperator.computeOffDiag, reference
//                  src/BatchedOperator.chpl:82-213) fused with the destination hash (localeIdxOf,
//                  src/StatesEnumeration.chpl:129-136), the per-destination bucketing (radixOneStep,
//                  DMV:265-311) and -- for the records this rank owns -- the index search and atomic
//                  accumulate (localProcess, DMV:73-127).
//   k_accumulate : localProcess for records received from other ranks.
//
// Work decomposition of k_generate: a warp owns 32 consecutive source states (one per lane, coalesced
// 8-byte loads of sigma_i and x_i), walks the flip-mask groups of the operator in lock step (tables in
// shared memory, broadcast reads), and compacts the emitted (beta, c*x_i) pairs into a warp-private
// ring buffer in shared memory.  Whenever 32 entries are queued the warp drains them with all lanes
// busy: symmetry projection (orbit scan in registers), hash, directory + bounded binary search in the
// sorted representatives, FP64 atomic add.  This keeps the expensive part (projection, search,
// atomics) at full lane occupancy although only ~half of the (state, bond) pairs emit a term.
#include <cuda_runtime.h>

#include <atomic>
#include <stdexcept>
#include <string>

#include "dmv_host.h"

namespace dmv {

static std::atomic<int64_t> g_launches{0};
int64_t launch_counter() { return g_launches.load(); }
static void count_launch() { g_launches++; }

void check_launch(const char *what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
  count_launch();
}

// each process or thread of a multi-GPU run asks for its own device, so the count is kept per device ordinal
int sm_count() {
  constexpr int kDevices = 64;
  static std::atomic<int> cached[kDevices];
  int dev = 0;
  cudaGetDevice(&dev);
  const bool cacheable = dev >= 0 && dev < kDevices;
  int n = cacheable ? cached[dev].load(std::memory_order_relaxed) : 0;
  if (n > 0) return n;
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  if (n <= 0) n = 132;
  if (cacheable) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kQueue = 128;  // ring capacity per warp (>= 63 pending + 32 appended)

// ---- value helpers: V = double (real coefficients and real x) or double2 (complex) -------------
template <bool CV> struct ValT { using type = double; };
template <> struct ValT<true> { using type = double2; };

__device__ __forceinline__ double v_make(double re, double, double *) { return re; }
__device__ __forceinline__ double2 v_make(double re, double im, double2 *) { return make_double2(re, im); }
__device__ __forceinline__ double v_mul(double a, double b) { return a * b; }
__device__ __forceinline__ double2 v_mul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double v_scale(double a, double s) { return a * s; }
__device__ __forceinline__ double2 v_scale(double2 a, double s) { return make_double2(a.x * s, a.y * s); }
__device__ __forceinline__ bool v_nonzero(double a) { return a != 0.0; }
__device__ __forceinline__ bool v_nonzero(double2 a) { return a.x != 0.0 || a.y != 0.0; }
__device__ __forceinline__ void v_acc(double &a, double re, double) { a += re; }
__device__ __forceinline__ void v_acc(double2 &a, double re, double im) { a.x += re; a.y += im; }

template <bool CE>
__device__ __forceinline__ void atomic_accumulate(void *y, int64_t idx, double re, double im) {
  if (CE) {
    double *p = reinterpret_cast<double *>(y) + 2 * idx;
    atomicAdd(p, re);
    atomicAdd(p + 1, im);
  } else {
    atomicAdd(reinterpret_cast<double *>(y) + idx, re);
  }
}
__device__ __forceinline__ double v_re(double a) { return a; }
__device__ __forceinline__ double v_re(double2 a) { return a.x; }
__device__ __forceinline__ double v_im(double) { return 0.0; }
__device__ __forceinline__ double v_im(double2 a) { return a.y; }

// ---- shared-memory staging of the operator / orbit tables ---------------------------------------
struct SmemLayout {
  size_t groups, gx, bp, lut, terms, diag, dclass, orbit64, orbit32, canon, binom, queues, total;
};
__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
__host__ __device__ inline SmemLayout smem_layout(const KernelParams &p, int proj, size_t val_bytes,
                                                  bool queues = true) {
  SmemLayout L;
  size_t off = 0;
  // bit-parallel mode keeps only the flip masks (compact) and the word descriptors; the full group
  // records are needed when groups are walked one by one or carry an outside sign mask
  const bool full_groups = p.n_bp == 0 || p.any_s_out;
  L.groups = off; off += full_groups ? sizeof(LutGroup) * p.n_groups : 0;
  L.gx = off; off += 8 * (size_t)p.n_groups;
  L.bp = off; off += sizeof(BpWord) * p.n_bp;
  off = align_up(off, 16);
  L.lut = off; off += val_bytes * p.n_lut;
  off = align_up(off, 8);
  L.terms = off; off += p.any_generic ? sizeof(OffTerm) * p.n_terms : 0;
  L.diag = off; off += sizeof(DiagTerm) * p.n_diag_rest;
  L.dclass = off; off += sizeof(DiagClass) * p.n_diag_classes;
  off = align_up(off, 16);   // packed orbit steps are read with 16-byte loads
  L.orbit64 = off;
  size_t n64 = 0, n32 = 0;
  if (proj == PROJ_GROUP) {
    const int np = p.orbit.n_left + p.orbit.n_right;
    const size_t steps = (size_t)(p.orbit.n_t - 1);
    n64 = (size_t)p.orbit.n_q * p.orbit.n_stages;
    if (n64 & 1) ++n64;   // keep the packed steps 16-byte aligned
    n32 = (size_t)p.orbit.n_stages;
    if (p.orbit.simple) n64 += p.orbit.step_pack32 ? 2 * steps : 3 * steps;   // packed steps only
    else { n64 += steps * np; n32 += steps * np; }
  }
  off += 8 * n64;
  L.orbit32 = off; off += 4 * n32;
  // canonical-form scan: coset chain (masks, then begin / delta) and the pair LUT
  off = align_up(off, 8);
  L.canon = off;
  if (proj == PROJ_GROUP && p.orbit.canon_mode != 0 && p.orbit.tor_mode != 0) {
    // full-space-group canonical form: delta-swap stages of rho / tau and the 32-bit pair table
    const size_t n_st = (size_t)(p.orbit.tor_rho_n + p.orbit.tor_tau_n);
    off += 8 * n_st + 4 * n_st;
    off = align_up(off, 16);                                    // bulk copies need 16-byte aligned destinations
    off += 4 * ((size_t)1 << (2 * p.orbit.canon_k));            // tor_lutm
    off += align_up((size_t)4 * p.orbit.canon_k << p.orbit.canon_k, 16);   // tor_frow
    off += 16;                                                  // mbarrier of the bulk copies
    off = align_up(off, 8);
  } else if (proj == PROJ_GROUP && p.orbit.canon_mode != 0) {
    const size_t n_st = p.orbit.cc_n > 0 ? (size_t)p.orbit.cc_stages : 0;
    off += 8 * n_st + 4 * (n_st + (p.orbit.cc_n > 0 ? (size_t)p.orbit.cc_n + 1 : 0));
    off = align_up(off, 4);
    if (p.orbit.canon_lut2) off += 4 * ((size_t)1 << (2 * p.orbit.canon_k));
  }
  L.binom = off;
  if (p.index.mode == INDEX_RANK) off += 4 * (size_t)p.index.n_sites * p.index.stride;
  off = align_up(off, 16);
  // per warp: ring of (beta, value) + (pull mode) source lane and a row accumulator
  L.queues = off; off += queues ? (size_t)kWarps * (kQueue * (8 + val_bytes) + kQueue + 32 * val_bytes) : 0;
  L.total = off;
  return L;
}

template <typename T>
__device__ __forceinline__ void stage(T *dst, const T *src, int count) {
  for (int i = threadIdx.x; i < count; i += blockDim.x) dst[i] = src[i];
}

// Two global -> shared bulk copies through the TMA engine (cp.async.bulk; sizes multiples of 16, 16-byte aligned), issued
// by one thread and awaited by the whole CTA on an mbarrier.  The source buffers are over-allocated to the padded size.
__device__ __forceinline__ void bulk_stage2(void *dst0, const void *src0, uint32_t bytes0, void *dst1, const void *src1,
                                            uint32_t bytes1, uint64_t *mbar) {
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(mbar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes0 + bytes1) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(dst0)), "l"(src0), "r"(bytes0), "r"(bar) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(dst1)), "l"(src1), "r"(bytes1), "r"(bar) : "memory");
  }
  uint32_t done = 0;
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar) : "memory");
  }
}

// Everything a CTA keeps in shared memory, set up once per CTA.
template <bool CV>
struct Tables {
  using V = typename ValT<CV>::type;
  const LutGroup *groups;
  const uint64_t *gx;   // flip mask of every group
  const BpWord *bp;
  int n_bp;
  const V *lut;
  const OffTerm *terms;
  const DiagTerm *diag;
  const DiagClass *dclass;
  int n_diag_rest, n_dclass;
  OrbitProgram orbit;
  StateIndex index;
};

template <int PROJ, bool CV>
__device__ __forceinline__ Tables<CV> stage_tables(const KernelParams &p, unsigned char *smem, const SmemLayout &L) {
  using V = typename ValT<CV>::type;
  Tables<CV> T;
  LutGroup *s_groups = reinterpret_cast<LutGroup *>(smem + L.groups);
  V *s_lut = reinterpret_cast<V *>(smem + L.lut);
  OffTerm *s_terms = reinterpret_cast<OffTerm *>(smem + L.terms);
  DiagTerm *s_diag = reinterpret_cast<DiagTerm *>(smem + L.diag);
  uint64_t *s_gx = reinterpret_cast<uint64_t *>(smem + L.gx);
  BpWord *s_bp = reinterpret_cast<BpWord *>(smem + L.bp);
  if (p.n_bp == 0 || p.any_s_out) stage(s_groups, p.groups, p.n_groups);
  for (int i = threadIdx.x; i < p.n_groups; i += blockDim.x) s_gx[i] = p.groups[i].x;
  stage(reinterpret_cast<uint64_t *>(s_bp), reinterpret_cast<const uint64_t *>(p.bp),
        p.n_bp * (int)(sizeof(BpWord) / 8));
  T.gx = s_gx; T.bp = s_bp; T.n_bp = p.n_bp;
  stage(s_lut, reinterpret_cast<const V *>(p.lut), p.n_lut);
  if (p.any_generic) stage(s_terms, p.terms, p.n_terms);
  stage(s_diag, p.diag, p.n_diag_rest);
  DiagClass *s_dclass = reinterpret_cast<DiagClass *>(smem + L.dclass);
  stage(reinterpret_cast<uint64_t *>(s_dclass), reinterpret_cast<const uint64_t *>(p.diag_classes),
        p.n_diag_classes * (int)(sizeof(DiagClass) / 8));
  T.groups = s_groups; T.lut = s_lut; T.terms = s_terms; T.diag = s_diag;
  T.dclass = s_dclass; T.n_diag_rest = p.n_diag_rest; T.n_dclass = p.n_diag_classes;
  T.orbit = p.orbit;
  if (PROJ == PROJ_GROUP) {
    const int np = T.orbit.n_left + T.orbit.n_right;
    uint64_t *s64 = reinterpret_cast<uint64_t *>(smem + L.orbit64);
    int32_t *s32 = reinterpret_cast<int32_t *>(smem + L.orbit32);
    const int nb = T.orbit.n_q * T.orbit.n_stages, steps = T.orbit.n_t - 1;
    const int nb_pad = nb + (nb & 1);
    stage(s64, p.orbit.benes_mask, nb);
    stage(s32, p.orbit.benes_delta, T.orbit.n_stages);
    T.orbit.benes_mask = s64;
    T.orbit.benes_delta = s32;
    if (T.orbit.simple) {
      // only the packed steps live in shared memory; the general arrays (rare paths) stay in global
      if (p.orbit.step_pack32) {
        stage(s64 + nb_pad, reinterpret_cast<const uint64_t *>(p.orbit.step_pack32), 2 * steps);
        T.orbit.step_pack32 = reinterpret_cast<const uint4 *>(s64 + nb_pad);
      } else {
        stage(s64 + nb_pad, p.orbit.step_pack64, 3 * steps);
        T.orbit.step_pack64 = s64 + nb_pad;
      }
    } else {
      stage(s64 + nb_pad, p.orbit.step_mask, steps * np);
      stage(s32 + T.orbit.n_stages, p.orbit.step_shift, steps * np);
      T.orbit.step_mask = s64 + nb_pad;
      T.orbit.step_shift = s32 + T.orbit.n_stages;
    }
  }
  if (PROJ == PROJ_GROUP && T.orbit.canon_mode != 0 && T.orbit.tor_mode != 0) {
    unsigned char *base = smem + L.canon;
    const int n_st = T.orbit.tor_rho_n + T.orbit.tor_tau_n;
    uint64_t *nm = reinterpret_cast<uint64_t *>(base);
    int32_t *nd = reinterpret_cast<int32_t *>(base + 8 * (size_t)n_st);
    uint32_t *lm = reinterpret_cast<uint32_t *>(smem + align_up((size_t)(base - smem) + 12 * (size_t)n_st, 16));
    stage(nm, p.orbit.tor_net_mask, n_st);
    stage(nd, p.orbit.tor_net_delta, n_st);
    // the pair table (16 KB for k = 6) and the row table arrive as two TMA bulk copies (cp.async.bulk, one elected
    // thread, completion on an mbarrier) instead of a strided loop of every thread
    const uint32_t lut_bytes = 4u << (2 * T.orbit.canon_k);
    const uint32_t frow_bytes = (uint32_t)align_up((size_t)4 * T.orbit.canon_k << T.orbit.canon_k, 16);
    uint8_t *fr = reinterpret_cast<uint8_t *>(lm) + lut_bytes;
    uint64_t *mbar = reinterpret_cast<uint64_t *>(fr + frow_bytes);
    bulk_stage2(lm, p.orbit.tor_lutm, lut_bytes, fr, p.orbit.tor_frow, frow_bytes, mbar);
    T.orbit.tor_net_mask = nm; T.orbit.tor_net_delta = nd; T.orbit.tor_lutm = lm; T.orbit.tor_frow = fr;
  } else if (PROJ == PROJ_GROUP && T.orbit.canon_mode != 0) {
    unsigned char *base = smem + L.canon;
    if (T.orbit.cc_n > 0) {
      const int n_st = T.orbit.cc_stages;
      uint64_t *cm = reinterpret_cast<uint64_t *>(base);
      int32_t *cb = reinterpret_cast<int32_t *>(base + 8 * (size_t)n_st);
      int32_t *cd = cb + (T.orbit.cc_n + 1);
      stage(cm, p.orbit.cc_mask, n_st);
      stage(cb, p.orbit.cc_begin, T.orbit.cc_n + 1);
      stage(cd, p.orbit.cc_delta, n_st);
      T.orbit.cc_mask = cm; T.orbit.cc_begin = cb; T.orbit.cc_delta = cd;
      base += 8 * (size_t)n_st + 4 * ((size_t)n_st + T.orbit.cc_n + 1);
    }
    base = smem + align_up((size_t)(base - smem), 4);
    if (T.orbit.canon_lut2) {
      uint32_t *l2 = reinterpret_cast<uint32_t *>(base);
      stage(l2, p.orbit.canon_lut2, 1 << (2 * T.orbit.canon_k));
      T.orbit.canon_lut2 = l2;
    }
  }
  T.index = p.index;
  if (T.index.mode == INDEX_RANK) {
    uint32_t *sb = reinterpret_cast<uint32_t *>(smem + L.binom);
    stage(sb, p.index.binom, T.index.n_sites * T.index.stride);
    T.index.binom = sb;
  }
  return T;
}

// ---- term generation ----------------------------------------------------------------------------
// generic (term by term) evaluation of one group: c = sum_t v_t [a & m == r] (-1)^popc(a & s)
template <bool CV>
__device__ __noinline__ typename ValT<CV>::type generic_coefficient(const OffTerm *terms, int first, int count,
                                                                     uint64_t a, bool *hit) {
  using V = typename ValT<CV>::type;
  V c = v_make(0.0, 0.0, (V *)nullptr);
  bool any = false;
  for (int t = first; t < first + count; ++t) {
    const OffTerm term = terms[t];
    if ((a & term.m) == term.r) {
      const double sg = (__popcll(a & term.s) & 1) ? -1.0 : 1.0;
      v_acc(c, sg * term.v_re, sg * term.v_im);
      any = true;
    }
  }
  *hit = any;
  return c;
}

// The terms one row emits within a word of <= 64 groups.
struct RowTerms {
  uint64_t mask;     // bit g - g0 set <=> group g emits
  uint64_t a0, a1;   // bit-parallel mode: the two support bits of every group (for the LUT index)
};

// All lanes evaluate the same word in lock step (table reads are shared-memory broadcasts).
template <bool CV>
__device__ __forceinline__ RowTerms row_terms(const Tables<CV> &T, int w, int g0, int g1, uint64_t a) {
  RowTerms rt;
  rt.mask = 0; rt.a0 = 0; rt.a1 = 0;
  if (T.n_bp > 0) {
    const BpWord &W = T.bp[w];
#pragma unroll 1
    for (int k = 0; k < W.n0; ++k) { const BpPair q = W.p0[k]; rt.a0 |= ((a << q.l) >> q.r) & q.m; }
#pragma unroll 1
    for (int k = 0; k < W.n1; ++k) { const BpPair q = W.p1[k]; rt.a1 |= ((a << q.l) >> q.r) & q.m; }
    rt.mask = (~rt.a0 & ~rt.a1 & W.tt[0]) | (rt.a0 & ~rt.a1 & W.tt[1]) | (~rt.a0 & rt.a1 & W.tt[2]) |
              (rt.a0 & rt.a1 & W.tt[3]);
    return rt;
  }
  for (int g = g0; g < g1; ++g) {
    const uint64_t posk = T.groups[g].posk;
    bool emit;
    if (posk >> 56) {
      bool hit;
      const auto c = generic_coefficient<CV>(T.terms, T.groups[g].first, T.groups[g].count, a, &hit);
      emit = hit && v_nonzero(c);   // same decision in the counting pass: the plan is exact
    } else {
      emit = (T.groups[g].emit_bits >> lut_index(posk, a)) & 1ull;
    }
    rt.mask |= (uint64_t)emit << (g - g0);
  }
  return rt;
}

// Pops the lowest emitting group of the row: returns its flip mask and coefficient for state a.
template <bool CV>
__device__ __forceinline__ typename ValT<CV>::type pop_term(const Tables<CV> &T, RowTerms &rt, int g0, uint64_t a,
                                                             bool any_s_out, uint64_t &flip) {
  using V = typename ValT<CV>::type;
  const int gl = __ffsll((long long)rt.mask) - 1;
  rt.mask &= rt.mask - 1;
  const int g = g0 + gl;
  flip = T.gx[g];
  V c;
  if (T.n_bp > 0) {
    const unsigned idx = (unsigned)((rt.a0 >> gl) & 1ull) | ((unsigned)((rt.a1 >> gl) & 1ull) << 1);
    c = T.lut[4 * g + idx];
    if (any_s_out && (__popcll(a & T.groups[g].s_out) & 1)) c = v_scale(c, -1.0);
    return c;
  }
  const LutGroup grp = T.groups[g];
  if (grp.posk >> 56) {
    bool hit;
    return generic_coefficient<CV>(T.terms, grp.first, grp.count, a, &hit);
  }
  c = T.lut[grp.lut_offset + lut_index(grp.posk, a)];
  if (any_s_out && (__popcll(a & grp.s_out) & 1)) c = v_scale(c, -1.0);
  return c;
}

template <bool CV>
__device__ __forceinline__ void diagonal(const Tables<CV> &T, int /*n_diag*/, uint64_t a, double &dre, double &dim) {
  dre = 0.0; dim = 0.0;
  // zz-like couplings, one class per distinct coefficient: count - 2 popc(antiparallel bonds)
  for (int c = 0; c < T.n_dclass; ++c) {
    const DiagClass &D = T.dclass[c];
    uint64_t a0 = 0, a1 = 0;
#pragma unroll 1
    for (int k = 0; k < D.n0; ++k) { const BpPair q = D.p0[k]; a0 |= ((a << q.l) >> q.r) & q.m; }
#pragma unroll 1
    for (int k = 0; k < D.n1; ++k) { const BpPair q = D.p1[k]; a1 |= ((a << q.l) >> q.r) & q.m; }
    const double w = (double)(D.count - 2 * __popcll((a0 ^ a1) & D.mask));
    dre += w * D.v_re;
    dim += w * D.v_im;
  }
  for (int t = 0; t < T.n_diag_rest; ++t) {
    const DiagTerm d = T.diag[t];
    if ((a & d.m) == d.r) {
      const double sg = (__popcll(a & d.s) & 1) ? -1.0 : 1.0;
      dre += sg * d.v_re;
      dim += sg * d.v_im;
    }
  }
}

// ---- the consumer side: one record per lane -----------------------------------------------------
// route(): projects beta (inversion / full group) and appends the record to the bucket of its owner when
// that is another rank.  Returns true when the record is this rank's own (to be searched + accumulated).
// All 32 lanes must call it (warp collectives); `active` lanes carry a record.
// FS (fermionic bases, PROJ_GROUP): the character of the element carries the exchange sign sign(g, beta) (orbit_sign)
template <int PROJ, bool CV, bool CE, bool COUNT_ONLY, bool FS = false>
__device__ __forceinline__ bool route(const KernelParams &p, const OrbitProgram &orbit, bool active,
                                      uint64_t &beta, typename ValT<CV>::type &c, unsigned long long &cur) {
  using V = typename ValT<CV>::type;
  const unsigned lane = threadIdx.x & 31u;
  if (PROJ == PROJ_INVERSION) {
    // reference src/BatchedOperator.chpl:145-152
    const uint64_t inv = beta ^ p.site_mask;
    if (inv < beta) { beta = inv; c = v_scale(c, p.inversion_character); }
  } else if (PROJ == PROJ_GROUP) {
    if (active) {
      if (orbit.trivial_characters) {
        beta = orbit_representative(orbit, beta);
      } else {
        const OrbitResult r = orbit_scan<false, false>(orbit, beta);
        const double2 chi = __ldg(orbit.characters + r.arg);   // state_info returns conj(chi)
        c = v_mul(c, v_make(chi.x, -chi.y, (V *)nullptr));
        if (FS) c = v_scale(c, orbit_sign(orbit, r.arg, beta));   // fermionic exchange sign
        beta = r.rep;
      }
    }
  }
  int owner = p.rank;
  if (p.num_ranks > 1) owner = locale_idx_of(beta, p.num_ranks);

  if (p.emit_all) {   // BatchedOperator.computeOffDiag output: (beta, coeff, key) flat, unordered
    if (active && !COUNT_ONLY) {
      if (PROJ == PROJ_GROUP) {   // norm of the representative: BO:200 `norms[k]`
        const double stab = orbit.trivial_characters ? (double)orbit_scan<true, false>(orbit, beta).stab
                                                     : orbit_stabiliser_sum<FS>(orbit, beta);
        const double nn = stab / (double)orbit.group_order;
        c = v_scale(c, nn > 1e-12 ? sqrt(nn) : 0.0);
      }
      const unsigned long long pos = atomicAdd(p.out_count, 1ull);
      if ((int64_t)pos < p.out_offset[1]) {
        p.out_betas[pos] = beta;
        reinterpret_cast<V *>(p.out_coeffs)[pos] = c;
        p.out_keys[pos] = (uint8_t)owner;
      }
    }
    return false;
  }

  if (p.num_ranks <= 32 && (p.num_ranks > 1 || COUNT_ONLY)) {
    // ---- remote records: lane d keeps this warp's cursor into destination d's region (exact regions
    // from the plan: no atomics).  In the counting pass every record (own ones too) is counted.
    const bool remote = active && (COUNT_ONLY || owner != p.rank);
    for (int d = 0; d < p.num_ranks; ++d) {   // warp-uniform
      const bool mine = remote && owner == d;
      const unsigned m = __ballot_sync(0xffffffffu, mine);
      if (m) {
        const unsigned long long base = __shfl_sync(0xffffffffu, cur, d);
        if (!COUNT_ONLY && mine) {
          const int64_t slot = (int64_t)base + __popc(m & ((1u << lane) - 1u));
          if (slot < p.out_capacity[d]) {
            p.out_betas_ptr[d][slot] = beta;
            reinterpret_cast<V *>(p.out_coeffs_ptr[d])[slot] = c;
          } else {
            atomicAdd(p.status + 2, 1ull);
          }
        }
        if ((int)lane == d) cur += __popc(m);
      }
    }
    if (COUNT_ONLY) return false;
    return active && owner == p.rank;
  }
  if (p.num_ranks > 1) {
    // ---- more than 32 ranks: warp-aggregated slot claim per destination with global atomics
    const bool remote = active && (COUNT_ONLY || owner != p.rank);
    const unsigned remote_mask = __ballot_sync(0xffffffffu, remote);
    if (remote) {
      const unsigned peers = __match_any_sync(remote_mask, owner);
      const int leader = __ffs(peers) - 1;
      unsigned long long base = 0;
      if ((int)lane == leader) base = atomicAdd(p.out_count + owner, (unsigned long long)__popc(peers));
      base = __shfl_sync(peers, base, leader);
      if (!COUNT_ONLY) {
        const int64_t pos = (int64_t)base + __popc(peers & ((1u << lane) - 1u));
        const int64_t cap = p.out_offset[owner + 1] - p.out_offset[owner];
        if (pos < cap) {
          const int64_t slot = p.out_offset[owner] + pos;
          p.out_betas[slot] = beta;
          reinterpret_cast<V *>(p.out_coeffs)[slot] = c;
        } else {
          atomicAdd(p.status + 2, 1ull);
        }
      }
    }
    if (COUNT_ONLY) return false;
    return active && owner == p.rank;
  }
  return active;
}

// finish(): localProcess (reference DMV:73-127) for one located record
template <int PROJ, bool CV, bool CE, bool FS = false>
__device__ __forceinline__ void finish(const KernelParams &p, const OrbitProgram &orbit, bool active,
                                       uint64_t beta, typename ValT<CV>::type c, int64_t idx) {
  if (!active) return;
  if (idx >= 0) {
    if (PROJ == PROJ_GROUP) c = v_scale(c, __ldg(p.norms + idx));
    if (v_nonzero(c)) atomic_accumulate<CE>(p.y, idx, v_re(c), v_im(c));   // DMV:110: skip c == 0
  } else if (v_nonzero(c)) {
    bool fatal = true;
    if (PROJ == PROJ_GROUP && !orbit.trivial_characters)
      fatal = orbit_stabiliser_sum<FS>(orbit, beta) > 1e-12 * (double)orbit.group_order;  // zero-norm orbit
    if (fatal) {                                                             // DMV:115-118
      if (atomicAdd(p.status, 1ull) == 0) p.status[1] = beta;
    }
  }
}

// Two independent searches advanced in lock step: both directory loads, then both probes of every
// level, are in flight together (the search is a chain of dependent L2 accesses; this doubles the
// memory-level parallelism of a warp).
__device__ __forceinline__ void locate2(const StateIndex &ix, bool a0, uint64_t k0, bool a1, uint64_t k1,
                                        int64_t &i0, int64_t &i1) {
  if (ix.mode != INDEX_DIRECTORY) {
    i0 = a0 ? locate(ix, k0) : -1;
    i1 = a1 ? locate(ix, k1) : -1;
    return;
  }
  i0 = -1; i1 = -1;
  const uint64_t b0 = k0 >> ix.shift, b1 = k1 >> ix.shift;
  a0 = a0 && b0 < ix.n_buckets;
  a1 = a1 && b1 < ix.n_buckets;
  uint2 r0 = make_uint2(0, 0), r1 = make_uint2(0, 0);
  if (a0) r0 = __ldg(reinterpret_cast<const uint2 *>(ix.dir) + b0);
  if (a1) r1 = __ldg(reinterpret_cast<const uint2 *>(ix.dir) + b1);
  uint32_t lo0 = r0.x, hi0 = r0.y, lo1 = r1.x, hi1 = r1.y;
  while (lo0 < hi0 || lo1 < hi1) {
    const bool s0 = lo0 < hi0, s1 = lo1 < hi1;
    const uint32_t m0 = (lo0 + hi0) >> 1, m1 = (lo1 + hi1) >> 1;
    uint64_t v0 = 0, v1 = 0;
    if (s0) v0 = __ldg(ix.reps + m0);
    if (s1) v1 = __ldg(ix.reps + m1);
    if (s0) {
      if (v0 == k0) { i0 = m0; lo0 = hi0; }
      else if (v0 < k0) lo0 = m0 + 1; else hi0 = m0;
    }
    if (s1) {
      if (v1 == k1) { i1 = m1; lo1 = hi1; }
      else if (v1 < k1) lo1 = m1 + 1; else hi1 = m1;
    }
  }
}

// Drain up to 64 queued records of this warp: lane handles entries `lane` and `lane + 32`.
template <int PROJ, bool CV, bool CE, bool COUNT_ONLY, bool FS>
__device__ __forceinline__ void drain(const KernelParams &p, const OrbitProgram &orbit, const StateIndex &index,
                                      const uint64_t *qb, const typename ValT<CV>::type *qc, unsigned head,
                                      unsigned n, unsigned long long &cur) {
  using V = typename ValT<CV>::type;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned p0 = (head + lane) & (kQueue - 1), p1 = (head + lane + 32) & (kQueue - 1);
  bool a0 = lane < n, a1 = lane + 32 < n;
  uint64_t k0 = a0 ? qb[p0] : 0ull, k1 = a1 ? qb[p1] : 0ull;
  V c0 = a0 ? qc[p0] : v_make(0.0, 0.0, (V *)nullptr), c1 = a1 ? qc[p1] : v_make(0.0, 0.0, (V *)nullptr);
  a0 = route<PROJ, CV, CE, COUNT_ONLY, FS>(p, orbit, a0, k0, c0, cur);
  if (n > 32) a1 = route<PROJ, CV, CE, COUNT_ONLY, FS>(p, orbit, a1, k1, c1, cur);   // n is warp-uniform
  else a1 = false;
  if (COUNT_ONLY) return;
  int64_t i0, i1;
  locate2(index, a0, k0, a1, k1, i0, i1);
  finish<PROJ, CV, CE, FS>(p, orbit, a0, k0, c0, i0);
  finish<PROJ, CV, CE, FS>(p, orbit, a1, k1, c1, i1);
}

// (symmetric bases: the orbit scan wants > 100 registers; three resident CTAs per SM hide its latencies better than
// two, at the price of a few spills outside the scan)
template <int PROJ, bool CV, bool CE, bool COUNT_ONLY, bool FS>
__global__ void __launch_bounds__(kThreads, PROJ == PROJ_GROUP ? 3 : 1) k_generate(const KernelParams p) {
  using V = typename ValT<CV>::type;
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ, sizeof(V));
  const Tables<CV> T = stage_tables<PROJ, CV>(p, smem, L);
  __syncthreads();

  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  uint64_t *qb = reinterpret_cast<uint64_t *>(smem + L.queues) + warp * kQueue;
  V *qc = reinterpret_cast<V *>(smem + L.queues + (size_t)kWarps * kQueue * 8) + warp * kQueue;
  unsigned head = 0, count = 0;  // warp-uniform
  const bool any_s_out = p.any_s_out != 0;
  // lane d: cursor of this warp in destination d's region (see route())
  const int64_t gw = (int64_t)blockIdx.x * kWarps + warp;
  unsigned long long cur = 0;
  if (!COUNT_ONLY && p.num_ranks > 1 && p.num_ranks <= 32 && (int)lane < p.num_ranks)
    cur = (unsigned long long)p.warp_offsets[gw * p.num_ranks + lane];

  // row_split = S lanes share one source state (each takes every S-th flip-mask group): small bases get
  // S times more warps and S times shorter per-warp latency chains; large ones run with S = 1
  const int S = p.row_split > 1 ? p.row_split : 1;
  const int rows_per_tile = 32 / S;
  const unsigned slice = lane & (unsigned)(S - 1);
  uint64_t slice_mask = ~0ull;
  if (S > 1) {
    slice_mask = 0;
    for (int g = (int)slice; g < 64; g += S) slice_mask |= 1ull << g;
  }
  const int64_t n_rows = p.row_end - p.row_begin;
  const int64_t n_tiles = (n_rows + rows_per_tile - 1) / rows_per_tile;
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += warps_total) {
    const int64_t i = p.row_begin + tile * rows_per_tile + lane / S;
    const bool valid = i < p.row_end;
    uint64_t alpha = 0;
    V xi = v_make(0.0, 0.0, (V *)nullptr);
    if (valid) {
      alpha = __ldg(p.index.reps + i);
      if (!COUNT_ONLY) {
        if (CE) {
          const double2 t = __ldg(reinterpret_cast<const double2 *>(p.x) + i);
          xi = v_make(t.x, t.y, (V *)nullptr);
        } else {
          xi = v_make(__ldg(reinterpret_cast<const double *>(p.x) + i), 0.0, (V *)nullptr);
        }
      }
    }
    // ---- diagonal: y[i] += x[i] * sum_t v_t [alpha & m == r] (-1)^popc(alpha & s)   (DMV:36-53)
    if (!COUNT_ONLY && !p.emit_all && p.n_diag > 0 && valid && slice == 0) {
      double dre, dim;
      diagonal<CV>(T, p.n_diag, alpha, dre, dim);
      if (CE) {
        const double2 t = __ldg(reinterpret_cast<const double2 *>(p.x) + i);
        atomic_accumulate<true>(p.y, i, dre * t.x - dim * t.y, dre * t.y + dim * t.x);
      } else {
        // real vectors take the real part of the diagonal (ls_internal_operator_apply_diag_x1 on real(64))
        atomic_accumulate<false>(p.y, i, dre * __ldg(reinterpret_cast<const double *>(p.x) + i), 0.0);
      }
    }
    if (PROJ == PROJ_GROUP && valid && !COUNT_ONLY)
      xi = v_scale(xi, 1.0 / __ldg(p.norms + i));   // 1 / norm(alpha): BO:200

    // ---- off-diagonal: which groups emit (bit mask), then compact the emitted terms into the ring
    for (int g0 = 0, w = 0; g0 < p.n_groups; g0 += 64, ++w) {
      const int g1 = min(g0 + 64, p.n_groups);
      RowTerms rt = row_terms<CV>(T, w, g0, g1, alpha);
      rt.mask &= slice_mask;
      if (!valid) rt.mask = 0;
      for (;;) {
        const bool has = rt.mask != 0;
        const unsigned m = __ballot_sync(0xffffffffu, has);
        if (m == 0) break;
        if (has) {
          uint64_t flip;
          const V c = pop_term<CV>(T, rt, g0, alpha, any_s_out, flip);
          const unsigned pos = (head + count + __popc(m & ((1u << lane) - 1u))) & (kQueue - 1);
          qb[pos] = alpha ^ flip;
          if (!COUNT_ONLY) qc[pos] = v_mul(c, xi);
        }
        count += __popc(m);
        if (count >= 64) {
          __syncwarp();
          drain<PROJ, CV, CE, COUNT_ONLY, FS>(p, T.orbit, T.index, qb, qc, head, 64, cur);
          head = (head + 64) & (kQueue - 1);
          count -= 64;
          __syncwarp();
        }
      }
    }
  }
  if (count > 0) {
    __syncwarp();
    drain<PROJ, CV, CE, COUNT_ONLY, FS>(p, T.orbit, T.index, qb, qc, head, count, cur);
  }
  if (COUNT_ONLY && p.num_ranks <= 32 && (int)lane < p.num_ranks)
    p.warp_counts[gw * p.num_ranks + lane] = cur;
}

// -------------------------------------------------------------------------------------------------
// k_pull: the same product traversed by ROWS (gather) -- used when one rank owns the whole basis.
//   y[b] = D(b) x[b] + sum_t <b|t|b^x_t> chi(g) n_a / n_b x[index(a)],   a = rep(b ^ x_t), g(b^x_t) = a
// with <b|t|b^x> = v (-1)^popc(x&s) [b & m == r ^ (x & m)] (-1)^popc(b & s): the term table is
// transformed once on the host (terms_adj).  Same generate -> project -> search pipeline as
// k_generate, but the scattered FP64 atomics of localProcess (DMV:107-120) become scattered loads of x
// and every y element is written exactly once (deterministic, no memset, half the L2 traffic).
// -------------------------------------------------------------------------------------------------
template <bool CE>
__device__ __forceinline__ typename ValT<CE>::type load_x(const void *x, int64_t i) {
  if (CE) {
    const double2 t = __ldg(reinterpret_cast<const double2 *>(x) + i);
    return v_make(t.x, t.y, (typename ValT<CE>::type *)nullptr);
  }
  return v_make(__ldg(reinterpret_cast<const double *>(x) + i), 0.0, (typename ValT<CE>::type *)nullptr);
}
__device__ __forceinline__ double to_v(double a, double *) { return a; }
__device__ __forceinline__ double2 to_v(double a, double2 *) { return make_double2(a, 0.0); }
__device__ __forceinline__ double2 to_v(double2 a, double2 *) { return a; }
__device__ __forceinline__ void v_add(double &a, double b) { a += b; }
__device__ __forceinline__ void v_add(double2 &a, double2 b) { a.x += b.x; a.y += b.y; }
__device__ __forceinline__ void smem_add(double *p, double v) { atomicAdd(p, v); }
__device__ __forceinline__ void smem_add(double2 *p, double2 v) { atomicAdd(&p->x, v.x); atomicAdd(&p->y, v.y); }

template <int PROJ, bool CV, bool CE, bool FS>
__global__ void __launch_bounds__(kThreads) k_pull(const KernelParams p) {
  using V = typename ValT<CV>::type;
  using E = typename ValT<CE>::type;
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ, sizeof(V));
  const Tables<CV> T = stage_tables<PROJ, CV>(p, smem, L);   // p.groups / p.lut / p.terms: row-traversal tables
  const OrbitProgram &orbit = T.orbit;
  const StateIndex &index = T.index;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  unsigned char *qbase = smem + L.queues;
  uint64_t *qb = reinterpret_cast<uint64_t *>(qbase) + warp * kQueue;
  V *qc = reinterpret_cast<V *>(qbase + (size_t)kWarps * kQueue * 8) + warp * kQueue;
  V *acc_s = reinterpret_cast<V *>(qbase + (size_t)kWarps * kQueue * (8 + sizeof(V))) + warp * 32;
  unsigned char *ql = qbase + (size_t)kWarps * (kQueue * (8 + sizeof(V)) + 32 * sizeof(V)) + warp * kQueue;
  if (PROJ == PROJ_GROUP) acc_s[lane] = v_make(0.0, 0.0, (V *)nullptr);
  __syncthreads();
  unsigned head = 0, count = 0;
  const bool any_s_out = p.any_s_out != 0;
  // replicated-x product: rows are this rank's block, `index` / `norms` describe the global basis, global index g
  // lives at x[pos[g]] (see dmv_host.h)
  const uint64_t *__restrict__ row_states = p.row_states ? p.row_states : p.index.reps;
  const double *__restrict__ row_norms = p.row_norms ? p.row_norms : p.norms;
  const uint32_t *__restrict__ xslot = p.pos;

  // drains `k` queued entries (PROJ_GROUP): orbit scan, search, gather, add into the owner row's slot
  auto drain = [&](unsigned k) {
    const bool active = lane < k;
    if (active) {
      const unsigned pos = (head + lane) & (kQueue - 1);
      const uint64_t raw = qb[pos];
      V h = qc[pos];
      const unsigned src = ql[pos];
      OrbitResult r;
      if (orbit.trivial_characters) {
        r.rep = orbit_representative(orbit, raw);
      } else {
        r = orbit_scan<false, false>(orbit, raw);
        const double2 chi = __ldg(orbit.characters + r.arg);   // chi(g), not conjugated (see header)
        h = v_mul(h, v_make(chi.x, chi.y, (V *)nullptr));
        if (FS) h = v_scale(h, orbit_sign(orbit, r.arg, raw));   // fermionic exchange sign
      }
      const int64_t idx = locate(index, r.rep);
      if (idx >= 0) {
        h = v_scale(h, __ldg(p.norms + idx));
        const int64_t xi = xslot ? (int64_t)__ldg(xslot + idx) : idx;
        const V val = v_mul(h, to_v(load_x<CE>(p.x, xi), (V *)nullptr));
        smem_add(acc_s + src, val);
      } else if (v_nonzero(h)) {
        bool fatal = true;
        if (!orbit.trivial_characters)
          fatal = orbit_stabiliser_sum<FS>(orbit, r.rep) > 1e-12 * (double)orbit.group_order;
        if (fatal && atomicAdd(p.status, 1ull) == 0) p.status[1] = r.rep;
      }
    }
  };

  const int64_t n_rows = p.row_end - p.row_begin;
  const int64_t n_tiles = (n_rows + 31) / 32;
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += warps_total) {
    const int64_t i = p.row_begin + tile * 32 + lane;
    const bool valid = i < p.row_end;
    const uint64_t b = valid ? __ldg(row_states + i) : 0ull;
    V acc = v_make(0.0, 0.0, (V *)nullptr);
    double inv_nb = 1.0;
    if (PROJ == PROJ_GROUP && valid) inv_nb = 1.0 / __ldg(row_norms + i);

    for (int g0 = 0, w = 0; g0 < p.n_groups; g0 += 64, ++w) {
      const int g1 = min(g0 + 64, p.n_groups);
      RowTerms rt = row_terms<CV>(T, w, g0, g1, b);
      if (!valid) rt.mask = 0;
      if (PROJ != PROJ_GROUP) {
        // every lane walks the set bits of ITS row: no lane idles on a bond that does not emit
        while (rt.mask) {
          uint64_t flip;
          V h = pop_term<CV>(T, rt, g0, b, any_s_out, flip);
          uint64_t a = b ^ flip;
          bool flipped = false;
          if (PROJ == PROJ_INVERSION) {
            const uint64_t inv = a ^ p.site_mask;
            flipped = inv < a;
            if (flipped) h = v_scale(h, p.inversion_character);
          }
          int64_t idx;
          if (index.mode == INDEX_RANK) {
            // rank over the full fixed-weight set, incrementally from rank(b) = i
            const int lo = __ffsll((long long)flip) - 1;
            const int hi = 63 - __clzll((long long)flip);
            const uint64_t span = ((hi == 63) ? ~0ull : ((1ull << (hi + 1)) - 1)) & ~((1ull << lo) - 1);
            const uint64_t ob = b & span, nb = a & span;
            idx = -1;
            if ((a & ~index.site_mask) == 0 && __popcll(ob) == __popcll(nb)) {
              const int k0 = __popcll(b & ((1ull << lo) - 1));
              int64_t r = i - (int64_t)combinadic_sum(index.binom, index.stride, ob, k0) +
                          (int64_t)combinadic_sum(index.binom, index.stride, nb, k0);
              if (flipped) r = (int64_t)p.rank_total - 1 - r;   // complement reverses the order
              if (r >= 0 && r < index.n) idx = r;
            }
          } else {
            idx = locate(index, flipped ? (a ^ p.site_mask) : a);
          }
          if (idx >= 0) {
            const int64_t xi = xslot ? (int64_t)__ldg(xslot + idx) : idx;
            v_add(acc, v_mul(h, to_v(load_x<CE>(p.x, xi), (V *)nullptr)));
          } else if (v_nonzero(h) && atomicAdd(p.status, 1ull) == 0) {
            p.status[1] = a;
          }
        }
      } else {
        for (;;) {
          const bool has = rt.mask != 0;
          const unsigned m = __ballot_sync(0xffffffffu, has);
          if (m == 0) break;
          if (has) {
            uint64_t flip;
            const V c = pop_term<CV>(T, rt, g0, b, any_s_out, flip);
            const unsigned pos = (head + count + __popc(m & ((1u << lane) - 1u))) & (kQueue - 1);
            qb[pos] = b ^ flip;
            qc[pos] = v_scale(c, inv_nb);
            ql[pos] = (unsigned char)lane;
          }
          count += __popc(m);
          if (count >= 32) {
            __syncwarp();
            drain(32);
            head = (head + 32) & (kQueue - 1);
            count -= 32;
            __syncwarp();
          }
        }
      }
    }
    if (PROJ == PROJ_GROUP) {
      if (count > 0) {
        __syncwarp();
        drain(count);
        head = (head + count) & (kQueue - 1);
        count = 0;
      }
      __syncwarp();
      acc = acc_s[lane];
      acc_s[lane] = v_make(0.0, 0.0, (V *)nullptr);
      __syncwarp();
    }
    if (valid) {
      // diagonal (DMV:36-53) and the single store of y[i]; without diagonal terms y is accumulated into
      E out;
      if (p.n_diag > 0) {
        double dre, dim;
        diagonal<CV>(T, p.n_diag, b, dre, dim);
        const E xi = load_x<CE>(p.x, p.x_row_offset + i);
        if (CE) out = v_make(dre * v_re(xi) - dim * v_im(xi), dre * v_im(xi) + dim * v_re(xi), (E *)nullptr);
        else out = v_make(dre * v_re(xi), 0.0, (E *)nullptr);
      } else {
        out = reinterpret_cast<const E *>(p.y)[i];
      }
      out = v_make(v_re(out) + v_re(acc), v_im(out) + v_im(acc), (E *)nullptr);
      reinterpret_cast<E *>(p.y)[i] = out;
    }
  }
}

// -------------------------------------------------------------------------------------------------
// k_rows: the row traversal for bases with permutation symmetries, real operators with a bit-parallel emit test and
// trivial characters (every symmetric model input of the reference) -- the product kernel of one rank and of the
// replicated-x form on several ranks.
//   y[b] = D(b) x[b] + 1/n_b sum_t h_t(b) (n x)[rep(b ^ x_t)]
// One lane owns one row and walks ITS emitting groups: no warp queue, no shared-memory atomics, y written once.  Per term:
// orbit minimum in registers (canonical form, dmv_device.cuh), then ONE dependent memory access -- the slot of the
// representative in a hash table that carries the scaled vector element (table_slot) -- and that access is software
// pipelined: the slot of term j is requested right after its orbit minimum and consumed after the orbit minimum of
// term j + 2, so its latency hides behind ~10^3 integer instructions of the same lane.  (Deeper pipelines -- four requests per
// lane through prefetch.global.L2 or through cp.async into shared memory -- were slower: the look-ups are bound by the
// rate of random requests the memory system takes, not by their latency.)
// -------------------------------------------------------------------------------------------------
// one bucket = two slots (layout: table_slot in dmv_device.cuh); a bucket is one 32-byte sector, read as two independent
// 128-bit loads (the widest global load sm_90 has; both halves of the sector are in flight together), not allocated in
// L1: a bucket is touched once per product, and gigabytes of them streaming through L1 would evict the small tables the
// orbit minimum reads from global memory
__device__ __forceinline__ void load256(const unsigned char *q, uint64_t &a, uint64_t &b, uint64_t &c, uint64_t &d) {
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(q));
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2+16];" : "=l"(c), "=l"(d) : "l"(q));
}
// the same through L1 (perfect-hash blocks: a few bits per state, read by every look-up)
__device__ __forceinline__ void load256_cached(const unsigned char *q, uint64_t &a, uint64_t &b, uint64_t &c, uint64_t &d) {
  asm volatile("ld.global.nc.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(q));
  asm volatile("ld.global.nc.v2.u64 {%0, %1}, [%2+16];" : "=l"(c), "=l"(d) : "l"(q));
}
// one 32-byte sector written whole by one thread (two 128-bit stores): a full-sector write needs no read-modify-write
__device__ __forceinline__ void store256(unsigned char *q, uint64_t a, uint64_t b, uint64_t c, uint64_t d) {
  asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(q), "l"(a), "l"(b) : "memory");
  asm volatile("st.global.v2.u64 [%0+16], {%1, %2};" ::"l"(q), "l"(c), "l"(d) : "memory");
}
// L2 eviction priority of single accesses (the ordered table of k_rows, option rows_l2): a policy is made once per
// thread and handed to each load or store.  It travels in a uniform register, so it is one value per warp and
// instruction: lanes that want different policies for the same access branch to different instructions.
enum L2Evict { L2_NORMAL = 0, L2_FIRST = 1, L2_LAST = 2 };
__device__ __forceinline__ uint64_t l2_policy(int evict) {
  uint64_t policy;
  if (evict == L2_FIRST) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  else if (evict == L2_LAST) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(policy));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(policy));
  return policy;
}
__device__ __forceinline__ void load256_hint(const unsigned char *q, uint64_t policy, uint64_t &a, uint64_t &b, uint64_t &c,
                                             uint64_t &d) {
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;"
               : "=l"(a), "=l"(b) : "l"(q), "l"(policy));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2+16], %3;"
               : "=l"(c), "=l"(d) : "l"(q), "l"(policy));
}
// 8 or 16 bytes that are read or written once per product (a row's state, norm, x and y)
__device__ __forceinline__ uint64_t load64_hint(const void *q, uint64_t policy) {
  uint64_t a;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(a) : "l"(q), "l"(policy));
  return a;
}
__device__ __forceinline__ double load_hint(const double *q, uint64_t policy) {
  return __longlong_as_double((long long)load64_hint(q, policy));
}
__device__ __forceinline__ double2 load_hint(const double2 *q, uint64_t policy) {
  uint64_t a, b;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;"
               : "=l"(a), "=l"(b) : "l"(q), "l"(policy));
  return make_double2(__longlong_as_double((long long)a), __longlong_as_double((long long)b));
}
__device__ __forceinline__ void store_hint(double *q, double v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(q), "d"(v), "l"(policy) : "memory");
}
__device__ __forceinline__ void store_hint(double2 *q, double2 v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(q), "d"(v.x), "d"(v.y), "l"(policy) : "memory");
}
// HINT: through load256_hint with `policy`
template <bool CE, bool HINT = false>
__device__ __forceinline__ void bucket_load(const unsigned char *__restrict__ table, uint32_t b, ulonglong2 &keys,
                                            typename ValT<CE>::type &v0, typename ValT<CE>::type &v1,
                                            uint64_t policy = 0) {
  uint64_t w0, w1, w2, w3;
  // one bucket = one 32-byte sector = one request
  if constexpr (HINT) load256_hint(table + (size_t)b * 32, policy, w0, w1, w2, w3);
  else load256(table + (size_t)b * 32, w0, w1, w2, w3);
  if constexpr (CE) {   // { key, spare, re, im }
    keys = make_ulonglong2(w0, w1);                  // (one slot: the second word is spare)
    v0 = make_double2(__longlong_as_double((long long)w2), __longlong_as_double((long long)w3));
    v1 = v0;
  } else {              // { key0, key1, value0, value1 }
    keys = make_ulonglong2(w0, w1);
    v0 = __longlong_as_double((long long)w2);
    v1 = __longlong_as_double((long long)w3);
  }
}
// slot s of the dense tables (perfect hash, dense ordered): complex128 { key, spare, re, im }, float64 { key, value }
template <bool CE, bool HINT = false>
__device__ __forceinline__ void slot_load(const unsigned char *__restrict__ dense, uint32_t s, uint64_t &key,
                                          typename ValT<CE>::type &v, uint64_t policy = 0) {
  uint64_t a, b;
  if constexpr (CE) {
    uint64_t c, d;
    if constexpr (HINT) load256_hint(dense + (size_t)s * 32, policy, a, b, c, d);
    else load256(dense + (size_t)s * 32, a, b, c, d);
    key = a;
    v = make_double2(__longlong_as_double((long long)c), __longlong_as_double((long long)d));
  } else {
    const unsigned char *q = dense + (size_t)s * 16;
    if constexpr (HINT) {
      asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;"
                   : "=l"(a), "=l"(b) : "l"(q), "l"(policy));
    } else {
      const ulonglong2 t = __ldg(reinterpret_cast<const ulonglong2 *>(q));
      a = t.x; b = t.y;
    }
    key = a;
    v = __longlong_as_double((long long)b);
  }
}
__device__ __forceinline__ void axpy(double &acc, double c, double v) { acc = fma(c, v, acc); }
__device__ __forceinline__ void axpy(double2 &acc, double c, double2 v) { acc.x = fma(c, v.x, acc.x); acc.y = fma(c, v.y, acc.y); }

// k_rows keeps two tables behind the staged ones: the directory of the ordered table (ORD) and, for the square-torus
// form (TK > 0), the transposed flip mask of every group (torus_sq_columns), one 64-bit word per group
struct RowsSmem { size_t dir, gxt, total; };
__host__ __device__ inline RowsSmem rows_smem(const KernelParams &p, const SmemLayout &L, bool ord, int tk) {
  RowsSmem R;
  size_t off = align_up(L.total, 16);
  R.dir = off;
  if (ord) off += 4 * ((size_t)p.table_dir.last + 2);
  off = align_up(off, 8);
  R.gxt = off;
  if (tk > 0) off += 8 * (size_t)p.n_groups;
  R.total = (ord || tk > 0) ? off : L.total;
  return R;
}

// CTAS resident CTAs per SM (see launch_rows): the pipeline state must stay in registers (a spilled request waits for its
// load at once); within that, more warps per scheduler hide more of the latency the lane's pipeline leaves
// ORD: ordered table layout (see ordered_block); its directory is staged into shared memory behind the other tables, so
// a home costs two shared-memory reads and adds no dependent global access to the pipeline
// DORD (with ORD): the dense ordered table (see DenseOrder); request 0 is the rank block, request 1 the slot
template <bool CE, int TK, bool MPH, int CTAS, bool ORD, bool DORD = false>
__global__ void __launch_bounds__(kThreads, CTAS) k_rows(const KernelParams p) {
  using E = typename ValT<CE>::type;
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ_GROUP, sizeof(double), false);
  const Tables<false> T = stage_tables<PROJ_GROUP, false>(p, smem, L);   // p.groups / p.lut: row-traversal tables
  const RowsSmem RS = rows_smem(p, L, ORD, TK);
  uint32_t *sdir = reinterpret_cast<uint32_t *>(smem + RS.dir);
  if constexpr (ORD) stage(sdir, p.table_dir.dir, (int)p.table_dir.last + 2);
  uint64_t *sgxt = reinterpret_cast<uint64_t *>(smem + RS.gxt);
  if constexpr (TK > 0)
    for (int i = threadIdx.x; i < p.n_groups; i += blockDim.x) sgxt[i] = torus_sq_columns<TK>(p.groups[i].x);
  __syncthreads();
  const OrbitProgram &orbit = T.orbit;
  if constexpr (TK > 0) {
    // stage_tables has put the pair and row tables of the square-torus form in shared memory: say so, and the look-ups
    // of orbit_min_torus_sq compile to LDS instead of generic loads that resolve their address space at run time
    __builtin_assume(__isShared(orbit.tor_lutm));
    __builtin_assume(__isShared(orbit.tor_frow));
  }
  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  const bool any_s_out = p.any_s_out != 0;
  const unsigned char *__restrict__ table = reinterpret_cast<const unsigned char *>(p.table);
  const uint32_t n_buckets = p.table_slots;
  const uint64_t *__restrict__ row_states = p.row_states ? p.row_states : p.index.reps;
  const double *__restrict__ row_norms = p.row_norms ? p.row_norms : p.norms;
  unsigned long long bad = 0, bad_state = 0;
  const E zero = v_make(0.0, 0.0, (E *)nullptr);
  const PerfectHash H = p.mph;
  const unsigned char *__restrict__ dense = reinterpret_cast<const unsigned char *>(p.dense);
  // ORD, p.rows_l2: the buckets within p.rows_l2_window of the row's own place in the table are the ones the rows in
  // flight share (near), every other bucket is read once while they pass (far), and so is what belongs to the row alone
  const uint64_t far_policy = l2_policy(ORD && p.rows_l2 >= 1 ? L2_FIRST : L2_NORMAL);
  const uint64_t near_policy = l2_policy(ORD && p.rows_l2 == 2 ? L2_LAST : L2_NORMAL);

  const int64_t n_rows = p.row_end - p.row_begin;
  const int64_t n_tiles = (n_rows + 31) / 32;
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += warps_total) {
    const int64_t i = p.row_begin + tile * 32 + lane;
    const bool valid = i < p.row_end;
    uint64_t b = 0;
    if (valid) b = ORD ? load64_hint(row_states + i, far_policy) : __ldg(row_states + i);
    // near: near_lo <= bucket < near_lo + near_span.  A state of rank r lives in its block's buckets, and those lie
    // around buckets-per-state * r; rows that are a part of the table's basis (p.row_states) take their own home
    uint32_t near_lo = 0, near_span = 0;
    if constexpr (ORD) {
      uint32_t centre;
      if (p.row_states == nullptr) {
        centre = p.rows_l2_per_state * (uint32_t)i;
      } else {
        const uint32_t blk = ordered_block(b, p.table_dir.k_lo, p.table_dir.shift, p.table_dir.last);
        centre = ordered_slot(b, sdir[blk], sdir[blk + 1]);
      }
      near_lo = centre > p.rows_l2_window ? centre - p.rows_l2_window : 0u;
      near_span = centre - near_lo + p.rows_l2_window;
    }
    const uint64_t bt = TK > 0 ? torus_sq_columns<TK>(b) : 0ull;   // the row's transposed state: see orbit_min_torus_sq_t
    E acc = zero;
    int w = 0;
    RowTerms rt = row_terms<false>(T, 0, 0, min(64, p.n_groups), b);
    if (!valid) rt.mask = 0;
    if constexpr (DORD) {
      // ---- dense ordered table: request 0 holds the rank block of its state, request 1 a slot of the dense table (the
      // state's own, or the next of its rank block's leftovers)
      static_assert(ORD, "the dense ordered table uses the ordered directory");
      const DenseOrder DO = p.dord;
      bool live0 = false, live1 = false;
      uint64_t want0 = 0, want1 = 0;
      double c0 = 0.0, c1 = 0.0;
      uint32_t bits0 = 0, s1 = 0, end1 = 0;
      uint64_t A0 = 0, A1 = 0, A2 = 0, A3 = 0, k1 = 0;
      E v1 = zero;
      auto request1 = [&]() {   // ask for slot s1
        if (p.rows_l2 == 0) slot_load<CE>(dense, s1, k1, v1);
        else if (s1 - near_lo < near_span) slot_load<CE, true>(dense, s1, k1, v1, near_policy);
        else slot_load<CE, true>(dense, s1, k1, v1, far_policy);
      };
      for (;;) {
        while (valid && rt.mask == 0 && 64 * (w + 1) < p.n_groups) {
          ++w;
          rt = row_terms<false>(T, w, 64 * w, min(64 * w + 64, p.n_groups), b);
        }
        const bool has = rt.mask != 0;
        if (!has && !live0 && !live1) break;
        // ---- consume request 1
        if (live1) {
          if (k1 == want1) {
            axpy(acc, c1, v1);
          } else if (s1 + 1 < end1) {   // a leftover of the rank block that is not this state: the next one; request 0
            ++s1;                       // and the row wait one trip
            request1();
            continue;
          } else if (c1 != 0.0) {       // the slot belongs to another state: not in the basis (DMV:115-118)
            ++bad; bad_state = want1;
          }
        }
        // ---- request 0 -> request 1: the slot from the rank block
        live1 = false;
        if (live0) {
          want1 = want0; c1 = c0;
          s1 = dord_slot(A0, A1, A2, A3, bits0, end1);
          if (s1 < end1) {
            request1();
            live1 = true;
          } else if (c1 != 0.0) {       // not placed and the rank block has no leftovers: not in the basis
            ++bad; bad_state = want1;
          }
        }
        // ---- a new request 0: the next term of the row
        live0 = has;
        if (has) {
          uint64_t flip;
          const uint64_t flip_t = TK > 0 ? sgxt[64 * w + __ffsll((long long)rt.mask) - 1] : 0ull;
          c0 = pop_term<false>(T, rt, 64 * w, b, any_s_out, flip);
          const uint64_t raw = b ^ flip;
          if constexpr (TK > 0) want0 = orbit_min_torus_sq_t<TK>(orbit, raw, bt ^ flip_t);
          else want0 = orbit_representative(orbit, raw);
          const uint64_t h = dord_hash(want0);
          const uint32_t blk = ordered_block(want0, p.table_dir.k_lo, p.table_dir.shift, p.table_dir.last);
          const uint32_t rb = dord_block(h, sdir[blk], sdir[blk + 1]);
#ifdef DMV_ROWS_ORBIT_ONLY   // measurement builds only: no look-up, wrong results on purpose (minimum and rank block stay live)
          axpy(acc, c0, v_make((double)(rb & 7u), 0.0, (E *)nullptr));
          live0 = false;
          continue;
#endif
          const unsigned char *q = reinterpret_cast<const unsigned char *>(DO.blocks) + (size_t)rb * 32;
          bits0 = dord_bits(h);
          if (p.rows_l2 == 0) load256(q, A0, A1, A2, A3);
          else load256_hint(q, near_policy, A0, A1, A2, A3);
        }
      }
    } else if constexpr (MPH) {
      // ---- dense index: request 0 holds the two perfect-hash blocks of its state (L2 hits), request 1 the slot of
      // the dense table (or, for the few states the two levels could not place, a bucket of the open-addressing table)
      bool live0 = false, live1 = false, in_table1 = false;
      uint64_t want0 = 0, want1 = 0;
      double c0 = 0.0, c1 = 0.0;
      uint32_t bits0 = 0, b1 = 0;
      uint64_t A0 = 0, A1 = 0, A2 = 0, A3 = 0, B0 = 0, B1 = 0, B2 = 0, B3 = 0;
      ulonglong2 k1 = make_ulonglong2(0, 0);
      E v10 = zero, v11 = zero;
      for (;;) {
        while (valid && rt.mask == 0 && 64 * (w + 1) < p.n_groups) {
          ++w;
          rt = row_terms<false>(T, w, 64 * w, min(64 * w + 64, p.n_groups), b);
        }
        const bool has = rt.mask != 0;
        if (!has && !live0 && !live1) break;
        // ---- consume request 1
        bool retry = false;
        if (live1) {
          if (!in_table1) {
            if (k1.x == want1) axpy(acc, c1, v10);
            else if (c1 != 0.0) { ++bad; bad_state = want1; }   // the slot belongs to another state: not in the basis
          } else {
            const bool hit0 = k1.x == want1, hit1 = !CE && k1.y == want1;
            if (hit0 | hit1) axpy(acc, c1, hit0 ? v10 : v11);
            else if (k1.x == kEmptyKey || (!CE && k1.y == kEmptyKey)) { if (c1 != 0.0) { ++bad; bad_state = want1; } }
            else retry = true;
          }
        }
        if (retry) {   // next bucket of the open-addressing table; request 0 and the row wait one trip
          b1 = b1 + 1 == n_buckets ? 0 : b1 + 1;
          bucket_load<CE>(table, b1, k1, v10, v11);
          continue;
        }
        // ---- request 0 -> request 1: resolve the slot, ask for it
        live1 = live0;
        if (live0) {
          want1 = want0; c1 = c0;
          uint32_t slot = mph_rank(A0, A1, A2, A3, bits0 & 0xffu);
          if (slot == kMphMissing && H.n_blocks1 != 0) slot = mph_rank(B0, B1, B2, B3, bits0 >> 8);
          in_table1 = slot == kMphMissing;
          if (!in_table1) {
            if constexpr (CE) {
              uint64_t u0, u1, u2, u3;
              load256(dense + (size_t)slot * 32, u0, u1, u2, u3);
              k1 = make_ulonglong2(u0, u1);
              v10 = make_double2(__longlong_as_double((long long)u2), __longlong_as_double((long long)u3));
            } else {
              const ulonglong2 t = __ldg(reinterpret_cast<const ulonglong2 *>(dense + (size_t)slot * 16));
              k1 = make_ulonglong2(t.x, 0);
              v10 = __longlong_as_double((long long)t.y);
            }
          } else {
            b1 = table_slot(want1, n_buckets);
            bucket_load<CE>(table, b1, k1, v10, v11);
          }
        }
        // ---- a new request 0: the next term of the row
        live0 = has;
        if (has) {
          uint64_t flip;
          const uint64_t flip_t = TK > 0 ? sgxt[64 * w + __ffsll((long long)rt.mask) - 1] : 0ull;
          c0 = pop_term<false>(T, rt, 64 * w, b, any_s_out, flip);
          const uint64_t raw = b ^ flip;
          if constexpr (TK > 0) want0 = orbit_min_torus_sq_t<TK>(orbit, raw, bt ^ flip_t);
          else want0 = orbit_representative(orbit, raw);
          uint32_t blk, bit, blk1 = 0, bit1 = 0;
          mph_position(want0, 0, H.n_blocks0, blk, bit);
          load256_cached(H.blocks + (size_t)blk * 32, A0, A1, A2, A3);
          if (H.n_blocks1 != 0) {
            mph_position(want0, 1, H.n_blocks1, blk1, bit1);
            load256_cached(H.blocks + ((size_t)H.n_blocks0 + blk1) * 32, B0, B1, B2, B3);
          }
          bits0 = bit | (bit1 << 8);
        }
      }
    } else {
    // two requests in flight per lane: wanted key, coefficient, bucket, and what the bucket held
    bool live0 = false, live1 = false;
    uint64_t want0 = 0, want1 = 0;
    double c0 = 0.0, c1 = 0.0;
    uint32_t b0 = 0, b1 = 0;
    ulonglong2 k0 = make_ulonglong2(0, 0), k1 = k0;
    E v00 = zero, v01 = zero, v10 = zero, v11 = zero;
    auto request = [&]() {   // ask for bucket b0
      if (!ORD || p.rows_l2 == 0) bucket_load<CE>(table, b0, k0, v00, v01);
      else if (b0 - near_lo < near_span) bucket_load<CE, true>(table, b0, k0, v00, v01, near_policy);
      else bucket_load<CE, true>(table, b0, k0, v00, v01, far_policy);
    };
    for (;;) {
      while (valid && rt.mask == 0 && 64 * (w + 1) < p.n_groups) {
        ++w;
        rt = row_terms<false>(T, w, 64 * w, min(64 * w + 64, p.n_groups), b);
      }
      const bool has = rt.mask != 0;
      if (!has && !live0 && !live1) break;
      // ---- consume the older request
      bool retry = false;
      if (live1) {
        const bool hit0 = k1.x == want1, hit1 = !CE && k1.y == want1;
        if (hit0 | hit1) {
          axpy(acc, c1, hit0 ? v10 : v11);
        } else if (k1.x == kEmptyKey || (!CE && k1.y == kEmptyKey)) {   // a free slot in the bucket: not a basis state
          if (c1 != 0.0) { ++bad; bad_state = want1; }         // DMV:115-118
        } else {
          retry = true;                                        // both slots taken by other states: next bucket
        }
      }
      const uint64_t want_r = want1;
      const double c_r = c1;
      const uint32_t b_r = b1 + 1 == n_buckets ? 0 : b1 + 1;
      live1 = live0; want1 = want0; c1 = c0; b1 = b0; k1 = k0; v10 = v00; v11 = v01;
      // ---- issue a new request: the continuation of a missed one, else the next term of the row
      if (retry) {
        want0 = want_r; c0 = c_r; b0 = b_r;
        request();
        live0 = true;
      } else if (has) {
        uint64_t flip;
        const uint64_t flip_t = TK > 0 ? sgxt[64 * w + __ffsll((long long)rt.mask) - 1] : 0ull;
        c0 = pop_term<false>(T, rt, 64 * w, b, any_s_out, flip);
        const uint64_t raw = b ^ flip;
        if constexpr (TK > 0) want0 = orbit_min_torus_sq_t<TK>(orbit, raw, bt ^ flip_t);
        else want0 = orbit_representative(orbit, raw);
        if constexpr (ORD) {
          const uint32_t blk = ordered_block(want0, p.table_dir.k_lo, p.table_dir.shift, p.table_dir.last);
          b0 = ordered_slot(want0, sdir[blk], sdir[blk + 1]);
        } else {
          b0 = table_slot(want0, n_buckets);
        }
#ifdef DMV_ROWS_ORBIT_ONLY   // measurement builds only: no look-up, wrong results on purpose (the minimum and the bucket stay live)
        k0 = make_ulonglong2(want0, want0);
        v00 = v01 = v_make((double)(b0 & 7u), 0.0, (E *)nullptr);
#else
        request();
#endif
        live0 = true;
      } else {
        live0 = false;
      }
    }
    }
    if (valid) {
      const double inv_nb = 1.0 / (ORD ? load_hint(row_norms + i, far_policy) : __ldg(row_norms + i));
      E out;
      if (p.n_diag > 0) {
        double dre, dim;
        diagonal<false>(T, p.n_diag, b, dre, dim);
        E xi;
        if constexpr (ORD) xi = load_hint(reinterpret_cast<const E *>(p.x) + p.x_row_offset + i, far_policy);
        else xi = load_x<CE>(p.x, p.x_row_offset + i);
        out = v_scale(xi, dre);   // real operator: the diagonal is real
      } else {
        out = reinterpret_cast<const E *>(p.y)[i];
      }
      axpy(out, inv_nb, acc);
      if constexpr (ORD) store_hint(reinterpret_cast<E *>(p.y) + i, out, far_policy);
      else reinterpret_cast<E *>(p.y)[i] = out;
    }
  }
  if (bad) {
    if (atomicAdd(p.status, bad) == 0) p.status[1] = bad_state;
  }
}

// -------------------------------------------------------------------------------------------------
// The term store (RowsStoreView in dmv_host.h, built by dmv_store.cu).  Every term's target and coefficient depend on the
// basis and the operator only, so they are found once: k_store_build walks the rows exactly as k_rows does (row_terms,
// pop_term, the same orbit minimum) and finds each target's index in the sorted basis with `locate`.  The count pass
// counts the entries of every (column block, row), evaluates the row's diagonal and reports what the store cannot hold;
// the write pass puts each entry at its place.  k_rows_stored then needs no orbit minimum and no look-up: a pass over
// adjacent column blocks gathers (n x) from the compact scaled x of those blocks only, which stays in L2 while the
// pass runs, in place of one random HBM sector per term.
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t warp_exclusive_sum(uint32_t v, unsigned lane) {
  uint32_t s = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, s, d);
    if (lane >= (unsigned)d) s += t;
  }
  return s - v;
}

template <int TK, bool WRITE>
__global__ void __launch_bounds__(kThreads) k_store_build(const KernelParams p, const RowsStoreView s,
                                                          unsigned long long *flags) {
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ_GROUP, sizeof(double), false);
  const Tables<false> T = stage_tables<PROJ_GROUP, false>(p, smem, L);
  const RowsSmem RS = rows_smem(p, L, false, TK);
  uint64_t *sgxt = reinterpret_cast<uint64_t *>(smem + RS.gxt);
  if constexpr (TK > 0)
    for (int i = threadIdx.x; i < p.n_groups; i += blockDim.x) sgxt[i] = torus_sq_columns<TK>(p.groups[i].x);
  __syncthreads();
  const OrbitProgram &orbit = T.orbit;
  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  const bool any_s_out = p.any_s_out != 0;
  const uint64_t *__restrict__ row_states = p.row_states ? p.row_states : p.index.reps;
  unsigned long long bad = 0, over = 0, uncoded = 0;
  uint64_t cursor[WRITE ? kStoreMaxChunks : 1];   // write pass: next entry of the row in every block
  uint32_t count[WRITE ? 1 : kStoreMaxChunks];    // count pass: entries of the row in every block
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < s.n_tiles; tile += warps_total) {
    const int64_t i = tile * 32 + lane;
    const bool valid = i < s.n_rows;
    for (int k = 0; k < s.chunks; ++k) {
      if constexpr (WRITE) {
        const uint32_t c = valid ? s.counts[k * s.n_rows + i] : 0u;
        cursor[k] = s.tile_off[k * s.n_tiles + tile] + warp_exclusive_sum(c, lane);
      } else {
        count[k] = 0;
      }
    }
    const uint64_t b = valid ? row_states[i] : 0ull;
    const uint64_t bt = TK > 0 ? torus_sq_columns<TK>(b) : 0ull;
    int w = 0;
    RowTerms rt = row_terms<false>(T, 0, 0, min(64, p.n_groups), b);
    if (!valid) rt.mask = 0;
    for (;;) {
      while (valid && rt.mask == 0 && 64 * (w + 1) < p.n_groups) {
        ++w;
        rt = row_terms<false>(T, w, 64 * w, min(64 * w + 64, p.n_groups), b);
      }
      if (rt.mask == 0) break;
      uint64_t flip;
      const uint64_t flip_t = TK > 0 ? sgxt[64 * w + __ffsll((long long)rt.mask) - 1] : 0ull;
      const double c = pop_term<false>(T, rt, 64 * w, b, any_s_out, flip);
      const uint64_t raw = b ^ flip;
      uint64_t want;
      if constexpr (TK > 0) want = orbit_min_torus_sq_t<TK>(orbit, raw, bt ^ flip_t);
      else want = orbit_representative(orbit, raw);
      const int64_t idx = locate(p.index, want);
      if (idx < 0) {   // not in the basis: k_rows skips it when c = 0 and reports it otherwise (DMV:115-118)
        if (c != 0.0) ++bad;
        continue;
      }
      const int k = (int)(idx / s.block_states);
      int code = 0;
      while (code < kStoreCodes && __double_as_longlong(s.coef[code]) != __double_as_longlong(c)) ++code;
      if constexpr (WRITE) {
        s.entries[cursor[k]++] = (uint32_t)(idx - (int64_t)k * s.block_states) | ((uint32_t)code << kStoreIndexBits);
      } else {
        if (code == kStoreCodes) ++uncoded;
        ++count[k];
      }
    }
    if constexpr (!WRITE) {
      if (valid) {
        for (int k = 0; k < s.chunks; ++k) {
          if (count[k] > 255u) ++over;
          s.counts[k * s.n_rows + i] = (uint8_t)min(count[k], 255u);
        }
        if (s.diag) {
          double dre, dim;
          diagonal<false>(T, p.n_diag, b, dre, dim);
          s.diag[i] = dre;
        }
      }
    }
  }
  if (bad) atomicAdd(flags, bad);
  if (over) atomicAdd(flags + 1, over);
  if (uncoded) atomicAdd(flags + 2, uncoded);
}

// per tile and block: the sum of its 32 rows' counts
__global__ void k_store_tile_sums(const RowsStoreView s) {
  const int64_t total = s.n_tiles * s.chunks;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int64_t k = q / s.n_tiles, t = q - k * s.n_tiles;
    const uint8_t *c = s.counts + k * s.n_rows + t * 32;
    const int64_t rows = min((int64_t)32, s.n_rows - t * 32);
    uint64_t sum = 0;
    for (int64_t r = 0; r < rows; ++r) sum += c[r];
    s.tile_off[q] = sum;
  }
}

// exclusive prefix sum of a[0, n) in place, a[n] = the total: one CTA, deterministic (once per basis)
__global__ void k_store_scan(uint64_t *a, int64_t n) {
  __shared__ uint64_t part[1024];
  const int64_t per = (n + blockDim.x - 1) / blockDim.x;
  const int64_t lo = min(n, (int64_t)threadIdx.x * per), hi = min(n, lo + per);
  uint64_t sum = 0;
  for (int64_t q = lo; q < hi; ++q) sum += a[q];
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t run = 0;
    for (unsigned t = 0; t < blockDim.x; ++t) { const uint64_t v = part[t]; part[t] = run; run += v; }
    a[n] = run;
  }
  __syncthreads();
  uint64_t run = part[threadIdx.x];
  for (int64_t q = lo; q < hi; ++q) { const uint64_t v = a[q]; a[q] = run; run += v; }
}

__device__ __forceinline__ uint32_t load_u8_hint(const uint8_t *q, uint64_t policy) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(q), "l"(policy));
  return v;
}
// an entry: the warp reads whole lines of a run (read once: not allocated in L1, evict_first in L2)
__device__ __forceinline__ uint32_t load_entry(const uint32_t *q, uint64_t policy) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(q), "l"(policy));
  return v;
}
// a gather from the current block of the compact x (an L2 hit): not allocated in L1
__device__ __forceinline__ double gather_x(const double *q) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(q));
  return v;
}
__device__ __forceinline__ double2 gather_x(const double2 *q) {
  double2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(q));
  return v;
}

// Entries of a tile's run that its warp gathers at once (kStoreWindow / 32 per lane), and the shared memory of their
// values and codes: one window per warp.
constexpr int kStoreWindow = 128;
template <bool CE>
constexpr size_t rows_stored_smem() {
  return (size_t)kWarps * kStoreWindow * (sizeof(typename ValT<CE>::type) + 1);
}

// One warp per tile of 32 rows, one lane per row for the sums, as k_rows.  In every block the tile's entries are one run
// in lane order (k_store_build).  The warp reads the run of its valid lanes in windows of kStoreWindow entries: lane l
// loads the entries at positions l, l + 32, ... of the window (one line per warp instruction), issues their gathers back
// to back and puts each value and code at its position in the warp's window, whichever row it belongs to.  Then each
// lane sums the part of its own row's range that lies in the window, in order.  So a row's sum runs over blocks
// k0 .. k1 - 1 and within each block in k_rows' term order, with k_rows' coefficients and (n x) products: over the whole
// basis at once (one block) y equals k_rows' bit for bit.  The entries, counts, row data and partial sums are read once
// per product (evict_first).
template <bool CE>
__global__ void __launch_bounds__(kThreads) k_rows_stored(const KernelParams p, const RowsStoreView s,
                                                          const typename ValT<CE>::type *__restrict__ xs,
                                                          typename ValT<CE>::type *partial, int k0, int k1) {
  using E = typename ValT<CE>::type;
  constexpr int kPer = kStoreWindow / 32;
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double scoef[kStoreCodes];
  if (threadIdx.x < kStoreCodes) scoef[threadIdx.x] = s.coef[threadIdx.x];
  __syncthreads();
  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  E *const sval = reinterpret_cast<E *>(smem) + warp * kStoreWindow;
  uint8_t *const scode = smem + kWarps * kStoreWindow * sizeof(E) + warp * kStoreWindow;
  const bool first = k0 == 0, last = k1 == s.chunks;
  const uint64_t stream = l2_policy(L2_FIRST);
  const double *__restrict__ row_norms = p.row_norms ? p.row_norms : p.norms;
  constexpr uint32_t kMask = (1u << kStoreIndexBits) - 1u;
  const E zero = v_make(0.0, 0.0, (E *)nullptr);
  const int64_t t0 = p.row_begin / 32, t1 = (p.row_end + 31) / 32;
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = t0 + (int64_t)blockIdx.x * kWarps + warp; tile < t1; tile += warps_total) {
    const int64_t i = tile * 32 + lane;
    const bool valid = i >= p.row_begin && i < p.row_end;
    // the valid lanes are contiguous: lane_lo .. lane_hi
    const int lane_lo = (int)max(p.row_begin - tile * 32, (int64_t)0);
    const int lane_hi = (int)min(p.row_end - tile * 32, (int64_t)32) - 1;
    E acc = zero;
#ifndef DMV_STORE_NO_PARTIAL   // measurement builds only: the partial sums neither read nor written, wrong results
    if (!first && valid) acc = load_hint(partial + i, stream);
#endif
    for (int k = k0; k < k1; ++k) {
      uint32_t cnt = i < s.n_rows ? load_u8_hint(s.counts + k * s.n_rows + i, stream) : 0u;
      const uint32_t excl = warp_exclusive_sum(cnt, lane);
      if (!valid) cnt = 0;
      // the run of the valid lanes, [run_lo, run_lo + run_n) from the tile's first entry in the block; this row's
      // entries are [lo, lo + cnt) of it
      const uint32_t run_lo = __shfl_sync(0xffffffffu, excl, lane_lo);
      const uint32_t run_n = __shfl_sync(0xffffffffu, excl + cnt, lane_hi) - run_lo;
      const uint32_t lo = valid ? excl - run_lo : 0u, hi = lo + cnt;
      const uint32_t *e = s.entries + load64_hint(s.tile_off + k * s.n_tiles + tile, stream) + run_lo;
#ifdef DMV_STORE_NO_GATHER   // measurement builds only: entries streamed, no gather, wrong results on purpose
      auto gather_x = [](const E *q) { return v_make((double)(((uintptr_t)q >> 4) & 7u), 0.0, (E *)nullptr); };
#endif
      const E *xb = xs + (int64_t)k * s.block_states;
      for (uint32_t w0 = 0; w0 < run_n; w0 += kStoreWindow) {
        uint32_t ent[kPer];
#pragma unroll
        for (int q = 0; q < kPer; ++q)
          ent[q] = w0 + lane + 32 * q < run_n ? load_entry(e + w0 + lane + 32 * q, stream) : 0u;
        E v[kPer];
#pragma unroll
        for (int q = 0; q < kPer; ++q)
          v[q] = w0 + lane + 32 * q < run_n ? gather_x(xb + (ent[q] & kMask)) : zero;
#pragma unroll
        for (int q = 0; q < kPer; ++q) {
          sval[lane + 32 * q] = v[q];
          scode[lane + 32 * q] = (uint8_t)(ent[q] >> kStoreIndexBits);
        }
        __syncwarp();
        const uint32_t end = min(hi, w0 + kStoreWindow);
        for (uint32_t j = max(lo, w0); j < end; ++j) axpy(acc, scoef[scode[j - w0]], sval[j - w0]);
        __syncwarp();
      }
    }
    if (!valid) continue;
    if (!last) {
#ifndef DMV_STORE_NO_PARTIAL
      store_hint(partial + i, acc, stream);
#endif
      continue;
    }
    // diagonal and the single store of y[i], as k_rows
    const double inv_nb = 1.0 / load_hint(row_norms + i, stream);
    E out;
    if (s.diag) out = v_scale(load_hint(reinterpret_cast<const E *>(p.x) + p.x_row_offset + i, stream), load_hint(s.diag + i, stream));
    else out = reinterpret_cast<const E *>(p.y)[i];
    axpy(out, inv_nb, acc);
    store_hint(reinterpret_cast<E *>(p.y) + i, out, stream);
  }
}

// -------------------------------------------------------------------------------------------------
// k_rows_batch: k_rows on up to six real (three complex) vectors at once -- the product the block eigensolver asks for
// (reference src/Diagonalize.chpl:134-162: PRIMME hands `blockSize` vectors to one matvec call).  The orbit minimum and the
// look-up of a term are shared by the vectors: one bucket = 64 bytes = { key, d[0..5], spare }, d = the scaled elements of
// the vectors at that state (three (re, im) pairs or six reals: the operator is real, so every double is treated alike),
// fetched as two 32-byte halves (load256 each).  One request per lane in flight, consumed after the orbit minimum of the
// NEXT term; a bucket taken by another state continues with the next bucket through the same slot.
// Cost model: one 64-byte request per term against one 32-byte request per term AND vector in k_rows.
// -------------------------------------------------------------------------------------------------
template <int TK, int CTAS>
__global__ void __launch_bounds__(kThreads, CTAS) k_rows_batch(const KernelParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ_GROUP, sizeof(double), false);
  const Tables<false> T = stage_tables<PROJ_GROUP, false>(p, smem, L);
  __syncthreads();
  const OrbitProgram &orbit = T.orbit;
  if constexpr (TK > 0) {
    // stage_tables has put the pair and row tables of the square-torus form in shared memory: say so, and the look-ups
    // of orbit_min_torus_sq compile to LDS instead of generic loads that resolve their address space at run time
    __builtin_assume(__isShared(orbit.tor_lutm));
    __builtin_assume(__isShared(orbit.tor_frow));
  }
  const unsigned lane = threadIdx.x & 31u;
  const unsigned warp = threadIdx.x >> 5;
  const bool any_s_out = p.any_s_out != 0;
  const unsigned char *__restrict__ table = reinterpret_cast<const unsigned char *>(p.table);
  const uint32_t n_buckets = p.table_slots;
  const int elt = p.batch_elt;            // doubles per vector element (1 | 2)
  const int nd = p.batch * elt;           // doubles per state in use (<= 6)
  const int64_t stride = p.batch_stride;  // elements between consecutive vectors
  const double *__restrict__ xd = reinterpret_cast<const double *>(p.x);
  double *__restrict__ yd = reinterpret_cast<double *>(p.y);
  unsigned long long bad = 0, bad_state = 0;

  const int64_t n_rows = p.row_end - p.row_begin;
  const int64_t n_tiles = (n_rows + 31) / 32;
  const int64_t warps_total = (int64_t)gridDim.x * kWarps;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += warps_total) {
    const int64_t i = p.row_begin + tile * 32 + lane;
    const bool valid = i < p.row_end;
    const uint64_t b = valid ? __ldg(p.index.reps + i) : 0ull;
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int w = 0;
    RowTerms rt = row_terms<false>(T, 0, 0, min(64, p.n_groups), b);
    if (!valid) rt.mask = 0;
    bool live = false, held = false;       // a request in flight; a term popped but not yet requested
    uint64_t want = 0, want_n = 0;
    double c = 0.0, c_n = 0.0;
    uint32_t bk = 0;
    uint64_t q0 = 0, q1 = 0, q2 = 0, q3 = 0, q4 = 0, q5 = 0, q6 = 0, q7 = 0;
    for (;;) {
      while (valid && rt.mask == 0 && 64 * (w + 1) < p.n_groups) {
        ++w;
        rt = row_terms<false>(T, w, 64 * w, min(64 * w + 64, p.n_groups), b);
      }
      const bool has = rt.mask != 0;
      if (!has && !live && !held) break;
      // ---- the next term of the row (its orbit minimum covers the latency of the request in flight)
      if (has && !held) {
        uint64_t flip;
        c_n = pop_term<false>(T, rt, 64 * w, b, any_s_out, flip);
        const uint64_t raw = b ^ flip;
        if constexpr (TK > 0) want_n = orbit_min_torus_sq<TK>(orbit, raw);
        else want_n = orbit_representative(orbit, raw);
        held = true;
      }
      // ---- consume the request in flight
      bool retry = false;
      if (live) {
        if (q0 == want) {
          acc[0] = fma(c, __longlong_as_double((long long)q1), acc[0]);
          acc[1] = fma(c, __longlong_as_double((long long)q2), acc[1]);
          acc[2] = fma(c, __longlong_as_double((long long)q3), acc[2]);
          acc[3] = fma(c, __longlong_as_double((long long)q4), acc[3]);
          acc[4] = fma(c, __longlong_as_double((long long)q5), acc[4]);
          acc[5] = fma(c, __longlong_as_double((long long)q6), acc[5]);
        } else if (q0 == kEmptyKey) {
          if (c != 0.0) { ++bad; bad_state = want; }       // not a basis state (DMV:115-118)
        } else {
          retry = true;
        }
      }
      // ---- issue: the continuation of a missed request, else the held term
      if (retry) {
        bk = bk + 1 == n_buckets ? 0 : bk + 1;
      } else if (held) {
        want = want_n; c = c_n; held = false;
        bk = table_slot(want, n_buckets);
        live = true;
      } else {
        live = false;
      }
      if (live) {
        const unsigned char *q = table + (size_t)bk * 64;
        load256(q, q0, q1, q2, q3);
        load256(q + 32, q4, q5, q6, q7);
      }
    }
    if (valid) {
      const double inv_nb = 1.0 / __ldg(p.norms + i);
      double dre = 0.0, dim = 0.0;
      if (p.n_diag > 0) diagonal<false>(T, p.n_diag, b, dre, dim);
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        if (j < nd) {
          const int64_t at = ((int64_t)(j / elt) * stride + i) * elt + (j % elt);
          const double base = p.n_diag > 0 ? dre * __ldg(xd + at) : yd[at];
          yd[at] = fma(inv_nb, acc[j], base);
        }
      }
    }
  }
  if (bad) {
    if (atomicAdd(p.status, bad) == 0) p.status[1] = bad_state;
  }
}

// hash table set-up: claim a slot per state (keys pre-set to kEmptyKey; slot 0 of a bucket, then slot 1 when the bucket
// has two, then the next bucket), remember it in slot_of (= 2 bucket + slot)
__global__ void k_table_insert(const uint64_t *__restrict__ reps, int64_t n, unsigned char *table, uint32_t n_buckets,
                               int slots_per_bucket, uint32_t *slot_of, int bucket_bytes, OrderedDir ord) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t key = reps[i];
  uint32_t b = table_home(key, n_buckets, ord);
  for (;;) {
    unsigned long long *q = reinterpret_cast<unsigned long long *>(table + (size_t)b * bucket_bytes);
    if (atomicCAS(q, (unsigned long long)kEmptyKey, (unsigned long long)key) == (unsigned long long)kEmptyKey) {
      slot_of[i] = 2 * b;
      return;
    }
    if (slots_per_bucket == 2 &&
        atomicCAS(q + 1, (unsigned long long)kEmptyKey, (unsigned long long)key) == (unsigned long long)kEmptyKey) {
      slot_of[i] = 2 * b + 1;
      return;
    }
    b = b + 1 == n_buckets ? 0 : b + 1;
  }
}

__global__ void k_ordered_dir(const uint64_t *__restrict__ reps, int64_t n, OrderedDir ord, uint32_t buckets_per_state,
                              uint32_t *dir) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p <= (int64_t)ord.last + 1) dir[p] = ordered_dir_entry(reps, n, ord, buckets_per_state, (uint32_t)p);
}

// per product: value of slot_of[i] = x[src(i)] * norm[i]   (src(i) = pos ? pos[i] : i).  complex128 rewrites the WHOLE
// 32-byte slot {key, spare, re, im} with store256: a full-sector write needs no read-modify-write in DRAM.
// slot_of[i] < 2^31: slot of the dense table (perfect hash); else 0x80000000 | slot of the open-addressing table.
template <bool CE>
__global__ void k_table_fill(int64_t n, const void *__restrict__ x, const double *__restrict__ norms,
                             const uint32_t *__restrict__ pos, const uint32_t *__restrict__ slot_of,
                             const uint64_t *__restrict__ reps, unsigned char *table, unsigned char *dense,
                             unsigned char *compact) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t src = pos ? (int64_t)__ldg(pos + i) : i;
    const double nrm = __ldg(norms + i);
    if (compact) {   // the term store's scaled x: the same products, in state order
      if constexpr (CE) {
        const double2 v = __ldg(reinterpret_cast<const double2 *>(x) + src);
        reinterpret_cast<double2 *>(compact)[i] = make_double2(v.x * nrm, v.y * nrm);
      } else {
        reinterpret_cast<double *>(compact)[i] = __ldg(reinterpret_cast<const double *>(x) + src) * nrm;
      }
      continue;
    }
    uint32_t s = __ldg(slot_of + i);
    const bool in_table = dense == nullptr || (s & 0x80000000u);
    s &= 0x7fffffffu;
    const uint64_t key = __ldg(reps + i);
    if constexpr (CE) {
      const double2 v = __ldg(reinterpret_cast<const double2 *>(x) + src);
      const uint64_t re = (uint64_t)__double_as_longlong(v.x * nrm), im = (uint64_t)__double_as_longlong(v.y * nrm);
      unsigned char *q = in_table ? table + (size_t)(s >> 1) * 32 : dense + (size_t)s * 32;
      store256(q, key, 0ull, re, im);
    } else {
      const double v = __ldg(reinterpret_cast<const double *>(x) + src) * nrm;
      if (in_table) *reinterpret_cast<double *>(table + (size_t)(s >> 1) * 32 + 16 + 8 * (s & 1)) = v;
      else *reinterpret_cast<ulonglong2 *>(dense + (size_t)s * 16) = make_ulonglong2(key, (uint64_t)__double_as_longlong(v));
    }
  }
}

// per batched product: bucket slot_of[i] / 2 of the 64-byte table <- { key, x_v[i] * norm[i] for the vectors v, 0 ... }
// (two store256 = two full sectors)
__global__ void k_table_fill_batch(int64_t n, int nd, int elt, const double *__restrict__ x, int64_t stride,
                                   const double *__restrict__ norms, const uint32_t *__restrict__ slot_of,
                                   const uint64_t *__restrict__ reps, unsigned char *table) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
    const double nrm = __ldg(norms + i);
    uint64_t d[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      double v = 0.0;
      if (j < nd) v = __ldg(x + ((int64_t)(j / elt) * stride + i) * elt + (j % elt)) * nrm;
      d[j] = (uint64_t)__double_as_longlong(v);
    }
    unsigned char *q = table + (size_t)(__ldg(slot_of + i) >> 1) * 64;
    const uint64_t key = __ldg(reps + i);
    store256(q, key, d[0], d[1], d[2]);
    store256(q + 32, d[3], d[4], d[5], 0ull);
  }
}

// ---- perfect-hash set-up (see PerfectHash in dmv_device.cuh) ----
__global__ void k_mph_mark(const uint64_t *__restrict__ keys, int64_t n, int level, uint32_t n_blocks,
                           unsigned long long *seen, unsigned long long *collide) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t block, bit;
  mph_position(keys[i], level, n_blocks, block, bit);
  const size_t w = (size_t)block * 3 + (bit >> 6);
  const unsigned long long m = 1ull << (bit & 63u);
  if (atomicOr(seen + w, m) & m) atomicOr(collide + w, m);
}
__global__ void k_mph_compact(const uint64_t *__restrict__ keys, int64_t n, int level, uint32_t n_blocks,
                              const unsigned long long *__restrict__ collide, uint64_t *next,
                              unsigned long long *next_count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t block, bit;
  mph_position(keys[i], level, n_blocks, block, bit);
  if ((collide[(size_t)block * 3 + (bit >> 6)] >> (bit & 63u)) & 1ull) next[atomicAdd(next_count, 1ull)] = keys[i];
}
__device__ __forceinline__ uint32_t mph_lookup(const PerfectHash &H, uint64_t key) {
  uint32_t block, bit;
  mph_position(key, 0, H.n_blocks0, block, bit);
  const unsigned long long *q = reinterpret_cast<const unsigned long long *>(H.blocks) + (size_t)block * 4;
  uint32_t r = mph_rank(q[0], q[1], q[2], q[3], bit);
  if (r != kMphMissing || H.n_blocks1 == 0) return r;
  mph_position(key, 1, H.n_blocks1, block, bit);
  q = reinterpret_cast<const unsigned long long *>(H.blocks) + ((size_t)H.n_blocks0 + block) * 4;
  return mph_rank(q[0], q[1], q[2], q[3], bit);
}
__global__ void k_mph_slots(const uint64_t *__restrict__ keys, int64_t n, PerfectHash H, const unsigned char *table,
                            uint32_t n_buckets, int slots_per_bucket, uint32_t *slot_of, unsigned long long *status) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t key = keys[i];
  const uint32_t r = mph_lookup(H, key);
  if (r != kMphMissing) { slot_of[i] = r; return; }
  uint32_t b = table_slot(key, n_buckets);
  for (uint32_t tries = 0; tries <= n_buckets; ++tries) {   // the state was inserted before: the probe sequence finds it
    const unsigned long long *q = reinterpret_cast<const unsigned long long *>(table + (size_t)b * 32);
    if (q[0] == key) { slot_of[i] = 0x80000000u | (2 * b); return; }
    if (slots_per_bucket == 2 && q[1] == key) { slot_of[i] = 0x80000000u | (2 * b + 1); return; }
    b = b + 1 == n_buckets ? 0 : b + 1;
  }
  atomicAdd(status + 2, 1ull);
}

// localProcess for records that arrived from other ranks: already projected and hashed by the sender.
// Two records per thread with their searches advanced in lock step (see locate2).
template <int PROJ, bool CV, bool CE, bool FS>
__global__ void __launch_bounds__(kThreads) k_accumulate(const KernelParams p, int64_t count,
                                                         const uint64_t *__restrict__ betas,
                                                         const double *__restrict__ coeffs) {
  using V = typename ValT<CV>::type;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t half = (count + 1) / 2;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < half; k += stride) {
    const int64_t k1 = k + half;
    const bool a1 = k1 < count;
    const uint64_t b0 = __ldg(betas + k), b1 = a1 ? __ldg(betas + k1) : 0ull;
    const V c0 = __ldg(reinterpret_cast<const V *>(coeffs) + k);
    const V c1 = a1 ? __ldg(reinterpret_cast<const V *>(coeffs) + k1) : v_make(0.0, 0.0, (V *)nullptr);
    int64_t i0, i1;
    locate2(p.index, true, b0, a1, b1, i0, i1);
    finish<PROJ, CV, CE, FS>(p, p.orbit, true, b0, c0, i0);
    finish<PROJ, CV, CE, FS>(p, p.orbit, a1, b1, c1, i1);
  }
}

// ls_chpl_operator_apply_diag / ls_chpl_operator_apply_off_diag (reference src/BatchedOperator.chpl:217-275):
// the term kernels applied to caller-given states with xs = nil ("times one", BO:230,263), no projection.
//   apply_diag:     coeffs[i] = Re sum_t v_t [alpha_i & m == r] (-1)^popc(alpha_i & s)
//   apply_off_diag: CSR by row -- pass 0 counts the emitting groups of every row, the host turns the counts into
//                   the row pointer `offsets`, pass 1 writes (beta, coefficient) of row i at offsets[i]...
// One lane per state; tables in shared memory as in k_generate.
__global__ void __launch_bounds__(kThreads) k_apply_diag(const KernelParams p, int64_t count,
                                                         const uint64_t *__restrict__ alphas, double *coeffs) {
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ_NONE, sizeof(double2));
  const Tables<true> T = stage_tables<PROJ_NONE, true>(p, smem, L);
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
    double dre, dim;
    diagonal<true>(T, p.n_diag, alphas[i], dre, dim);
    coeffs[i] = dre;
  }
}

template <bool WRITE>
__global__ void __launch_bounds__(kThreads) k_apply_off_diag(const KernelParams p, int64_t count,
                                                             const uint64_t *__restrict__ alphas,
                                                             const int64_t *__restrict__ offsets, int64_t *counts,
                                                             uint64_t *betas, double2 *coeffs) {
  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = smem_layout(p, PROJ_NONE, sizeof(double2));
  const Tables<true> T = stage_tables<PROJ_NONE, true>(p, smem, L);
  __syncthreads();
  const bool any_s_out = p.any_s_out != 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
    const uint64_t alpha = alphas[i];
    int64_t o = WRITE ? offsets[i] : 0;
    for (int g0 = 0, w = 0; g0 < p.n_groups; g0 += 64, ++w) {
      RowTerms rt = row_terms<true>(T, w, g0, min(g0 + 64, p.n_groups), alpha);
      if (!WRITE) { o += __popcll(rt.mask); continue; }
      while (rt.mask) {
        uint64_t flip;
        const double2 c = pop_term<true>(T, rt, g0, alpha, any_s_out, flip);
        betas[o] = alpha ^ flip;
        coeffs[o] = c;
        ++o;
      }
    }
    if (!WRITE) counts[i] = o;
  }
}

// dir[2b] = lower_bound(reps, b << shift), dir[2b+1] = lower_bound(reps, (b+1) << shift) for b in [0, n_buckets)
__global__ void k_build_directory(const uint64_t *__restrict__ reps, int64_t n, uint32_t *dir,
                                  uint64_t n_buckets, int shift) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n_buckets) return;
  const uint64_t b = (t >> 1) + (t & 1);
  int64_t lo = 0, hi = n;
  const bool past_end = shift > 0 ? (b > (~0ull >> shift)) : false;
  if (past_end) lo = n;
  const uint64_t key = b << shift;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (reps[mid] < key) lo = mid + 1; else hi = mid;
  }
  dir[t] = (uint32_t)lo;
}

__global__ void k_state_index(const StateIndex ix, int64_t count, const uint64_t *__restrict__ spins,
                              int64_t *indices) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) indices[k] = locate(ix, spins[k]);
}

__global__ void k_verify_rank(const StateIndex ix, unsigned long long *status) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < ix.n && locate(ix, ix.reps[k]) != k) atomicAdd(status, 1ull);
}

__global__ void k_locale_idx(int64_t count, const uint64_t *__restrict__ states, int num_ranks, uint8_t *keys) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) keys[k] = (uint8_t)locale_idx_of(states[k], num_ranks);
}

// ls_hs_state_info (reference src/FFI.chpl:181-184): representative, conj(character), norm
template <int PROJ, bool FS>
__global__ void k_state_info(const OrbitProgram P, uint64_t site_mask, double inv_char, int64_t count,
                             const uint64_t *__restrict__ alphas, uint64_t *betas, double2 *characters,
                             double *norms) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const uint64_t a = alphas[k];
  if (PROJ == PROJ_NONE) {
    betas[k] = a; characters[k] = make_double2(1.0, 0.0); norms[k] = 1.0;
  } else if (PROJ == PROJ_INVERSION) {
    const uint64_t inv = a ^ site_mask;
    const bool flip = inv < a;
    betas[k] = flip ? inv : a;
    characters[k] = make_double2(flip ? inv_char : 1.0, 0.0);
    norms[k] = sqrt(0.5);   // stabiliser = {identity}: |Stab| / |G| = 1/2
    if (inv == a) norms[k] = (inv_char > 0) ? 1.0 : 0.0;
  } else {
    const OrbitResult r = orbit_scan<true, false>(P, a);
    betas[k] = r.rep;
    double2 chi = make_double2(1.0, 0.0);
    double stab = (double)r.stab;
    if (!P.trivial_characters) {
      chi = P.characters[r.arg];
      if (FS) { const double sg = orbit_sign(P, r.arg, a); chi.x *= sg; chi.y *= sg; }
      stab = orbit_stabiliser_sum<FS>(P, a);
    }
    characters[k] = make_double2(chi.x, -chi.y);
    const double nn = stab / (double)P.group_order;
    norms[k] = nn > 1e-12 ? sqrt(nn) : 0.0;
  }
}

template <bool FS>
__global__ void k_compute_norms(const OrbitProgram P, int64_t count, const uint64_t *__restrict__ reps,
                                double *norms) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  double stab;
  if (P.trivial_characters) stab = (double)orbit_scan<true, false>(P, reps[k]).stab;
  else stab = orbit_stabiliser_sum<FS>(P, reps[k]);
  const double nn = stab / (double)P.group_order;
  norms[k] = nn > 1e-12 ? sqrt(nn) : 0.0;
}

// nextStateFixedHamming (reference src/StatesEnumeration.chpl:31-34)
__device__ __forceinline__ uint64_t next_state_fixed_hamming(uint64_t v) {
  const uint64_t t = v | (v - 1);
  return (t + 1) | (((~t & (t + 1)) - 1) >> (__ffsll((long long)v)));
}

// One thread per chunk of consecutive candidates [first, last]; keeps a candidate iff it is owned by
// this rank, is the minimum of its orbit and has non-zero norm (reference
// src/StatesEnumeration.chpl:158-224).  Pass 0 counts, pass 1 writes at chunk_offset[c].
// half_mask != 0 (spinful fermions): only candidates with popcount(v & half_mask) == half_weight are kept.
template <int PROJ, bool WRITE, bool FS>
__global__ void k_enumerate(const OrbitProgram P, uint64_t site_mask, bool fixed_hamming, uint64_t half_mask,
                            int half_weight, int rank, int num_ranks, int64_t n_chunks,
                            const uint64_t *__restrict__ chunk_first,
                            const uint64_t *__restrict__ chunk_last, unsigned long long *chunk_count,
                            const unsigned long long *__restrict__ chunk_offset, uint64_t *out,
                            double *out_norms) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  uint64_t v = chunk_first[c];
  const uint64_t last = chunk_last[c];
  unsigned long long n = 0;
  unsigned long long base = WRITE ? chunk_offset[c] : 0ull;
  for (;;) {
    bool keep = (half_mask == 0 || __popcll(v & half_mask) == half_weight) &&
                ((num_ranks <= 1) || (locale_idx_of(v, num_ranks) == rank));
    double norm = 1.0;
    if (keep) {
      if (PROJ == PROJ_INVERSION) {
        keep = v < (v ^ site_mask);
      } else if (PROJ == PROJ_GROUP) {
        const OrbitResult r = orbit_scan<true, true>(P, v);
        keep = (r.rep == v);
        if (keep) {
          const double stab = P.trivial_characters ? (double)r.stab : orbit_stabiliser_sum<FS>(P, v);
          const double nn = stab / (double)P.group_order;
          norm = nn > 1e-12 ? sqrt(nn) : 0.0;
          keep = norm > 0.0;
        }
      }
    }
    if (keep) {
      if (WRITE) { out[base + n] = v; if (out_norms) out_norms[base + n] = norm; }
      ++n;
    }
    if (v == last) break;
    v = fixed_hamming ? next_state_fixed_hamming(v) : v + 1;
  }
  if (!WRITE) chunk_count[c] = n;
}

// f(PROJ, CV, CE, FS) as integral constants for the value kinds k_generate, k_pull and k_accumulate are built for: real
// values and vectors, complex values with real or complex vectors; FS (the fermionic exchange sign) with PROJ_GROUP only
template <typename F>
void with_values(Projection proj, bool complex_values, bool complex_elements, const OrbitProgram &orbit, F &&f) {
  if (complex_elements && !complex_values) throw std::runtime_error("complex vectors need complex values");
  with_choice<PROJ_NONE, PROJ_INVERSION, PROJ_GROUP>(proj, [&](auto pj) {
    with_bool(complex_values, [&](auto cv) {
      with_bool(complex_elements, [&](auto ce) {
        with_bool(pj() == PROJ_GROUP && orbit.fermionic != 0, [&](auto fs) {
          if constexpr ((cv() || !ce()) && (pj() == PROJ_GROUP || !fs())) f(pj, cv, ce, fs);
        });
      });
    });
  });
}

}  // namespace

// lanes per source state: enough warps to fill the machine (>= 8 per SM) on small bases, never more than the
// number of flip-mask groups
int choose_row_split(int64_t rows, int n_groups) {
  const int n = sm_count();
  int s = 1;
  while (s < 32 && 2 * s <= n_groups && (rows * s) / 32 < (int64_t)n * 16) s *= 2;
  return s;
}

int planned_grid(int64_t rows, int row_split) {   // grid of the planned launches: fixed, not occupancy-derived
  const int rows_per_tile = 32 / (row_split > 1 ? row_split : 1);
  return capped_grid(((rows + rows_per_tile - 1) / rows_per_tile + kWarps - 1) / kWarps, (int64_t)sm_count() * 4);
}

// k_rows: CTAs per SM (rows_ctas) 2 (106-128 registers, nothing spills beyond a few words), 3 (80 registers) or 4 (64
// registers).  Auto (-1) runs three with the square-torus forms, whose three-CTA builds spill no more than their two-CTA
// ones, when the occupancy query finds three resident (the shared memory of a CTA decides: the directory of the ordered
// table is staged in it, 16 KB at the default 2^12 blocks), and two with the generic orbit walk, whose three-CTA build
// spills 100 bytes or more of the pipeline state.  On an H100 (700 W, L2 flushed, 6x6 square, 2^12 blocks) three CTAs take
// 19.1 ms against 20.7 ms at two (complex128), 18.3 against 19.9 ms (float64); a three-CTA build with only two resident
// is twice as slow as the two-CTA one.  Returns the CTAs per SM the launch had resident.
int launch_rows(const KernelParams &p, bool complex_elements, cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return 0;
  const bool mph = p.dense != nullptr && p.dord.blocks == nullptr;
  const int k = rows_torus_k(p.orbit, mph, p.rows_ctas);
  const SmemLayout L = smem_layout(p, PROJ_GROUP, sizeof(double), false);
  const int64_t work = ((p.row_end - p.row_begin + 31) / 32 + kWarps - 1) / kWarps;
  int resident = 0;
  auto launch = [&](auto kernel, bool ord, int tk) {
    const size_t smem = rows_smem(p, L, ord, tk).total;
    resident = resident_ctas(kernel, smem);
    kernel<<<capped_grid(work, (int64_t)sm_count() * std::max(resident, 1)), kThreads, smem, stream>>>(p);
    check_launch("k_rows");
  };
  with_bool(complex_elements, [&](auto ce) {
    with_choice<6, 4, 0>(k, [&](auto tk) {
      if (mph) {   // the dense index (perfect hash) is built for two CTAs per SM and the hashed layout only
        launch(k_rows<ce(), tk(), true, 2, false>, false, tk());
        return;
      }
      const bool ord = p.table_dir.dir != nullptr;   // the ordered layout, or the dense ordered table on its directory
      auto kernel_at = [&](auto ctas) {               // the build of k_rows for p's table at `ctas` CTAs per SM
        constexpr int TK = ctas() == 4 && tk() == 4 ? 0 : tk();   // no 4x4 build at 64 registers (see rows_torus_k)
        if (p.dord.blocks != nullptr) return k_rows<ce(), TK, false, ctas(), true, true>;
        return ord ? k_rows<ce(), TK, false, ctas(), true> : k_rows<ce(), TK, false, ctas(), false>;
      };
      int ctas = p.rows_ctas;
      if (ctas < 0) {
        const size_t smem = rows_smem(p, L, ord, tk()).total;
        ctas = tk() > 0 && resident_ctas(kernel_at(std::integral_constant<int, 3>{}), smem) >= 3 ? 3 : 2;
      }
      with_choice<2, 3, 4>(ctas, [&](auto c) {
        launch(kernel_at(c), ord, c() == 4 && tk() == 4 ? 0 : tk());
      });
    });
  });
  return resident;
}

int rows_torus_k(const OrbitProgram &o, bool dense, int rows_ctas) {
  const int k = (o.canon_mode != 0 && o.tor_mode == 2 && o.canon_k == o.canon_r) ? o.canon_k : 0;
  if (k != 4 && k != 6) return 0;
  if (!o.tor_sq_rows) return 0;   // the row form failed its self-check (upload_orbit): the generic walk
  if (k == 4 && !dense && rows_ctas == 4) return 0;   // no 4x4 build at 64 registers: the generic walk
  return k;
}

// p.batch vectors of p.batch_elt doubles per element (p.batch * p.batch_elt <= 6), p.table = the 64-byte-bucket table
void launch_store_build(const KernelParams &p, const RowsStoreView &s, bool write_pass, unsigned long long *flags,
                        cudaStream_t stream) {
  if (s.n_rows <= 0) return;
  if (s.chunks < 1 || s.chunks > kStoreMaxChunks) throw std::runtime_error("term store: 1 .. 64 column blocks");
  const int k = rows_torus_k(p.orbit, false, 2);
  const SmemLayout L = smem_layout(p, PROJ_GROUP, sizeof(double), false);
  with_choice<6, 4, 0>(k, [&](auto tk) {
    with_bool(write_pass, [&](auto wr) {
      auto kernel = k_store_build<tk(), wr()>;
      const size_t smem = rows_smem(p, L, false, tk()).total;
      opt_in_smem(kernel, smem);
      const int grid = one_wave(kernel, (s.n_tiles + kWarps - 1) / kWarps, smem);
      kernel<<<grid, kThreads, smem, stream>>>(p, s, flags);
      check_launch("k_store_build");
    });
  });
}

void launch_store_offsets(const RowsStoreView &s, cudaStream_t stream) {
  const int64_t n = s.n_tiles * s.chunks;
  k_store_tile_sums<<<capped_grid((n + 255) / 256, (int64_t)sm_count() * 8), 256, 0, stream>>>(s);
  check_launch("k_store_tile_sums");
  k_store_scan<<<1, 1024, 0, stream>>>(s.tile_off, n);
  check_launch("k_store_scan");
}

void launch_rows_stored(const KernelParams &p, const RowsStoreView &s, const void *xs, void *partial, int k0, int k1,
                        bool complex_elements, cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return;
  const int64_t tiles = (p.row_end + 31) / 32 - p.row_begin / 32;
  with_bool(complex_elements, [&](auto ce) {
    using E = typename ValT<ce()>::type;
    auto kernel = k_rows_stored<ce()>;
    constexpr size_t smem = rows_stored_smem<ce()>();
    const int grid = one_wave(kernel, (tiles + kWarps - 1) / kWarps, smem);
    kernel<<<grid, kThreads, smem, stream>>>(p, s, reinterpret_cast<const E *>(xs), reinterpret_cast<E *>(partial), k0,
                                             k1);
    check_launch("k_rows_stored");
  });
}

void launch_rows_batch(const KernelParams &p, cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return;
  if (p.batch < 1 || (p.batch_elt != 1 && p.batch_elt != 2) || p.batch * p.batch_elt > 6)
    throw std::runtime_error("k_rows_batch: at most six doubles per state");
  const OrbitProgram &o = p.orbit;
  const int k = (o.canon_mode != 0 && o.tor_mode == 2 && o.canon_k == o.canon_r) ? o.canon_k : 0;
  const size_t smem = smem_layout(p, PROJ_GROUP, sizeof(double), false).total;
  // two CTAs per SM (120-128 registers: the eight words of the request stay in registers; at 80 registers part of them
  // spills)
  with_choice<6, 4, 0>(k == 6 || k == 4 ? k : 0, [&](auto tk) {
    auto kernel = k_rows_batch<tk(), 2>;
    const int grid = one_wave(kernel, ((p.row_end - p.row_begin + 31) / 32 + kWarps - 1) / kWarps, smem);
    kernel<<<grid, kThreads, smem, stream>>>(p);
    check_launch("k_rows_batch");
  });
}

void launch_table_fill_batch(int64_t n, int num_vectors, int elt, const void *x, int64_t stride, const double *norms,
                             const uint32_t *slot_of, const uint64_t *reps, void *table, cudaStream_t stream) {
  if (n <= 0) return;
  const int blocks = capped_grid((n + 255) / 256, (int64_t)sm_count() * 16);
  k_table_fill_batch<<<blocks, 256, 0, stream>>>(n, num_vectors * elt, elt, reinterpret_cast<const double *>(x), stride, norms,
                                                 slot_of, reps, reinterpret_cast<unsigned char *>(table));
  check_launch("k_table_fill_batch");
}

void launch_table_insert(const uint64_t *reps, int64_t n, void *table, uint32_t n_buckets, int slots_per_bucket,
                         uint32_t *slot_of, cudaStream_t stream, int bucket_bytes, OrderedDir ord) {
  if (n <= 0) return;
  k_table_insert<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reps, n, reinterpret_cast<unsigned char *>(table),
                                                                 n_buckets, slots_per_bucket, slot_of, bucket_bytes, ord);
  check_launch("k_table_insert");
}

void launch_ordered_dir(const uint64_t *reps, int64_t n, OrderedDir ord, uint32_t buckets_per_state, cudaStream_t stream) {
  const int64_t entries = (int64_t)ord.last + 2;
  k_ordered_dir<<<(unsigned)((entries + 255) / 256), 256, 0, stream>>>(reps, n, ord, buckets_per_state,
                                                                        const_cast<uint32_t *>(ord.dir));
  check_launch("k_ordered_dir");
}

void launch_table_fill(int64_t n, bool complex_elements, const void *x, const double *norms, const uint32_t *pos,
                       const uint32_t *slot_of, const uint64_t *reps, void *table, void *dense, cudaStream_t stream,
                       void *compact) {
  if (n <= 0) return;
  const int blocks = capped_grid((n + 255) / 256, (int64_t)sm_count() * 16);
  unsigned char *t = reinterpret_cast<unsigned char *>(table), *d = reinterpret_cast<unsigned char *>(dense);
  unsigned char *c = reinterpret_cast<unsigned char *>(compact);
  with_bool(complex_elements, [&](auto ce) {
    k_table_fill<ce()><<<blocks, 256, 0, stream>>>(n, x, norms, pos, slot_of, reps, t, d, c);
  });
  check_launch("k_table_fill");
}

void launch_mph_mark(const uint64_t *keys, int64_t n, int level, uint32_t n_blocks, unsigned long long *seen,
                     unsigned long long *collide, cudaStream_t stream) {
  if (n <= 0) return;
  k_mph_mark<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(keys, n, level, n_blocks, seen, collide);
  check_launch("k_mph_mark");
}
void launch_mph_compact(const uint64_t *keys, int64_t n, int level, uint32_t n_blocks, const unsigned long long *collide,
                        uint64_t *next, unsigned long long *next_count, cudaStream_t stream) {
  if (n <= 0) return;
  k_mph_compact<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(keys, n, level, n_blocks, collide, next, next_count);
  check_launch("k_mph_compact");
}
void launch_mph_slots(const uint64_t *keys, int64_t n, PerfectHash mph, const void *table, uint32_t n_buckets,
                      int slots_per_bucket, uint32_t *slot_of, unsigned long long *status, cudaStream_t stream) {
  if (n <= 0) return;
  k_mph_slots<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(keys, n, mph, reinterpret_cast<const unsigned char *>(table),
                                                              n_buckets, slots_per_bucket, slot_of, status);
  check_launch("k_mph_slots");
}

void launch_generate(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements, bool count_only,
                     cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return;
  with_values(proj, complex_values, complex_elements, p.orbit, [&](auto pj, auto cv, auto ce, auto fs) {
    with_bool(count_only, [&](auto co) {
      auto kernel = k_generate<pj(), cv(), ce(), co(), fs()>;
      const SmemLayout L = smem_layout(p, pj(), sizeof(typename ValT<cv()>::type));
      if (L.total > 40 * 1024)   // let several CTAs with large tables share the SM
        CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      const int rpt = 32 / (p.row_split > 1 ? p.row_split : 1);
      const int64_t tiles = (p.row_end - p.row_begin + rpt - 1) / rpt;
      // grid = a whole number of waves of resident CTAs (SMs x per_sm), or fewer when the work is small
      const int wave = one_wave(kernel, (tiles + kWarps - 1) / kWarps, L.total);
      kernel<<<p.grid_blocks > 0 ? p.grid_blocks : wave, kThreads, L.total, stream>>>(p);
      check_launch("k_generate");
    });
  });
}

void launch_pull(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements, cudaStream_t stream) {
  if (p.row_end <= p.row_begin) return;
  with_values(proj, complex_values, complex_elements, p.orbit, [&](auto pj, auto cv, auto ce, auto fs) {
    auto kernel = k_pull<pj(), cv(), ce(), fs()>;
    const SmemLayout L = smem_layout(p, pj(), sizeof(typename ValT<cv()>::type));
    const int grid = one_wave(kernel, ((p.row_end - p.row_begin + 31) / 32 + kWarps - 1) / kWarps, L.total);
    kernel<<<grid, kThreads, L.total, stream>>>(p);
    check_launch("k_pull");
  });
}

void launch_accumulate(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements, int64_t count,
                       const uint64_t *betas, const double *coeffs, cudaStream_t stream) {
  if (count <= 0) return;
  const int blocks = capped_grid(((count + 1) / 2 + kThreads - 1) / kThreads, (int64_t)sm_count() * 8);
  with_values(proj, complex_values, complex_elements, p.orbit, [&](auto pj, auto cv, auto ce, auto fs) {
    k_accumulate<pj(), cv(), ce(), fs()><<<blocks, kThreads, 0, stream>>>(p, count, betas, coeffs);
    check_launch("k_accumulate");
  });
}

void launch_apply_diag(const KernelParams &p, int64_t count, const uint64_t *alphas, double *coeffs,
                       cudaStream_t stream) {
  if (count <= 0) return;
  const SmemLayout L = smem_layout(p, PROJ_NONE, sizeof(double2));
  opt_in_smem(k_apply_diag, L.total);
  const int blocks = capped_grid((count + kThreads - 1) / kThreads, (int64_t)sm_count() * 4);
  k_apply_diag<<<blocks, kThreads, L.total, stream>>>(p, count, alphas, coeffs);
  check_launch("k_apply_diag");
}

void launch_apply_off_diag(const KernelParams &p, int64_t count, const uint64_t *alphas, const int64_t *offsets,
                           int64_t *counts, uint64_t *betas, double *coeffs, bool write_pass, cudaStream_t stream) {
  if (count <= 0) return;
  const SmemLayout L = smem_layout(p, PROJ_NONE, sizeof(double2));
  const int blocks = capped_grid((count + kThreads - 1) / kThreads, (int64_t)sm_count() * 4);
  with_bool(write_pass, [&](auto write) {
    opt_in_smem(k_apply_off_diag<write()>, L.total);
    k_apply_off_diag<write()><<<blocks, kThreads, L.total, stream>>>(p, count, alphas, offsets, counts, betas,
                                                                      reinterpret_cast<double2 *>(coeffs));
  });
  check_launch("k_apply_off_diag");
}

void launch_build_directory(const uint64_t *reps, int64_t n, uint32_t *dir, uint64_t n_buckets, int shift,
                            cudaStream_t stream) {
  const int64_t items = 2 * (int64_t)n_buckets;
  k_build_directory<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(reps, n, dir, n_buckets, shift);
  check_launch("k_build_directory");
}

void launch_state_index(const StateIndex &ix, int64_t count, const uint64_t *spins, int64_t *indices,
                        cudaStream_t stream) {
  if (count <= 0) return;
  k_state_index<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(ix, count, spins, indices);
  check_launch("k_state_index");
}

void launch_verify_rank(const StateIndex &ix, unsigned long long *status, cudaStream_t stream) {
  if (ix.n <= 0) return;
  k_verify_rank<<<(unsigned)((ix.n + 255) / 256), 256, 0, stream>>>(ix, status);
  check_launch("k_verify_rank");
}

void launch_locale_idx(int64_t count, const uint64_t *states, int num_ranks, uint8_t *keys, cudaStream_t stream) {
  if (count <= 0) return;
  k_locale_idx<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(count, states, num_ranks, keys);
  check_launch("k_locale_idx");
}

void launch_state_info(const OrbitProgram &P, Projection proj, uint64_t site_mask, double inv_char,
                       int64_t count, const uint64_t *alphas, uint64_t *betas, double *characters,
                       double *norms, cudaStream_t stream) {
  if (count <= 0) return;
  const unsigned blocks = (unsigned)((count + 127) / 128);
  double2 *ch = reinterpret_cast<double2 *>(characters);
  with_choice<PROJ_NONE, PROJ_INVERSION, PROJ_GROUP>(proj, [&](auto pj) {
    with_bool(pj() == PROJ_GROUP && P.fermionic != 0, [&](auto fs) {
      if constexpr (pj() == PROJ_GROUP || !fs())
        k_state_info<pj(), fs()><<<blocks, 128, 0, stream>>>(P, site_mask, inv_char, count, alphas, betas, ch, norms);
    });
  });
  check_launch("k_state_info");
}

void launch_compute_norms(const OrbitProgram &P, int64_t count, const uint64_t *reps, double *norms,
                          cudaStream_t stream) {
  if (count <= 0) return;
  with_bool(P.fermionic != 0, [&](auto fs) {
    k_compute_norms<fs()><<<(unsigned)((count + 127) / 128), 128, 0, stream>>>(P, count, reps, norms);
  });
  check_launch("k_compute_norms");
}

void launch_enumerate(const OrbitProgram &P, Projection proj, uint64_t site_mask, bool fixed_hamming,
                      uint64_t half_mask, int half_weight, int rank, int num_ranks, int64_t n_chunks,
                      const uint64_t *chunk_first,
                      const uint64_t *chunk_last, unsigned long long *chunk_count,
                      const unsigned long long *chunk_offset, uint64_t *out, double *out_norms,
                      bool write_pass, cudaStream_t stream) {
  if (n_chunks <= 0) return;
  const unsigned blocks = (unsigned)((n_chunks + 127) / 128);
  with_choice<PROJ_NONE, PROJ_INVERSION, PROJ_GROUP>(proj, [&](auto pj) {
    with_bool(write_pass, [&](auto write) {
      with_bool(pj() == PROJ_GROUP && P.fermionic != 0, [&](auto fs) {
        if constexpr (pj() == PROJ_GROUP || !fs())
          k_enumerate<pj(), write(), fs()><<<blocks, 128, 0, stream>>>(P, site_mask, fixed_hamming, half_mask, half_weight,
                                                                       rank, num_ranks, n_chunks, chunk_first, chunk_last,
                                                                       chunk_count, chunk_offset, out, out_norms);
      });
    });
  });
  check_launch("k_enumerate");
}

}  // namespace dmv
