// dmv_device.cuh -- device-side data structures and helpers of the H.x hot path (sm_90a).
//
// Everything here is integer / bit-twiddling + sparse FP64 FMA: no tensor cores (north_star).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dmv {

// ---------------------------------------------------------------------------------------------
// Operator tables (device copies of dmv_operator_desc, regrouped by flip mask)
// ---------------------------------------------------------------------------------------------
struct OffTerm {      // one non-branching term of a group: c += v [alpha & m == r] (-1)^popc(alpha & s)
  uint64_t m, r, s;
  double v_re, v_im;
};
struct TermGroup {    // all terms with the same flip mask x: beta = alpha ^ x
  uint64_t x;
  int32_t first, count;
};
struct DiagTerm {
  uint64_t m, r, s;
  double v_re, v_im;
};

// Flip-mask group in look-up-table form.  All terms of the group act on the k <= 6 "support" bits
// pos[0..k) (the union of their masks m); the coefficient is a function of those bits only,
//     c(alpha) = lut[lut_offset + idx(alpha)] * (-1)^popc(alpha & s_out),   idx = sum_b bit(alpha, pos[b]) << b
// and the group emits iff bit idx of emit_bits is set.  For a Heisenberg bond k = 2 and the whole
// (state, bond) test is two bit extractions and one shift.  Groups that do not fit (k > 6, or terms with
// different sign masks outside the support) keep generic = 1 and are evaluated term by term.
struct LutGroup {
  uint64_t x;          // flip mask: beta = alpha ^ x
  uint64_t s_out;      // common sign mask outside the support
  uint64_t emit_bits;
  uint64_t posk;       // bytes 0..5: pos[b]; byte 6: k; byte 7: generic flag
  uint32_t lut_offset;
  int32_t first, count;  // term range for the generic evaluation
  uint32_t pad;
};
static_assert(sizeof(LutGroup) == 48, "LutGroup layout");

// Bit-parallel emit test for operators whose groups all have a support of <= 2 bits (every two-body
// spin Hamiltonian): for a word of <= 64 groups, A_b = "support bit b of every group" is gathered from
// the state by a few masked shifts (the host orders the groups so that few distinct shifts occur: a
// chain needs 2 per operand), and the groups that emit are
//     mask = (~A0 & ~A1 & tt[0]) | (A0 & ~A1 & tt[1]) | (~A0 & A1 & tt[2]) | (A0 & A1 & tt[3]).
constexpr int kBpPairs = 24;   // distinct shifts per operand and word; more -> walk the groups
struct BpPair {            // A |= ((a << l) >> r) & m   (one of l, r is zero); one 16-byte load
  uint64_t m;
  uint32_t l, r;
};
struct BpWord {
  uint64_t tt[4];
  BpPair p0[kBpPairs], p1[kBpPairs];
  int32_t n0, n1;
};
static_assert(sizeof(BpWord) == 32 + 32 * kBpPairs + 8, "BpWord layout");

// Diagonal terms of the form v (-1)^(bit_i ^ bit_j) (every sigma^z sigma^z coupling) grouped by coefficient:
//   sum over the class = v * (count - 2 popc((A0 ^ A1) & mask)),   A_b gathered by masked shifts as in BpWord.
struct DiagClass {
  double v_re, v_im;
  int32_t count, n0, n1, pad;
  uint64_t mask;
  BpPair p0[kBpPairs], p1[kBpPairs];
};
static_assert(sizeof(DiagClass) == 40 + 32 * kBpPairs, "DiagClass layout");

__host__ __device__ __forceinline__ unsigned lut_index(uint64_t posk, uint64_t a) {
  const unsigned k = (unsigned)(posk >> 48) & 0xffu;
  unsigned idx = 0;
  for (unsigned b = 0; b < k; ++b) idx |= (unsigned)((a >> ((posk >> (8 * b)) & 0xffu)) & 1ull) << b;
  return idx;
}

// ---------------------------------------------------------------------------------------------
// Orbit program: the symmetry group enumerated as  g = t_j . q_i  (+ optional spin flip)
//   q_i : coset representatives, applied as Benes butterfly networks (padded to n_stages)
//   t_j : a chain through a subgroup of "cheap" elements, t_j = c_j . t_{j-1}; every step c_j is a
//         short list of masked shifts (n_left left shifts + n_right right shifts, zero padded)
// Built on the host by compile_orbit_program() (dmv_group.cpp).
// ---------------------------------------------------------------------------------------------
struct OrbitProgram {
  int32_t n_sites;
  int32_t n_q, n_stages, n_t, n_left, n_right;
  int32_t has_flip;            // group doubled by global spin inversion
  int32_t trivial_characters;  // every character == 1
  uint64_t site_mask;
  const uint64_t *benes_mask;  // [n_q][n_stages]
  const int32_t *benes_delta;  // [n_stages]
  const uint64_t *step_mask;   // [n_t-1][n_left + n_right]  (mask in OUTPUT positions)
  const int32_t *step_shift;   // [n_t-1][n_left + n_right]
  const double2 *characters;   // [n_q][n_t][2]  character of (t_j . q_i, flip); conj NOT applied; fermionic programs
                               // continue with the inversion masks (orbit_sign)
  int64_t group_order;         // n_q * n_t * (has_flip ? 2 : 1)
  // fast paths for chains whose every step is one left + one right masked shift (translations):
  //   step_pack32[j] = {mask_left, mask_right, shift_left, shift_right}   (n_sites <= 32: 32-bit arithmetic)
  //   step_pack64[3j..3j+2] = {mask_left, mask_right, shift_left | shift_right << 32}
  int32_t simple;              // 0: general; 1: packed steps are valid
  // fermionic bases: characters[n_q * n_t * 2 ..] holds, as uint64, per element e = q * n_t + j and bit i the inversion mask
  //   M_e[i] = { j < i : image(j) > image(i) },   image(j) = the output bit that takes input bit j,
  // so U_g|s> = sign(g, s)|g(s)> with sign(g, s) = (-1)^(sum over set bits i of s of popc(s & M_e[i])) (orbit_sign).  A
  // fermionic program never takes the representative-only forms (canon_mode, tor_mode, simple, orbit_representative): they
  // give no element, so trivial_characters is 0 there.  (The masks share the characters' buffer, so OrbitProgram keeps
  // its size and the spin builds their code.)
  int32_t fermionic;
  const uint4 *step_pack32;    // [n_t - 1] or nullptr
  const uint64_t *step_pack64; // [3 (n_t - 1)]
  // canonical form under the chain subgroup WITHOUT walking it, when that subgroup is the group of block rotations
  //   { rotate the bits inside every k-bit block by a, rotate the R blocks by b },  n_sites = k R
  // (translations of a chain: R = 1; of an R x k torus numbered row by row): see translation_canon()
  //   1: k <= 8, R <= 8: the top block of the minimum is the smallest rotation of any block (LUT over 2^k block
  //      values); only the few (block, amount) pairs reaching it are expanded
  //   2: R = 1: the minimum rotation starts with the longest cyclic run of zeros; runs are found by iterated AND
  int32_t canon_mode, canon_k, canon_r;
  int32_t chain_dihedral;      // mode 2: G = rotations [x mirror] [x flip] exactly: one pass over the runs (min_rotation_dihedral); 1 | 2 (with mirror)
  const uint16_t *canon_lut;   // [2^k]: (set of amounts reaching the minimum) << 8 | minimum rotation of the block value
  const uint64_t *canon_masks; // [2 k]: masks of rotating every block right by a: (low part, wrapped part)
  //   mode 1 with 2 k <= 12: the LUT runs over PAIRS of adjacent blocks (top two blocks of a candidate), which leaves
  //   one candidate for all but symmetric states:  canon_lut2[hi << k | lo] = amounts << 16 | minimum rotated pair
  const uint32_t *canon_lut2;  // nullptr: single-block LUT
  int32_t canon_div;           // floor(bit / k) = (bit * canon_div) >> 16 for bit < 64
  // coset representatives for the canonical-form scan as a CHAIN: q_0 = identity, q_i = c_i . q_{i-1} with c_i a cheap
  // involution of the group (reflections: a few delta-swaps) or, failing that, a full network
  int32_t cc_n;                // number of cosets (0: use the independent networks above)
  int32_t cc_stages;           // total number of stages = cc_begin[cc_n]
  const int32_t *cc_begin;     // [cc_n + 1] stage ranges
  const uint64_t *cc_mask;     // delta-swap stages
  const int32_t *cc_delta;
  // canonical form under the FULL space group of an R x k torus (sites numbered row by row, trivial characters):
  //   G = {block rotations} x {1, rho} x {1, sigma} [x {1, tau}] [x {1, flip}]
  // rho = reverse the bits inside every row, sigma = reverse the order of the rows, tau = transpose (R == k).
  // Every image is "a row pair on top": m(hi, lo) is the smallest top pair over the 2k (x2 with the flip) maps
  // F = flip^f . rho^e . rot_a applied to both rows, tor_luts[hi << k | lo] the set of (f, e, a) reaching it
  // (bit (2f + e) k + a); only the few (row pair, F) whose top pair is the global minimum are expanded.  See
  // orbit_min_torus().  tor_lutm[hi << k | lo] = m(hi, lo) | m(lo, hi) << 16 holds both orders of the pair, so one
  // look-up per pair of adjacent rows serves both directions.
  int32_t tor_mode;            // 0: off; 1: rho and sigma (4 cosets of the block rotations); 2: and tau (8 cosets)
  int32_t tor_rho_n, tor_tau_n;   // delta-swap stages of rho / tau inside tor_net_*: rho first, then tau
  int32_t tor_div_r;           // floor(bit / R) = (bit * tor_div_r) >> 16 for bit < 32
  int32_t tor_sq_rows;         // 1: k_rows evaluates the square form per row (orbit_min_torus_sq_t), self-checked against
                               // orbit_min_torus_sq on the probe states x every flip mask of the operator
  const uint32_t *tor_lutm;    // [2^(2k)]
  const uint32_t *tor_luts;    // [2^(2k)]  (stays in global memory: read about once per state)
  const uint8_t *tor_frow;     // [4 k][2^k]: image of one row under F = flip^f rho^e rot_a, F = (2 f + e) k + a
  const uint64_t *tor_net_mask;
  const int32_t *tor_net_delta;
};

// ---------------------------------------------------------------------------------------------
// hash64_01 / localeIdxOf            reference: src/StatesEnumeration.chpl:122-136
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t hash64_01(uint64_t x) {
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  x = x ^ (x >> 31);
  return x;
}

// owner = hash % P.  P is tiny (<= 256): use a 32-bit friendly path for powers of two.
__host__ __device__ __forceinline__ int locale_idx_of(uint64_t state, int num_ranks) {
  if (num_ranks <= 1) return 0;
  const uint64_t h = hash64_01(state);
  if ((num_ranks & (num_ranks - 1)) == 0) return (int)(h & (uint64_t)(num_ranks - 1));
  return (int)(h % (uint64_t)num_ranks);
}

// ---------------------------------------------------------------------------------------------
// State -> index.  Replaces ls_hs_state_index (reference src/FFI.chpl:173-175, call DMV:102) and the
// per-basis `state_index_kernel` the third-party library installs (src/FFI.chpl:90-93):
//   INDEX_DIRECTORY : sorted representatives; directory over the top bits + bounded binary search
//   INDEX_IDENTITY  : state_index_is_identity (DMV:86): index == state
//   INDEX_RANK      : full fixed-Hamming-weight basis (optionally halved by spin inversion) on one
//                     rank: the index is the combinadic rank, computed from a binomial table with no
//                     memory traffic to the representatives (ls_hs_fixed_hamming_state_to_index,
//                     reference src/FFI.chpl:165).  Results are bit-identical to the search.
// ---------------------------------------------------------------------------------------------
//   INDEX_LIN       : same bases as INDEX_RANK: two-table (Lin) lookup  index = Ja[s >> h] + Jb[s & mask]:
//                     two independent small-table loads, no dependent probe chain, bit-identical results.
//   INDEX_LIN_SPLIT : spinful-fermion basis (hi = down half, lo = up half, both at fixed weight), ascending = (hi, lo)
//                     lexicographic: Ja[hi] = rank of hi among the N_dn-weight words x C(N, N_up), Jb[lo] = rank of lo
//                     among the N_up-weight words.  A wrong-weight hi has Ja = 0xffffffff and a wrong-weight lo Jb = 0:
//                     at the right total weight both halves are wrong together, so the sum is >= n and never wraps.
//                     The device runs it as INDEX_LIN (same look-up, other tables); only the host tells them apart.
enum IndexMode { INDEX_DIRECTORY = 0, INDEX_IDENTITY = 1, INDEX_RANK = 2, INDEX_LIN = 3, INDEX_LIN_SPLIT = 4 };

struct StateIndex {
  const uint64_t *reps;   // ascending, this rank's block
  int64_t n;
  const uint32_t *dir;    // pairs: dir[2b] = lower_bound(reps, b << shift), dir[2b+1] = lower_bound(reps, (b+1) << shift)
  uint64_t n_buckets;
  int32_t shift;
  int32_t mode;           // IndexMode
  // INDEX_RANK
  const uint32_t *binom;  // [n_sites][weight + 2]: binom[pos * stride + k] = C(pos, k) (saturated)
  int32_t stride, n_sites, weight;
  uint64_t site_mask;
  // INDEX_LIN
  const uint32_t *lin_a, *lin_b;   // Ja[2^(n - h)], Jb[2^h]
  int32_t lin_bits;                // h: number of low bits
};

__device__ __forceinline__ int64_t locate_directory(const StateIndex &ix, uint64_t key) {
  const uint64_t b = key >> ix.shift;
  if (b >= ix.n_buckets) return -1;
  // one 8-byte load: (first, one-past-last) position of the bucket
  const uint2 range = __ldg(reinterpret_cast<const uint2 *>(ix.dir) + b);
  uint32_t lo = range.x, hi = range.y;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint64_t v = __ldg(ix.reps + mid);
    if (v == key) return (int64_t)mid;   // states are unique: stop at the first hit
    if (v < key) lo = mid + 1; else hi = mid;
  }
  return -1;
}

// sum over the set bits of `bits` (ascending) of C(pos, k), k = k0 + 1, k0 + 2, ...
__device__ __forceinline__ uint32_t combinadic_sum(const uint32_t *binom, int stride, uint64_t bits, int k0) {
  uint32_t acc = 0;
  int k = k0;
  while (bits) {
    const int pos = __ffsll((long long)bits) - 1;
    ++k;
    acc += binom[pos * stride + k];
    bits &= bits - 1;
  }
  return acc;
}

__device__ __forceinline__ int64_t locate_rank(const StateIndex &ix, const uint32_t *binom, uint64_t key) {
  if ((key & ~ix.site_mask) != 0 || __popcll(key) != ix.weight) return -1;
  const int64_t r = (int64_t)combinadic_sum(binom, ix.stride, key, 0);
  return r < ix.n ? r : -1;   // with spin inversion only the first half are representatives
}

// Rank of key = src ^ flip given rank(src) = src_index: only the bits inside the span of `flip` move.
__device__ __forceinline__ int64_t locate_rank_incremental(const StateIndex &ix, const uint32_t *binom,
                                                           uint64_t key, uint64_t src, int64_t src_index,
                                                           uint64_t flip) {
  const int lo = __ffsll((long long)flip) - 1;
  const int hi = 63 - __clzll((long long)flip);
  const uint64_t span = ((hi == 63) ? ~0ull : ((1ull << (hi + 1)) - 1)) & ~((1ull << lo) - 1);
  const uint64_t ob = src & span, nb = key & span;
  if ((key & ~ix.site_mask) != 0 || __popcll(ob) != __popcll(nb)) return -1;   // weight not preserved
  const int k0 = __popcll(src & ((1ull << lo) - 1));
  const int64_t r = src_index - (int64_t)combinadic_sum(binom, ix.stride, ob, k0) +
                    (int64_t)combinadic_sum(binom, ix.stride, nb, k0);
  return r < ix.n ? r : -1;
}

__device__ __forceinline__ int64_t locate_lin(const StateIndex &ix, uint64_t key) {
  if ((key & ~ix.site_mask) != 0 || __popcll(key) != ix.weight) return -1;
  const uint32_t lo = (uint32_t)(key & ((1ull << ix.lin_bits) - 1)), hi = (uint32_t)(key >> ix.lin_bits);
  const int64_t r = (int64_t)__ldg(ix.lin_a + hi) + (int64_t)__ldg(ix.lin_b + lo);
  return r < ix.n ? r : -1;   // with spin inversion only the first half are representatives
}

__device__ __forceinline__ int64_t locate(const StateIndex &ix, uint64_t key) {
  if (ix.mode == INDEX_LIN) return locate_lin(ix, key);
  if (ix.mode == INDEX_IDENTITY) return (key < (uint64_t)ix.n) ? (int64_t)key : -1;
  if (ix.mode == INDEX_RANK) return locate_rank(ix, ix.binom, key);
  return locate_directory(ix, key);
}

// ---------------------------------------------------------------------------------------------
// State -> vector element in ONE dependent memory access: open-addressing hash table over the representatives with
// the vector element stored in the slot (row traversal of bases with permutation symmetries, k_rows).  The sorted
// array + directory needs  directory -> several probes -> norm -> x  dependent loads per term, and orbit minima
// cluster at small values, which unbalances any directory over the top bits; here a term costs the 32-byte sector of
// its bucket.  The values are refreshed once per product
// (k_table_fill: x[i] * norm[i] at slot_of[i]).  The table takes 64 .. 256 bytes per state (ensure_table: fewer
// for the ordered layout below and when free memory is short).  A bucket is ONE 32-byte sector, fetched with two independent 128-bit loads:
// random look-ups are bound by the rate at which HBM serves random sectors (tools/random_access.cu measures it), so
// the look-up costs what its sector costs.  A state goes to the first bucket from its home with a free slot; a look-up that finds its
// bucket taken by other states moves on to the next one (7 % of the look-ups for complex128, 2 % for float64).
//   complex128: bucket = one slot  { key, spare, re, im },            8 buckets per state
//   float64:    bucket = two slots { key0, key1, value0, value1 },    2 buckets per state
// ---------------------------------------------------------------------------------------------
constexpr uint64_t kEmptyKey = ~0ull;
__host__ __device__ __forceinline__ uint32_t table_slot(uint64_t key, uint32_t n_buckets) {
  const uint64_t h = key * 0x9E3779B97F4A7C15ull;
  return (uint32_t)(((h >> 32) * (uint64_t)n_buckets) >> 32);
}

// Ordered layout of the same table (k_rows, rows_table = 1).  The hash above scatters the representatives over the
// whole table, so no row order gives L2 reuse.  But most off-diagonal targets of a row share its leading key bits
// (tools/lookup_locality.py), and the rows run in ascending key order.  So the table is cut into blocks by key prefix:
// block p = (key - k_lo) >> shift holds buckets [dir[p], dir[p + 1]), buckets_per_state times the number of
// representatives with that prefix, and a state's home is hashed inside its block.  The part of the table that the rows
// in flight read is then a narrow window that the L2 holds.  Linear probing, the empty key and the look-up are as in
// the hashed layout.  dir[p] = buckets_per_state * (first representative >= k_lo + (p << shift)) in the sorted basis.
struct OrderedDir {
  const uint32_t *dir;   // last + 2 bucket offsets; null: hashed layout
  uint64_t k_lo;         // smallest representative
  uint32_t shift, last;  // block of a key = min((key - k_lo) >> shift, last)
};
__host__ __device__ __forceinline__ uint32_t ordered_block(uint64_t key, uint64_t k_lo, uint32_t shift, uint32_t last) {
  const uint64_t q = (key - k_lo) >> shift;   // keys below k_lo wrap to large values and go to the last block
  return q < last ? (uint32_t)q : last;
}
__host__ __device__ __forceinline__ uint32_t ordered_slot(uint64_t key, uint32_t lo, uint32_t hi) {
  return lo + table_slot(key, hi - lo);       // an empty block (hi = lo) sends its keys to the next block's start
}
// home bucket of a key in either layout
__host__ __device__ __forceinline__ uint32_t table_home(uint64_t key, uint32_t n_buckets, const OrderedDir &D) {
  if (D.dir == nullptr) return table_slot(key, n_buckets);
  const uint32_t p = ordered_block(key, D.k_lo, D.shift, D.last);
  return ordered_slot(key, D.dir[p], D.dir[p + 1]);
}
// first index of the sorted a[0, n) with a[i] >= v
__host__ __device__ __forceinline__ int64_t lower_bound_u64(const uint64_t *a, int64_t n, uint64_t v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
// directory entry p of the ordered layout over the sorted representatives reps[0, n)
__host__ __device__ __forceinline__ uint32_t ordered_dir_entry(const uint64_t *reps, int64_t n, const OrderedDir &D,
                                                               uint32_t buckets_per_state, uint32_t p) {
  const int64_t first = p > D.last ? n : lower_bound_u64(reps, n, D.k_lo + ((uint64_t)p << D.shift));
  return (uint32_t)(buckets_per_state * first);
}
// at most 2^bits blocks over the representatives k_lo .. k_hi (dir left null)
inline OrderedDir ordered_plan(uint64_t k_lo, uint64_t k_hi, int bits) {
  const uint64_t range = k_hi - k_lo;
  int used = 0;
  while (used < 64 && (range >> used) != 0) ++used;
  OrderedDir D{nullptr, k_lo, used > bits ? (uint32_t)(used - bits) : 0u, 0u};
  D.last = (uint32_t)(range >> D.shift);
  return D;
}

// ---------------------------------------------------------------------------------------------
// Dense index for k_rows: a two-level perfect hash over the representatives.  The open-addressing table above is bound by
// the rate at which HBM serves RANDOM sectors, and that rate falls as the table grows from a few times
// the L2 to gigabytes; a perfect hash needs no empty slots, so the table of (key, value) slots
// shrinks from 256 N to 32 N bytes.  Level l is an array of 32-byte blocks { w0, w1, w2, prefix }: 192 bits of which bit
// p is set iff exactly ONE state hashes to p at this level (then it owns the slot prefix + popcount of the set bits
// before p in the block); states that collide at level 0 try level 1, the few per cent left over live in the
// open-addressing table.  Both blocks of a look-up are requested together (two 32-byte blocks that hit L2: 5 bits per
// state), the slot one pipeline step later.
// ---------------------------------------------------------------------------------------------
struct PerfectHash {
  const unsigned char *blocks;   // [n_blocks0 + n_blocks1][32]
  uint32_t n_blocks0, n_blocks1; // blocks of level 0 / level 1
  uint32_t n_dense;              // states placed by the two levels = slots of the dense table
};
constexpr uint32_t kMphBits = 192;
constexpr uint32_t kMphMissing = 0xffffffffu;
// (block, bit) of a state at a level
__host__ __device__ __forceinline__ void mph_position(uint64_t key, int level, uint32_t n_blocks, uint32_t &block, uint32_t &bit) {
  uint64_t h = key * (level == 0 ? 0x9E3779B97F4A7C15ull : 0xC2B2AE3D27D4EB4Full);
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  block = (uint32_t)(((h >> 32) * (uint64_t)n_blocks) >> 32);
  bit = (uint32_t)(((h & 0xffffffffull) * (uint64_t)kMphBits) >> 32);
}
// slot owned at position `bit` of a block, or kMphMissing when the bit is not set
__host__ __device__ __forceinline__ uint32_t mph_rank(uint64_t w0, uint64_t w1, uint64_t w2, uint64_t prefix, uint32_t bit) {
  const uint32_t word = bit >> 6, b = bit & 63u;
  const uint64_t w = word == 0 ? w0 : (word == 1 ? w1 : w2);
  if (!((w >> b) & 1ull)) return kMphMissing;
  const uint64_t below = w & ((1ull << b) - 1ull);
#ifdef __CUDA_ARCH__
  uint32_t r = (uint32_t)prefix + (uint32_t)__popcll(below);
  if (word > 0) r += (uint32_t)__popcll(w0);
  if (word > 1) r += (uint32_t)__popcll(w1);
#else
  uint32_t r = (uint32_t)prefix + (uint32_t)__builtin_popcountll(below);
  if (word > 0) r += (uint32_t)__builtin_popcountll(w0);
  if (word > 1) r += (uint32_t)__builtin_popcountll(w1);
#endif
  return r;
}

// ---------------------------------------------------------------------------------------------
// Dense ordered table for k_rows (option rows_dense_order): ONE slot per state (32 bytes {key, spare, re, im} /
// 16 bytes {key, value}), the slots in key order at the granularity of the ordered layout's prefix blocks, so a near
// window of the table holds 8 times as many states as with 8 buckets per state.  The directory is the ordered layout's
// with one slot per state (dir[p] = first representative of prefix block p).  A key of block p hashes to a virtual
// position in [dir[p], dir[p + 1]); positions are cut into rank blocks of kDordStates states, and a rank block is one
// 32-byte sector { w0, w1, w2, first | level-2 bits << 32 | leftovers << 56 }:
//   level 0: 128 bits (w0, w1); bit b is set iff exactly one key of the rank block hashes to b;
//   level 1: 64 bits (w2) over the keys that collided at level 0, likewise;
//   level 2: 24 bits over the keys that collided at level 1, likewise;
//   the keys no level places ("leftovers", 0.3 % on the 6x6 square) follow the placed ones in key order.
// The keys of rank block R own slots [first, first + count): level-0 keys by rank among the set bits of w0 w1, then
// level-1 and level-2 keys, then the leftovers, found by a short scan.  first = number of keys of the rank blocks before
// R, so a key of block p lands in [dir[p], dir[p + 1]) up to about one rank block on either side (the rank blocks at the
// block's ends also hold keys of its neighbours, as many as hash there).  One rank-block read (L2-resident:
// 6.4 bits per state) and one slot read per look-up, both independent of how full the table is.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kDordStates = 40;
struct DenseOrder {
  const uint64_t *blocks;   // [n_blocks][4]; null: not in use
  uint32_t n_blocks;
  uint32_t n_placed;        // states the two levels place (the rest are leftovers)
};
__host__ __device__ __forceinline__ uint64_t dord_hash(uint64_t key) {
  uint64_t h = key * 0x9E3779B97F4A7C15ull;
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  return h ^ (h >> 31);
}
// rank block of a key with hash h whose prefix block holds states [lo, hi); level bits b0 | b1 << 8
__host__ __device__ __forceinline__ uint32_t dord_block(uint64_t h, uint32_t lo, uint32_t hi) {
  const uint32_t v = lo + (uint32_t)(((h >> 32) * (uint64_t)(hi - lo)) >> 32);
  return v / kDordStates;
}
__host__ __device__ __forceinline__ uint32_t dord_bits(uint64_t h) {
  return (uint32_t)(h & 127u) | (uint32_t)((h >> 7) & 63u) << 8 | (uint32_t)((((h >> 13) & 0xffffu) * 24u) >> 16) << 16;
}
__host__ __device__ __forceinline__ uint32_t dord_popc(uint64_t w) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__popcll(w);
#else
  return (uint32_t)__builtin_popcountll(w);
#endif
}
// first slot to read for a key of the rank block { w0, w1, w2, w3 }, and the end of the slots it may be in: one slot
// when a level places the key, else the block's leftovers (end == slot: none, the key is not a basis state)
__host__ __device__ __forceinline__ uint32_t dord_slot(uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3, uint32_t bits,
                                                       uint32_t &end) {
  const uint32_t b0 = bits & 127u, b1 = (bits >> 8) & 63u, first = (uint32_t)w3;
  const uint64_t m = b0 < 64 ? w0 : w1;
  const uint32_t p0 = dord_popc(w0);
  if ((m >> (b0 & 63u)) & 1ull) {
    const uint32_t s = first + (b0 < 64 ? 0u : p0) + dord_popc(m & ((1ull << (b0 & 63u)) - 1ull));
    end = s + 1;
    return s;
  }
  const uint32_t p01 = p0 + dord_popc(w1);
  if ((w2 >> b1) & 1ull) {
    const uint32_t s = first + p01 + dord_popc(w2 & ((1ull << b1) - 1ull));
    end = s + 1;
    return s;
  }
  const uint32_t p012 = p01 + dord_popc(w2), w3b = (uint32_t)(w3 >> 32) & 0xffffffu, b2 = bits >> 16;
  if ((w3b >> b2) & 1u) {
    const uint32_t s = first + p012 + dord_popc(w3b & ((1u << b2) - 1u));
    end = s + 1;
    return s;
  }
  const uint32_t s = first + p012 + dord_popc(w3b);
  end = s + (uint32_t)(w3 >> 56);
  return s;
}

// ---------------------------------------------------------------------------------------------
// Bit permutations
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t butterfly(uint64_t s, uint64_t mask, int delta) {
  const uint64_t t = ((s >> delta) ^ s) & mask;
  return s ^ t ^ (t << delta);
}

// Result of an orbit scan
struct OrbitResult {
  uint64_t rep;     // min_g g(s)
  int32_t arg;      // ((q * n_t + j) << 1) | flipped   of a minimising element
  int32_t stab;     // number of elements with g(s) == s   (only filled by orbit_scan<.., true>)
};

// min_g g(s) for trivial characters (no argmin needed), translation-like chains, <= 32 sites:
// everything in 32-bit registers, one 16-byte shared-memory load per group element.
__device__ __forceinline__ uint64_t orbit_min_narrow(const OrbitProgram &P, uint64_t s64) {
  const uint32_t s = (uint32_t)s64, site_mask = (uint32_t)P.site_mask;
  uint32_t best = 0xffffffffu;
  for (int q = 0; q < P.n_q; ++q) {
    uint32_t cur = s;
    const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
    for (int st = 0; st < P.n_stages; ++st) {
      const int d = P.benes_delta[st];
      const uint32_t t = ((cur >> d) ^ cur) & (uint32_t)bm[st];
      cur ^= t ^ (t << d);
    }
    best = min(best, P.has_flip ? min(cur, cur ^ site_mask) : cur);
#pragma unroll 4
    for (int j = 0; j < P.n_t - 1; ++j) {
      const uint4 st = P.step_pack32[j];
      cur = ((cur << st.z) & st.x) | ((cur >> st.w) & st.y);
      best = min(best, P.has_flip ? min(cur, cur ^ site_mask) : cur);
    }
  }
  return (uint64_t)best;
}

__device__ __forceinline__ uint64_t orbit_min_wide(const OrbitProgram &P, uint64_t s) {
  uint64_t best = ~0ull;
  for (int q = 0; q < P.n_q; ++q) {
    uint64_t cur = s;
    const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
    for (int st = 0; st < P.n_stages; ++st) cur = butterfly(cur, bm[st], P.benes_delta[st]);
    best = min(best, P.has_flip ? min(cur, cur ^ P.site_mask) : cur);
#pragma unroll 2
    for (int j = 0; j < P.n_t - 1; ++j) {
      const uint64_t ml = P.step_pack64[3 * j], mr = P.step_pack64[3 * j + 1], sh = P.step_pack64[3 * j + 2];
      cur = ((cur << (uint32_t)sh) & ml) | ((cur >> (uint32_t)(sh >> 32)) & mr);
      best = min(best, P.has_flip ? min(cur, cur ^ P.site_mask) : cur);
    }
  }
  return best;
}

// ---- minimum over all rotations of an n-bit word: it starts with the longest cyclic run of zeros ----------------
__host__ __device__ __forceinline__ int top_bit(uint64_t v) {
#ifdef __CUDA_ARCH__
  return 63 - __clzll((long long)v);
#else
  return 63 - __builtin_clzll(v);
#endif
}
__host__ __device__ __forceinline__ int low_bit(uint32_t v) {
#ifdef __CUDA_ARCH__
  return __ffs((int)v) - 1;
#else
  return __builtin_ffs((int)v) - 1;
#endif
}
__host__ __device__ __forceinline__ uint64_t rotl_n(uint64_t v, int sh, int n, uint64_t mask) {
  return sh ? (((v << sh) | (v >> (n - sh))) & mask) : v;
}
__host__ __device__ __forceinline__ uint64_t min_rotation_runs(uint64_t w, int n, uint64_t mask) {
  const uint64_t z = ~w & mask;
  if (w == 0 || z == 0) return w;          // all zeros / all ones: every rotation is the word itself
  // r = positions p such that bits p, p-1, ..., p-L+1 (cyclically) are all zero; grow L while some run survives
  uint64_t r = z, zr = z;
  for (;;) {
    zr = ((zr << 1) | (zr >> (n - 1))) & mask;     // zr bit p = z bit (p - L)
    const uint64_t r2 = r & zr;
    if (r2 == 0) break;
    r = r2;
  }
  uint64_t best = ~0ull;
  while (r) {                               // one candidate per maximal run: put its top end at the MSB
    const int p = top_bit(r);
    r &= ~(1ull << p);
    const uint64_t c = rotl_n(w, n - 1 - p, n, mask);
    best = c < best ? c : best;
  }
  return best;
}

// the same in 32-bit registers (n <= 32)
__host__ __device__ __forceinline__ uint32_t min_rotation_runs32(uint32_t w, int n, uint32_t mask) {
  const uint32_t z = ~w & mask;
  if (w == 0 || z == 0) return w;
  uint32_t r = z, zr = z;
  for (;;) {
    zr = ((zr << 1) | (zr >> (n - 1))) & mask;
    const uint32_t r2 = r & zr;
    if (r2 == 0) break;
    r = r2;
  }
  uint32_t best = 0xffffffffu;
  while (r) {
#ifdef __CUDA_ARCH__
    const int p = 31 - __clz((int)r);
#else
    const int p = 31 - __builtin_clz(r);
#endif
    r &= ~(1u << p);
    const int sh = n - 1 - p;
    const uint32_t c = sh ? (((w << sh) | (w >> (n - sh))) & mask) : w;
    best = c < best ? c : best;
  }
  return best;
}

// reverse the low n bits of v
__host__ __device__ __forceinline__ uint64_t reverse_bits_n(uint64_t v, int n) {
#ifdef __CUDA_ARCH__
  return __brevll(v) >> (64 - n);
#else
  v = ((v >> 1) & 0x5555555555555555ull) | ((v & 0x5555555555555555ull) << 1);
  v = ((v >> 2) & 0x3333333333333333ull) | ((v & 0x3333333333333333ull) << 2);
  v = ((v >> 4) & 0x0f0f0f0f0f0f0f0full) | ((v & 0x0f0f0f0f0f0f0f0full) << 4);
  v = ((v >> 8) & 0x00ff00ff00ff00ffull) | ((v & 0x00ff00ff00ff00ffull) << 8);
  v = ((v >> 16) & 0x0000ffff0000ffffull) | ((v & 0x0000ffff0000ffffull) << 16);
  v = (v >> 32) | (v << 32);
  return v >> (64 - n);
#endif
}

// min over the rotations of w, of its mirror image (reflect != 0: the group holds i -> n-1-i) and of the spin-flipped
// images (flip != 0), from ONE pass over the runs of w: a minimal image starts with a longest cyclic run of zeros of w
// or -- flipped -- of ones of w, the mirror image has the same runs, and only the kind with the longer longest run can
// win.  Replaces four independent run searches (w, ~w, mirror, ~mirror) and the reflection network.
template <typename W>
__host__ __device__ __forceinline__ W min_rotation_dihedral(W w, int n, W mask, int reflect, int flip) {
  constexpr int BITS = 8 * (int)sizeof(W);
  if (w == 0) return 0;
  if (w == mask) return flip ? (W)0 : mask;
  const W z = (W)(~w & mask);
  W r0 = z, r1 = w, a0 = z, a1 = w;       // r: top ends of the runs of length >= L; a: the mask rotated L times
  int L0 = 1, L1 = 1;
  bool more0 = true, more1 = flip != 0;
  while (more0 | more1) {
    if (more0) {
      a0 = (W)(((a0 << 1) | (a0 >> (n - 1))) & mask);
      const W t = r0 & a0;
      if (t) { r0 = t; ++L0; } else more0 = false;
    }
    if (more1) {
      a1 = (W)(((a1 << 1) | (a1 >> (n - 1))) & mask);
      const W t = r1 & a1;
      if (t) { r1 = t; ++L1; } else more1 = false;
    }
  }
  W best = (W)~(W)0;
  for (int kind = 0; kind < (flip ? 2 : 1); ++kind) {
    if (flip && (kind == 0 ? L0 < L1 : L1 < L0)) continue;
    const W src = kind ? (W)(w ^ mask) : w;           // zeros of src = the runs found
    const int L = kind ? L1 : L0;
    W r = kind ? r1 : r0;
    W mir = 0;
    if (reflect) {                                    // mirror image: bit i <-> bit n-1-i
      uint64_t t = (uint64_t)src;
#ifdef __CUDA_ARCH__
      t = __brevll(t) >> (64 - n);
#else
      t = reverse_bits_n(t, n);
#endif
      mir = (W)t;
    }
    while (r) {
      int p;
      if (BITS == 64) p = top_bit((uint64_t)r);
      else {
#ifdef __CUDA_ARCH__
        p = 31 - __clz((int)(uint32_t)r);
#else
        p = 31 - __builtin_clz((uint32_t)r);
#endif
      }
      r = (W)(r & ~((W)1 << p));
      int sh = n - 1 - p;                             // the run ends at bit p: bring p to the top
      W c = sh ? (W)(((src << sh) | (src >> (n - sh))) & mask) : src;
      best = c < best ? c : best;
      if (reflect) {                                  // in the mirror image the same run ends at bit n - 2 - p + L
        sh = p - L + 1;
        if (sh < 0) sh += n;
        c = sh ? (W)(((mir << sh) | (mir >> (n - sh))) & mask) : mir;
        best = c < best ? c : best;
      }
    }
  }
  return best;
}

// minimum over { rotate inside every k-bit block by a, rotate the R blocks by b }
__host__ __device__ __forceinline__ uint64_t min_rotation_blocks(const uint16_t *lut, const uint64_t *masks, int k,
                                                                 int R, int n, uint64_t mask, uint64_t w) {
  const uint32_t bm = (1u << k) - 1u;
  uint64_t pack_m = 0, pack_a = 0;          // per block: minimum rotation / set of amounts reaching it (k, R <= 8)
  uint32_t mstar = 0xffu;
  for (int y = 0; y < R; ++y) {
#ifdef __CUDA_ARCH__
    const uint32_t e = __ldg(lut + ((uint32_t)(w >> (k * y)) & bm));
#else
    const uint32_t e = lut[(uint32_t)(w >> (k * y)) & bm];
#endif
    pack_m |= (uint64_t)(e & 0xffu) << (8 * y);
    pack_a |= (uint64_t)(e >> 8) << (8 * y);
    mstar = (e & 0xffu) < mstar ? (e & 0xffu) : mstar;
  }
  uint64_t best = ~0ull;
  for (int y = 0; y < R; ++y) {
    if (((uint32_t)(pack_m >> (8 * y)) & 0xffu) != mstar) continue;
    uint32_t aset = (uint32_t)(pack_a >> (8 * y)) & 0xffu;
    const int sh = (R - 1 - y) * k;         // bring block y to the top
    while (aset) {
      const int a = low_bit(aset);
      aset &= aset - 1;
      const uint64_t wa = a ? (((w >> a) & masks[2 * a]) | ((w << (k - a)) & masks[2 * a + 1])) : w;
      const uint64_t c = rotl_n(wa, sh, n, mask);
      best = c < best ? c : best;
    }
  }
  return best;
}

// the same with a LUT over pairs of adjacent blocks; candidates are popped by bit index so that all lanes of a warp
// evaluate their (usually single) candidate together
__host__ __device__ __forceinline__ uint64_t min_rotation_pairs(const uint32_t *lut2, const uint64_t *masks, int k,
                                                                int R, int n, uint64_t mask, int div, uint64_t w) {
  const uint32_t bm = (1u << k) - 1u;
  uint64_t wy = w, wr = rotl_n(w, k, n, mask);   // block y of wr = block y - 1 of w: the block below the top one
  uint64_t cand = 0;                             // bit (k y + a): candidate "block y on top, rotated by a"
  uint32_t mstar = 0xffffffffu;
  for (int y = 0; y < R; ++y) {
    const uint32_t e = lut2[(((uint32_t)wy & bm) << k) | ((uint32_t)wr & bm)];
    const uint32_t m = e & 0xffffu;
    const uint64_t a = (uint64_t)(e >> 16) << (k * y);
    cand = m < mstar ? a : (m == mstar ? (cand | a) : cand);
    mstar = m < mstar ? m : mstar;
    wy >>= k;
    wr >>= k;
  }
  uint64_t best = ~0ull;
  while (cand) {
#ifdef __CUDA_ARCH__
    const int bit = __ffsll((long long)cand) - 1;
#else
    const int bit = __builtin_ffsll((long long)cand) - 1;
#endif
    cand &= cand - 1;
    const int y = (bit * div) >> 16, a = bit - y * k;
    const uint64_t wa = a ? (((w >> a) & masks[2 * a]) | ((w << (k - a)) & masks[2 * a + 1])) : w;
    const uint64_t c = rotl_n(wa, (R - 1 - y) * k, n, mask);
    best = c < best ? c : best;
  }
  return best;
}

// min over the block rotations of w AND of its spin-flipped image ~w: the blocks of ~w are the complements, so one
// extraction per block pair serves both look-ups
__host__ __device__ __forceinline__ uint64_t min_rotation_pairs_flip(const uint32_t *lut2, const uint64_t *masks, int k,
                                                                     int R, int n, uint64_t mask, int div, uint64_t w) {
  const uint32_t bm = (1u << k) - 1u, pm = (1u << (2 * k)) - 1u;
  uint64_t wy = w, wr = rotl_n(w, k, n, mask);
  uint64_t cand0 = 0, cand1 = 0;
  uint32_t m0 = 0xffffffffu, m1 = 0xffffffffu;
  for (int y = 0; y < R; ++y) {
    const uint32_t idx = (((uint32_t)wy & bm) << k) | ((uint32_t)wr & bm);
    const uint32_t e0 = lut2[idx], e1 = lut2[idx ^ pm];
    const uint32_t v0 = e0 & 0xffffu, v1 = e1 & 0xffffu;
    const uint64_t a0 = (uint64_t)(e0 >> 16) << (k * y), a1 = (uint64_t)(e1 >> 16) << (k * y);
    cand0 = v0 < m0 ? a0 : (v0 == m0 ? (cand0 | a0) : cand0);
    cand1 = v1 < m1 ? a1 : (v1 == m1 ? (cand1 | a1) : cand1);
    m0 = v0 < m0 ? v0 : m0;
    m1 = v1 < m1 ? v1 : m1;
    wy >>= k;
    wr >>= k;
  }
  // only the image(s) with the smaller top pair can hold the minimum
  uint64_t best = ~0ull;
  const uint64_t wf = w ^ mask;
  if (m1 < m0) cand0 = 0;
  if (m0 < m1) cand1 = 0;
  while (cand0 | cand1) {
    const bool flipped = cand0 == 0;
    uint64_t &cand = flipped ? cand1 : cand0;
#ifdef __CUDA_ARCH__
    const int bit = __ffsll((long long)cand) - 1;
#else
    const int bit = __builtin_ffsll((long long)cand) - 1;
#endif
    cand &= cand - 1;
    const uint64_t src = flipped ? wf : w;
    const int y = (bit * div) >> 16, a = bit - y * k;
    const uint64_t wa = a ? (((src >> a) & masks[2 * a]) | ((src << (k - a)) & masks[2 * a + 1])) : src;
    const uint64_t c = rotl_n(wa, (R - 1 - y) * k, n, mask);
    best = c < best ? c : best;
  }
  return best;
}


// min_g g(w) over the full space group of an R x k torus (see OrbitProgram::tor_mode).  An image of w is fixed by
//   t   : transpose first or not                       u = tau^t (w)
//   s,y : which row comes on top and whether the rows below it descend (s = 0: y, y-1, ...) or ascend (s = 1)
//   F   : the map applied to every row, F = flip^f . rho^e . rot_a
// and images compare lexicographically from the top row down, so the minimum has the smallest top PAIR of rows: pass 1
// looks the 2R (4R with tau) adjacent row pairs up in tor_lutm and keeps the set of pairs reaching the minimum, pass 2
// expands only those (about 1.3 images per state instead of |G|).
__host__ __device__ __forceinline__ uint64_t orbit_min_torus(const OrbitProgram &P, uint64_t w) {
  const int k = P.canon_k, R = P.canon_r, n = P.n_sites;
  const uint64_t mask = P.site_mask;
  const uint32_t bm = (1u << k) - 1u;
  uint64_t u1 = w;
  const int nt = P.tor_mode == 2 ? 2 : 1;
  if (nt == 2)
    for (int st = P.tor_rho_n; st < P.tor_rho_n + P.tor_tau_n; ++st) u1 = butterfly(u1, P.tor_net_mask[st], P.tor_net_delta[st]);
  uint32_t mstar = 0xffffffffu, cand = 0;   // cand bit (2 t + s) R + y
  uint32_t bit = 1u;
  for (int t = 0; t < nt; ++t) {
    const uint64_t u = t ? u1 : w;
    uint64_t wy = u;
    uint64_t wd = rotl_n(u, k, n, mask);        // block y of wd = block y - 1 of u
    uint64_t wu = rotl_n(u, n - k, n, mask);    // block y of wu = block y + 1 of u
    uint32_t bit_u = bit << R;
    for (int y = 0; y < R; ++y) {
      const uint32_t hi = ((uint32_t)wy & bm) << k;
      const uint32_t md = P.tor_lutm[hi | ((uint32_t)wd & bm)] & 0xffffu;
      const uint32_t mu = P.tor_lutm[hi | ((uint32_t)wu & bm)] & 0xffffu;
      cand = md < mstar ? bit : (md == mstar ? (cand | bit) : cand);
      mstar = md < mstar ? md : mstar;
      cand = mu < mstar ? bit_u : (mu == mstar ? (cand | bit_u) : cand);
      mstar = mu < mstar ? mu : mstar;
      wy >>= k; wd >>= k; wu >>= k;
      bit <<= 1; bit_u <<= 1;
    }
    bit <<= R;
  }
  uint64_t best = ~0ull;
  while (cand) {
#ifdef __CUDA_ARCH__
    const int cb = __ffs((int)cand) - 1;
#else
    const int cb = __builtin_ffs((int)cand) - 1;
#endif
    cand &= cand - 1;
    const int ts = (cb * P.tor_div_r) >> 16;   // (t, s) pair index = cb / R
    const int y = cb - ts * R, s = ts & 1;
    const uint64_t u = (ts >> 1) ? u1 : w;
    const int yn = s ? (y + 1 == R ? 0 : y + 1) : (y == 0 ? R - 1 : y - 1);
    const uint32_t idx = (((uint32_t)(u >> (k * y)) & bm) << k) | ((uint32_t)(u >> (k * yn)) & bm);
#ifdef __CUDA_ARCH__
    uint32_t S = __ldg(P.tor_luts + idx);
#else
    uint32_t S = P.tor_luts[idx];
#endif
    const int sh = (s ? y : R - 1 - y) * k;   // brings row y to the top (after the row order was reversed when s = 1)
    while (S) {
#ifdef __CUDA_ARCH__
      const int sb = __ffs((int)S) - 1;
#else
      const int sb = __builtin_ffs((int)S) - 1;
#endif
      S &= S - 1;
      const int fe = (sb * P.canon_div) >> 16, a = sb - fe * k, e = fe & 1;
      uint64_t v = (fe >> 1) ? (u ^ mask) : u;
      if (a) v = ((v >> a) & P.canon_masks[2 * a]) | ((v << (k - a)) & P.canon_masks[2 * a + 1]);
      if (e != s)                                            // rho alone, or sigma = (rho sigma) . rho
        for (int st = 0; st < P.tor_rho_n; ++st) v = butterfly(v, P.tor_net_mask[st], P.tor_net_delta[st]);
      if (s) v = reverse_bits_n(v, n);                       // rho sigma: reverse the whole word
      const uint64_t c = rotl_n(v, sh, n, mask);
      best = c < best ? c : best;
    }
  }
  return best;
}

// The same for a K x K torus with the transposition in the group (tor_mode == 2), on the word w and its transpose
// wt (the columns of w as rows): pass 1 is fully unrolled, 32-bit, with one shared-memory look-up per adjacent
// (row, row) / (column, column) pair, which gives the pair's minimum in both orders (2K look-ups in all).
// Both words are used with their rows repeated above bit n, uu = u | u << n (truncated to 64 bits), so that any K - 2
// or fewer consecutive rows, cyclically, are one shift and one mask: the pair j = (row j, row j+1) is bits K j ..
// K j + 2K - 1, i.e. the table index row(j+1) << K | row(j), whose entry holds
//   low half:  row j+1 on top, the rows below descending (s = 0)      high half: row j on top, ascending (s = 1)
// Candidate bit layout: bit t K + j for the low half of pair j of w (t = 0) or wt (t = 1), bit 16 + t K + j for the high.
// Pass 2 builds the image of a candidate row by row from tor_frow[F][row] (F = flip^f rho^e rot_a on one row): its top
// two rows are the minimal pair already, the other K - 2 are rows j+2, j+3, ..., j-1 (cyclically) in image order for
// s = 0 and in reverse image order for s = 1, byte look-ups on a 32-bit word -- no 64-bit networks.
// Column a of the lattice comes out of one masked multiply:
//   t = (w >> a) & STRIDE has site (y, a) at bit K y; t * CMUL puts it at bit S + y (S = (K-1)^2; no two partial
//   products meet, so there are no carries).
template <int K>
__host__ __device__ __forceinline__ uint32_t torus_sq_column(uint64_t w, int a) {
  constexpr uint32_t BM = (1u << K) - 1u;
  constexpr int S = (K - 1) * (K - 1);
  uint32_t stride = 0, cmul = 0;
#pragma unroll
  for (int y = 0; y < K; ++y) { stride |= 1u << (K * y); cmul |= 1u << ((K - 1) * (K - 1 - y)); }
  return ((((uint32_t)(w >> a) & stride) * cmul) >> S) & BM;
}

// The transposed lattice as a word: column a of w in bits K a .. K a + K - 1.  Transposition commutes with XOR, so the
// transpose of b ^ x is transpose(b) ^ transpose(x): a row of the product computes transpose(b) once and every term of
// the row only XORs in the transposed flip mask of its group (orbit_min_torus_sq_t).
template <int K>
__host__ __device__ __forceinline__ uint64_t torus_sq_columns(uint64_t w) {
  uint64_t t = 0;
#pragma unroll
  for (int a = 0; a < K; ++a) t |= (uint64_t)torus_sq_column<K>(w, a) << (K * a);
  return t;
}

// both 16-bit halves at once: the minimum of each half (VIMNMX.U16x2 on the device)
__host__ __device__ __forceinline__ uint32_t min_u16x2(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __vminu2(a, b);
#else
  const uint32_t lo = (a & 0xffffu) < (b & 0xffffu) ? (a & 0xffffu) : (b & 0xffffu);
  const uint32_t hi = (a >> 16) < (b >> 16) ? (a >> 16) : (b >> 16);
  return lo | hi << 16;
#endif
}

// min_g g(w) from w and its transpose wt = torus_sq_columns<K>(w) (layout above).  k_rows calls it per term: every term
// of a row is w = b ^ x for the row's state b and a group's flip mask x, so wt = transpose(b) ^ transpose(x) costs one
// XOR.  Exact for any flip mask x.  All 2K pairs are looked up, the unchanged ones too: the 32 lanes of a warp hold 32
// different rows at 32 different terms, so the pairs one lane could skip are pairs another lane needs, and the warp would
// issue every look-up anyway.
// Pass 1 handles both halves of a table entry together, in packed 16-bit minima (VIMNMX.U16x2 on the device): mstar is
// the minimum over every half, and with M1 = mstar + 1 in both halves, e_j = M1 - min(m2_j, M1) is 1 in a half equal to
// mstar and 0 in any other (no half is below mstar, so no borrow crosses halves).  The candidate set is
// sum_j e_j << j, taken as M1 sum_j 2^j - sum_j min(m2_j, M1) << j in 32-bit arithmetic: one packed minimum and one
// multiply-add per pair.
template <int K>
__host__ __device__ __forceinline__ uint64_t orbit_min_torus_sq_t(const OrbitProgram &P, uint64_t w, uint64_t wt) {
  constexpr int n = K * K;
  constexpr uint32_t BM = (1u << K) - 1u;
  constexpr uint32_t PM = (1u << (2 * K)) - 1u;
  constexpr int LOW = K * (K - 2);            // bits of the rows below the top pair
  static_assert(K * (K - 1) + LOW <= 64, "the rows below the top pair must lie inside the repeated word");
  const uint64_t uu0 = w | (w << n), uu1 = wt | (wt << n);
  const uint32_t *lutm = P.tor_lutm;
  uint32_t m2[2][K];
#pragma unroll
  for (int j = 0; j < K; ++j) {
    m2[0][j] = lutm[(uint32_t)(uu0 >> (K * j)) & PM];
    m2[1][j] = lutm[(uint32_t)(uu1 >> (K * j)) & PM];
  }
  uint32_t mm = m2[0][0];
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int j = 0; j < K; ++j)
      if (t + j > 0) mm = min_u16x2(mm, m2[t][j]);
  const uint32_t mstar = (mm & 0xffffu) < (mm >> 16) ? (mm & 0xffffu) : (mm >> 16);
  const uint32_t M1 = (mstar + 1u) * 0x00010001u;   // mstar <= PM < 2^12: mstar + 1 fits a half
  uint32_t cand = M1 * ((1u << (2 * K)) - 1u);
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int j = 0; j < K; ++j) cand -= min_u16x2(m2[t][j], M1) << (t * K + j);
  // pass 2
  const uint8_t *frow = P.tor_frow;
  uint32_t best = 0xffffffffu;   // rows below the top pair of the best image (the top pair is mstar for every candidate)
  while (cand) {
#ifdef __CUDA_ARCH__
    const int cb = __ffs((int)cand) - 1;
#else
    const int cb = __builtin_ffs((int)cand) - 1;
#endif
    cand &= cand - 1;
    const int s = cb >> 4, ty = cb & 15;
    const int t = ty >= K ? 1 : 0, j = ty - t * K;
    const uint64_t uu = t ? uu1 : uu0;
    const uint32_t c = (uint32_t)(uu >> (K * j)) & PM;           // row j+1 << K | row j
    const uint32_t idx = s ? ((c >> K) | ((c & BM) << K)) : c;   // top row << K | the row below it
#ifdef __CUDA_ARCH__
    uint32_t Sset = __ldg(P.tor_luts + idx);
#else
    uint32_t Sset = P.tor_luts[idx];
#endif
    const int jb = j + 2 >= K ? j + 2 - K : j + 2;
    const uint32_t below = (uint32_t)(uu >> (K * jb)) & ((1u << LOW) - 1u);   // rows j+2, ..., j-1: row j+2 lowest
    while (Sset) {
#ifdef __CUDA_ARCH__
      const int sb = __ffs((int)Sset) - 1;
#else
      const int sb = __builtin_ffs((int)Sset) - 1;
#endif
      Sset &= Sset - 1;
      const uint8_t *fr = frow + (sb << K);
      uint32_t img = 0;
#pragma unroll
      for (int q = 0; q < K - 2; ++q) {
        const uint32_t r = (below >> (K * q)) & BM;
        img |= (uint32_t)fr[r] << (s ? K * (K - 3 - q) : K * q);
      }
      best = img < best ? img : best;
    }
  }
  return ((uint64_t)mstar << LOW) | best;
}

// the same from w alone (the single-state entry point: self-checks, state_info, k_rows_batch)
template <int K>
__host__ __device__ __forceinline__ uint64_t orbit_min_torus_sq(const OrbitProgram &P, uint64_t w) {
  return orbit_min_torus_sq_t<K>(P, w, torus_sq_columns<K>(w));
}

__host__ __device__ __forceinline__ uint64_t translation_canon(const OrbitProgram &P, uint64_t w) {
  if (P.canon_mode == 2) return min_rotation_runs(w, P.n_sites, P.site_mask);
  if (P.canon_lut2)
    return min_rotation_pairs(P.canon_lut2, P.canon_masks, P.canon_k, P.canon_r, P.n_sites, P.site_mask, P.canon_div, w);
  return min_rotation_blocks(P.canon_lut, P.canon_masks, P.canon_k, P.canon_r, P.n_sites, P.site_mask, w);
}

// min_g g(s) through the canonical form of every coset representative (trivial characters)
__host__ __device__ __forceinline__ uint64_t orbit_min_canon(const OrbitProgram &P, uint64_t s) {
  if (P.tor_mode) return orbit_min_torus(P, s);
  if (P.canon_mode == 2 && P.chain_dihedral) {
    if (P.n_sites <= 32)
      return (uint64_t)min_rotation_dihedral<uint32_t>((uint32_t)s, P.n_sites, (uint32_t)P.site_mask, P.chain_dihedral == 2, P.has_flip);
    return min_rotation_dihedral<uint64_t>(s, P.n_sites, P.site_mask, P.chain_dihedral == 2, P.has_flip);
  }
  if (P.canon_mode == 2 && P.n_sites <= 32) {   // chains of up to 32 sites: everything in 32-bit registers
    const uint32_t site = (uint32_t)P.site_mask;
    uint32_t best32 = 0xffffffffu;
    for (int q = 0; q < P.n_q; ++q) {
      uint32_t cur = (uint32_t)s;
      const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
      for (int st = 0; st < P.n_stages; ++st) {
        const int d = P.benes_delta[st];
        const uint32_t t = ((cur >> d) ^ cur) & (uint32_t)bm[st];
        cur ^= t ^ (t << d);
      }
      uint32_t c = min_rotation_runs32(cur, P.n_sites, site);
      best32 = c < best32 ? c : best32;
      if (P.has_flip) {
        c = min_rotation_runs32(cur ^ site, P.n_sites, site);
        best32 = c < best32 ? c : best32;
      }
    }
    return (uint64_t)best32;
  }
  uint64_t best = ~0ull;
  if (P.cc_n > 0) {   // coset representatives as a chain of cheap steps
    uint64_t cur = s;
    for (int q = 0; q < P.cc_n; ++q) {
      for (int st = P.cc_begin[q]; st < P.cc_begin[q + 1]; ++st) cur = butterfly(cur, P.cc_mask[st], P.cc_delta[st]);
      if (P.canon_lut2 && P.has_flip) {
        const uint64_t c2 = min_rotation_pairs_flip(P.canon_lut2, P.canon_masks, P.canon_k, P.canon_r, P.n_sites,
                                                    P.site_mask, P.canon_div, cur);
        best = c2 < best ? c2 : best;
        continue;
      }
      uint64_t c = translation_canon(P, cur);
      best = c < best ? c : best;
      if (P.has_flip) {
        c = translation_canon(P, cur ^ P.site_mask);
        best = c < best ? c : best;
      }
    }
    return best;
  }
  for (int q = 0; q < P.n_q; ++q) {
    uint64_t cur = s;
    const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
    for (int st = 0; st < P.n_stages; ++st) cur = butterfly(cur, bm[st], P.benes_delta[st]);
    uint64_t c = translation_canon(P, cur);
    best = c < best ? c : best;
    if (P.has_flip) {
      c = translation_canon(P, cur ^ P.site_mask);
      best = c < best ? c : best;
    }
  }
  return best;
}

// representative only (characters trivial): picks the fastest applicable scan
__device__ __forceinline__ uint64_t orbit_representative(const OrbitProgram &P, uint64_t s);

// Scan the whole group.  COUNT_STAB additionally counts stabiliser elements (needs the full scan).
// EARLY_EXIT returns as soon as a candidate smaller than `s` is seen (is_representative test).
template <bool COUNT_STAB, bool EARLY_EXIT>
__host__ __device__ __forceinline__ OrbitResult orbit_scan(const OrbitProgram &P, uint64_t s) {
  OrbitResult out;
  out.rep = ~0ull;
  out.arg = 0;
  out.stab = 0;
  const int n_pairs = P.n_left + P.n_right;
  for (int q = 0; q < P.n_q; ++q) {
    uint64_t cur = s;
    const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
    for (int st = 0; st < P.n_stages; ++st) cur = butterfly(cur, bm[st], P.benes_delta[st]);
    for (int j = 0; j < P.n_t; ++j) {
      if (j > 0) {
        const uint64_t *sm = P.step_mask + (int64_t)(j - 1) * n_pairs;
        const int32_t *sh = P.step_shift + (int64_t)(j - 1) * n_pairs;
        uint64_t nxt = 0;
        for (int k = 0; k < P.n_left; ++k) nxt |= (cur << sh[k]) & sm[k];
        for (int k = P.n_left; k < n_pairs; ++k) nxt |= (cur >> sh[k]) & sm[k];
        cur = nxt;
      }
      uint64_t cand = cur;
      int flipped = 0;
      if (P.has_flip) {
        const uint64_t inv = cur ^ P.site_mask;
        if (COUNT_STAB) out.stab += (inv == s);
        if (inv < cur) { cand = inv; flipped = 1; }
      }
      if (COUNT_STAB) out.stab += (cur == s);
      if (cand < out.rep) {
        out.rep = cand;
        out.arg = (((q * P.n_t) + j) << 1) | flipped;
        if (EARLY_EXIT && cand < s) return out;
      }
    }
  }
  return out;
}

__device__ __forceinline__ uint64_t orbit_representative(const OrbitProgram &P, uint64_t s) {
  if (P.canon_mode) return orbit_min_canon(P, s);
  if (P.simple) return P.step_pack32 ? orbit_min_narrow(P, s) : orbit_min_wide(P, s);
  return orbit_scan<false, false>(P, s).rep;
}

// The fermionic exchange sign of element arg (an OrbitResult::arg) on the state s it is applied to: +1 or -1.  One load and
// one popcount per set bit of s; evaluated once per term, for the minimising element only.
__host__ __device__ __forceinline__ double orbit_sign(const OrbitProgram &P, int32_t arg, uint64_t s) {
  const uint64_t *M = reinterpret_cast<const uint64_t *>(P.characters + (int64_t)P.n_q * P.n_t * 2) +
                      (int64_t)(arg >> 1) * P.n_sites;
  uint32_t parity = 0;
  for (uint64_t b = s; b; b &= b - 1) {
#ifdef __CUDA_ARCH__
    parity += (uint32_t)__popcll(s & __ldg(M + (__ffsll((long long)b) - 1)));
#else
    parity += (uint32_t)__builtin_popcountll(s & M[__builtin_ctzll(b)]);
#endif
  }
  return (parity & 1u) ? -1.0 : 1.0;
}

// Full-precision stabiliser sum  sum_{g : g(s) = s} Re chi(g)  (only needed with non-trivial characters); FS (fermionic
// bases): sum_{g : g(s) = s} Re chi(g) sign(g, s), which vanishes on the orbits that are not basis states
template <bool FS = false>
__host__ __device__ inline double orbit_stabiliser_sum(const OrbitProgram &P, uint64_t s) {
  double acc = 0.0;
  const int n_pairs = P.n_left + P.n_right;
  for (int q = 0; q < P.n_q; ++q) {
    uint64_t cur = s;
    const uint64_t *bm = P.benes_mask + (int64_t)q * P.n_stages;
    for (int st = 0; st < P.n_stages; ++st) cur = butterfly(cur, bm[st], P.benes_delta[st]);
    for (int j = 0; j < P.n_t; ++j) {
      if (j > 0) {
        const uint64_t *sm = P.step_mask + (int64_t)(j - 1) * n_pairs;
        const int32_t *sh = P.step_shift + (int64_t)(j - 1) * n_pairs;
        uint64_t nxt = 0;
        for (int k = 0; k < P.n_left; ++k) nxt |= (cur << sh[k]) & sm[k];
        for (int k = P.n_left; k < n_pairs; ++k) nxt |= (cur >> sh[k]) & sm[k];
        cur = nxt;
      }
      const int64_t e = ((int64_t)q * P.n_t + j) * 2;
      if (FS && cur == s) acc += P.characters[e].x * orbit_sign(P, (int32_t)e, s);
      else if (cur == s) acc += P.trivial_characters ? 1.0 : P.characters[e].x;
      if (P.has_flip && (cur ^ P.site_mask) == s) acc += P.trivial_characters ? 1.0 : P.characters[e + 1].x;
    }
  }
  return acc;
}

}  // namespace dmv
