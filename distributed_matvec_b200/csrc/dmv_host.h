// dmv_host.h -- host-side declarations shared by the translation units of libdmv_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "dmv_device.cuh"

namespace dmv {

struct HostOrbitProgram {
  int32_t n_sites = 0, n_q = 0, n_stages = 0, n_t = 0, n_left = 0, n_right = 0;
  int32_t has_flip = 0, trivial_characters = 1;
  uint64_t site_mask = 0;
  int64_t group_order = 0;
  std::vector<uint64_t> benes_mask;
  std::vector<int32_t> benes_delta;
  std::vector<uint64_t> step_mask;
  std::vector<int32_t> step_shift;
  std::vector<double> characters;  // interleaved, [n_q][n_t][2][2]; fermionic: then the inversion masks' bits, [n_q][n_t][n_sites]
  int32_t fermionic = 0;
  std::vector<uint32_t> step_pack32;  // 4 words per step (empty unless simple and n_sites <= 32)
  std::vector<uint64_t> step_pack64;  // 3 words per step (empty unless simple)
  int32_t simple = 0;
  int32_t canon_mode = 0, canon_k = 0, canon_r = 0;   // block-rotation canonical form of the chain subgroup
  int32_t chain_dihedral = 0;
  std::vector<uint16_t> canon_lut;
  std::vector<uint64_t> canon_masks;
  std::vector<uint32_t> canon_lut2;      // pair LUT (empty: single-block LUT)
  int32_t canon_div = 0;
  std::vector<int32_t> cc_begin, cc_delta;   // coset chain of the canonical-form scan
  std::vector<uint64_t> cc_mask;
  int32_t tor_mode = 0, tor_rho_n = 0, tor_tau_n = 0, tor_div_r = 0;   // full-space-group canonical form of a torus
  std::vector<uint32_t> tor_lutm;
  std::vector<uint32_t> tor_luts;
  std::vector<uint8_t> tor_frow;
  std::vector<uint64_t> tor_net_mask;
  std::vector<int32_t> tor_net_delta;
  OrbitProgram view() const;       // pointers into the host vectors
};

// fermionic: n_sites counts the modes, and every element carries its inversion masks for the exchange sign
HostOrbitProgram compile_orbit_program(int n_sites, int64_t group_order, const int32_t *perms,
                                       const uint8_t *flips, const double *characters, bool fermionic = false);
// the states every orbit form is self-checked on: patterns with many tied images, then 256 seeded random words
std::vector<uint64_t> orbit_probe_states(uint64_t site_mask);
// orbit_min_torus_sq_t(s ^ x, transpose(s) ^ transpose(x)) == orbit_min_torus_sq(s ^ x) for every probe state s and
// flip mask x (host pointers in P; square torus with K = 4 or 6 only)
bool torus_sq_rows_check(const OrbitProgram &P, const std::vector<uint64_t> &flips);

// projection mode of the basis: which branch of BatchedOperator.computeOffDiag applies
// (reference src/BatchedOperator.chpl:89, 119, 163)
enum Projection { PROJ_NONE = 0, PROJ_INVERSION = 1, PROJ_GROUP = 2 };

// Everything a kernel needs, passed by value (fits the 4 KB kernel-parameter space).
struct KernelParams {
  // basis block of this rank
  StateIndex index;
  const double *norms;        // [n] (PROJ_GROUP only)
  // operator
  // (the host points these at the column-traversal (push) or row-traversal (pull) tables, see k_pull)
  const LutGroup *groups;  int32_t n_groups;
  const double *lut;       int32_t n_lut;     // real table (CV = false) or interleaved complex (CV = true)
  const OffTerm *terms;    int32_t n_terms;   // only read by groups with the generic flag
  int32_t any_generic, any_s_out;
  const BpWord *bp; int32_t n_bp;   // bit-parallel emit test (n_bp == 0: walk the groups one by one)
  uint64_t rank_total;        // INDEX_RANK: C(n_sites, weight)
  const DiagTerm *diag;    int32_t n_diag;       // all diagonal terms (n_diag > 0 <=> the operator has a diagonal)
  const DiagClass *diag_classes; int32_t n_diag_classes;   // bit-parallel part
  int32_t n_diag_rest;        // terms diag[0 .. n_diag_rest) are NOT covered by the classes (evaluated one by one)
  // symmetry
  OrbitProgram orbit;         // device pointers (PROJ_GROUP)
  uint64_t site_mask;
  double inversion_character; // PROJ_INVERSION: spin_inversion as a double
  // partition
  int32_t rank, num_ranks;
  // vectors
  const void *x; void *y;
  // outgoing buckets (num_ranks > 1): records for destination d go to out_betas + out_offset[d]
  uint64_t *out_betas; double *out_coeffs;
  const int64_t *out_offset;      // [num_ranks + 1] device
  unsigned long long *out_count;  // [num_ranks] device, reset before each generate
  // exact warp-private regions (num_ranks <= 32): the grid-stride tile loop is deterministic, so the
  // counting pass records how many records every warp emits per destination and the real pass starts
  // each warp at the prefix sum -- no slot-claim atomics, no slack, deterministic bucket layout.
  int32_t grid_blocks;              // 0: size the grid from occupancy; else exactly this many CTAs
  int32_t row_split;                // lanes sharing one source state (1, 2, 4, ... 32), see k_generate
  const int64_t *warp_offsets;      // [grid_blocks * 8][num_ranks]
  unsigned long long *warp_counts;  // counting pass output, same shape
  uint64_t *const *out_betas_ptr;   // [num_ranks]: base of MY region in the destination's record buffer
  double *const *out_coeffs_ptr;    //              (a local bucket, or the peer's incoming buffer over NVLink)
  const int64_t *out_capacity;      // [num_ranks]
  // emit_all: computeOffDiag mode -- every record goes to one flat output with its locale key
  int32_t emit_all; uint8_t *out_keys;
  // error reporting: status[0] = number of bad records, status[1] = first bad state, status[2] = overflow
  unsigned long long *status;
  // source range of this launch
  int64_t row_begin, row_end;
  // k_gather: the coefficient shared by every emitting (group, support bits) pair, when there is one
  double uni_re, uni_im;
  // k_gather / k_pull, replicated-x product (several ranks, every rank holds the whole basis and an all-gathered x):
  //   rows come from row_states (this rank's block) while `index` describes the GLOBAL basis; global index g lives
  //   at x[pos[g]]; the row's own element is x[x_row_offset + i].  All null / zero on one rank.
  const uint64_t *row_states;
  const double *row_norms;     // norms of the rows (k_pull on bases with permutation symmetries); `norms` is then global
  const uint32_t *pos;
  int64_t x_row_offset;
  // k_gather on several vectors at once: vector k of x / y starts batch_stride elements after vector k - 1
  int32_t gather_walk;         // k_gather: 0 per-lane walk from the top bit (default), 1 group-major, 2 per-lane from the bottom
  int32_t batch;               // 0 / 1: one vector; 4: four vectors per launch (k_gather); 2 .. 6: k_rows_batch
  int32_t batch_elt;           // k_rows_batch: doubles per vector element (1 | 2); batch * batch_elt <= 6
  int64_t batch_stride;
  // k_rows (row traversal of bases with permutation symmetries): hash table over the representatives with the scaled
  // vector element in the slot (see table_slot in dmv_device.cuh)
  const void *table;
  uint32_t table_slots;
  OrderedDir table_dir;        // ordered layout of `table` (rows_table = 1; see ordered_block), dir null: hashed layout
  // ... or, with a dense index: perfect hash -> slot of `dense` (32 bytes: {key, spare, re, im} / 16 bytes: {key, value});
  // `table` then only holds the few per cent of the states the two levels could not place
  PerfectHash mph;
  const void *dense;
  // ... or the dense ordered table (dord.blocks not null): rank blocks -> slot of `dense`, table_dir its directory
  DenseOrder dord;
  int32_t rows_ctas;           // k_rows: resident CTAs per SM the kernel is compiled for (-1 auto | 2 | 3 | 4)
  // k_rows on the ordered table: L2 eviction priorities (option rows_l2: 0 none | 1 far buckets and the row's own
  // accesses evict_first | 2 and near buckets evict_last); near = within rows_l2_window buckets of per_state * the row's rank
  // (the dense ordered table: slots of the row's rank, and its rank blocks take the near priority)
  int32_t rows_l2;
  uint32_t rows_l2_window, rows_l2_per_state;
};

// launchers (dmv_kernels.cu)
void launch_generate(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements,
                     bool count_only, cudaStream_t stream);
void launch_pull(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements,
                 cudaStream_t stream);
// row traversal without queue / atomics for bit-parallel operators on unprojected or inversion-only bases
void launch_gather(const KernelParams &p, bool inversion, bool complex_values, bool complex_elements,
                   bool narrow, bool lin, bool uniform, cudaStream_t stream);
// k_rows applies to real operators with a bit-parallel emit test on bases with trivial characters; returns the CTAs per
// SM the launch had resident
int launch_rows(const KernelParams &p, bool complex_elements, cudaStream_t stream);
// side of the square-torus orbit minimum k_rows is compiled for (4 | 6), 0: the generic orbit walk
int rows_torus_k(const OrbitProgram &o, bool dense, int rows_ctas);

// The term store of k_rows_stored (dmv_store.cu): every term k_rows accumulates, kept once per basis as a 32-bit entry
// (index of its target within its column block) | (code of its coefficient << kStoreIndexBits).  The basis' states are
// cut into `chunks` column blocks of block_states states; the entries are laid out block-major, and within a block by
// tile of 32 rows, row and k_rows' term order.  counts[k * n_rows + r] = entries of row r in block k, tile_off[k * n_tiles
// + t] = first entry of tile t in block k; row r's entries of block k follow those of the rows before it in its tile.
constexpr int kStoreIndexBits = 28;
constexpr int kStoreCodes = 16;          // 32 - kStoreIndexBits bits of coefficient code
constexpr int kStoreMaxChunks = 64;
struct RowsStoreView {
  uint32_t *entries;
  uint64_t *tile_off;
  uint8_t *counts;
  double *diag;                   // D(b) of every row (real operator), null without diagonal terms
  int64_t n_rows, n_tiles, block_states;
  int32_t chunks;
  double coef[kStoreCodes];       // the coefficient of every code
};
// build passes over rows [0, s.n_rows) of p (p.row_states, or the basis itself): count (counts, diag; flags[0] terms
// whose target is missing with c != 0, flags[1] a count past 255, flags[2] a coefficient without a code), then write
// (entries, from counts and tile_off)
void launch_store_build(const KernelParams &p, const RowsStoreView &s, bool write_pass, unsigned long long *flags,
                        cudaStream_t stream);
// tile sums of the counts (one per (block, tile), block-major) into tile_off[0 .. chunks * n_tiles); then the exclusive
// prefix sum over them, in place, with the total in tile_off[chunks * n_tiles]
void launch_store_offsets(const RowsStoreView &s, cudaStream_t stream);
// one pass of k_rows_stored over blocks [k0, k1) of rows [p.row_begin, p.row_end): the first pass starts each row's
// sum, the last one stores y as k_rows does; in between the sums wait in `partial` (one element per row)
void launch_rows_stored(const KernelParams &p, const RowsStoreView &s, const void *xs, void *partial, int k0, int k1,
                        bool complex_elements, cudaStream_t stream);
// hash table of k_rows: insert every state (slot_of[i] = its slot), then per product table[slot_of[i]] = x[src(i)] * norm[i]
// with src(i) = pos ? pos[i] : i
void launch_table_insert(const uint64_t *reps, int64_t n, void *table, uint32_t n_buckets, int slots_per_bucket,
                         uint32_t *slot_of, cudaStream_t stream, int bucket_bytes = 32, OrderedDir ord = OrderedDir{});
// directory of the ordered layout over the sorted representatives: ord.dir[0 .. ord.last + 1]
void launch_ordered_dir(const uint64_t *reps, int64_t n, OrderedDir ord, uint32_t buckets_per_state, cudaStream_t stream);
// k_rows on several vectors at once: 64-byte buckets { key, six doubles, spare } shared by the vectors of the batch
void launch_rows_batch(const KernelParams &p, cudaStream_t stream);
void launch_table_fill_batch(int64_t n, int num_vectors, int elt, const void *x, int64_t stride, const double *norms,
                             const uint32_t *slot_of, const uint64_t *reps, void *table, cudaStream_t stream);
// compact: the term store's scaled x instead (compact[i] = x[src(i)] * norm[i], 16 or 8 bytes in state order; slot_of,
// reps, table and dense unused)
void launch_table_fill(int64_t n, bool complex_elements, const void *x, const double *norms, const uint32_t *pos,
                       const uint32_t *slot_of, const uint64_t *reps, void *table, void *dense, cudaStream_t stream,
                       void *compact = nullptr);
// perfect-hash set-up (k_rows dense index): mark the positions of `n` states at a level in seen / collide bit arrays
// (192 bits per block, 3 words each), and compact the states whose position collided into `next`
void launch_mph_mark(const uint64_t *keys, int64_t n, int level, uint32_t n_blocks, unsigned long long *seen,
                     unsigned long long *collide, cudaStream_t stream);
void launch_mph_compact(const uint64_t *keys, int64_t n, int level, uint32_t n_blocks, const unsigned long long *collide,
                        uint64_t *next, unsigned long long *next_count, cudaStream_t stream);
// slot of every state: dense slot through the perfect hash, or 0x80000000 | (slot in the open-addressing table)
void launch_mph_slots(const uint64_t *keys, int64_t n, PerfectHash mph, const void *table, uint32_t n_buckets,
                      int slots_per_bucket, uint32_t *slot_of, unsigned long long *status, cudaStream_t stream);
void launch_accumulate(const KernelParams &p, Projection proj, bool complex_values, bool complex_elements,
                       int64_t count, const uint64_t *betas, const double *coeffs, cudaStream_t stream);
// plugin kernels (BO:217-275): diagonal coefficients / CSR list of off-diagonal terms of caller-given states
void launch_apply_diag(const KernelParams &p, int64_t count, const uint64_t *alphas, double *coeffs, cudaStream_t stream);
void launch_apply_off_diag(const KernelParams &p, int64_t count, const uint64_t *alphas, const int64_t *offsets,
                           int64_t *counts, uint64_t *betas, double *coeffs, bool write_pass, cudaStream_t stream);
void launch_build_directory(const uint64_t *reps, int64_t n, uint32_t *dir, uint64_t n_buckets, int shift,
                            cudaStream_t stream);
void launch_state_index(const StateIndex &ix, int64_t count, const uint64_t *spins, int64_t *indices,
                        cudaStream_t stream);
void launch_state_info(const OrbitProgram &P, Projection proj, uint64_t site_mask, double inv_char,
                       int64_t count, const uint64_t *alphas, uint64_t *betas, double *characters,
                       double *norms, cudaStream_t stream);
void launch_verify_rank(const StateIndex &ix, unsigned long long *status, cudaStream_t stream);
void launch_locale_idx(int64_t count, const uint64_t *states, int num_ranks, uint8_t *keys, cudaStream_t stream);
void launch_compute_norms(const OrbitProgram &P, int64_t count, const uint64_t *reps, double *norms,
                          cudaStream_t stream);
// enumeration: chunk c covers candidates [chunk_first[c], chunk_first[c] + chunk_len[c]) in the
// combinadic (fixed Hamming weight) or plain integer order; pass 0 counts, pass 1 writes.  half_mask != 0 keeps only
// the candidates with half_weight bits of half_mask set (the up half of a spinful-fermion basis).
void launch_enumerate(const OrbitProgram &P, Projection proj, uint64_t site_mask, bool fixed_hamming,
                      uint64_t half_mask, int half_weight, int rank, int num_ranks, int64_t n_chunks,
                      const uint64_t *chunk_first,
                      const uint64_t *chunk_last, unsigned long long *chunk_count,
                      const unsigned long long *chunk_offset, uint64_t *out, double *out_norms,
                      bool write_pass, cudaStream_t stream);
// replicated-x set-up: owner and position of every global state in the all-gathered x.
//   pass 0: chunk_counts[c * P + r] = states of chunk c owned by r;  pass 1: pos[g] = r * block + chunk_base[c * P + r] + k
// (owners from hash64_01(states[g]) % P, or from masks[g] when masks != nullptr)
void launch_owner_positions(const uint64_t *states, const uint8_t *masks, int64_t n, int num_ranks, int64_t chunk,
                            bool write_pass, unsigned long long *chunk_counts, const unsigned long long *chunk_base,
                            int64_t block, uint32_t *pos, cudaStream_t stream);
// out[pos[i]] = in[i] (gather == false) or out[i] = in[pos[i]]; elt = 8-byte words per element (1 or 2)
void launch_permute(int64_t n, int elt, const uint32_t *pos, const void *in, void *out, bool gather, cudaStream_t stream);
// peer-direct all-gather of x (replicated-x product): my block into slot `rank` of every rank's gathered vector over
// NVLink, then my flag in every peer; the consumer waits for all flags of the epoch
void launch_push_block(const void *x, int64_t n_doubles, int num_ranks, void *const *peer_slot, unsigned *done,
                       unsigned *const *peer_flags, int rank, unsigned epoch, bool wide, cudaStream_t stream);
void launch_raise_flags(unsigned *const *peer_flags, int num_ranks, int rank, unsigned value, cudaStream_t stream);
void launch_wait_flags(const unsigned *flags, int num_ranks, unsigned epoch, unsigned long long *status,
                       cudaStream_t stream);
// Lanczos vector kernels (dmv_solver.cu); n = elements, words = 8-byte words.  Every launcher of dmv_solver.cu but
// launch_reduce_partials returns the CTAs of its main launch (0 when it launched nothing).
int launch_dot(int64_t n, bool complex_elements, const double *a, const double *b, double *out2, cudaStream_t s);
int launch_lanczos_update(int64_t n, bool complex_elements, double *w, const double *v, const double *u,
                          const double *coef2, double *out1, cudaStream_t s);
int launch_scale(int64_t words, double scale, const double *x, double *y, bool accumulate, cudaStream_t s);
int launch_fill(int64_t words, uint64_t seed, uint64_t offset, double *x, cudaStream_t s);
// Krylov block kernels (dmv_solver.cu, used by dmv_expm_multiply): the stored vectors travel as a kernel parameter
constexpr int kMaxBlockVectors = 65;
struct VecList { const double *p[kMaxBlockVectors]; };
// CTAs of the largest block launch over n elements: `partials` must hold that many * (J + 1) * 2 doubles
int block_partials_grid(int64_t n, bool complex_elements);
// h[2k], h[2k + 1] = <V_k, w> for k < J (real vectors: imaginary part 0), h[2J] = |w|^2; w is read once
int launch_block_dot(int64_t n, bool complex_elements, const VecList &V, int J, const double *w, double *partials,
                     double *h, cudaStream_t s);
// out = a w - sum_{k < J} c_k V_k (c: J interleaved complex coefficients in device memory; w may be null, out may alias
// w), nrm2[0] = |out|^2
int launch_block_combine(int64_t n, bool complex_elements, double a, const double *w, const VecList &V, int J,
                         const double *coef, double *out, double *partials, double *nrm2, cudaStream_t s);
// Block kernels of dmv_eigsh: W = R <= kMaxBlockRhs vectors, w_stride elements apart; V and W are read once per call.
constexpr int kMaxBlockRhs = 6;
// doubles the `partials` buffer of launch_block_gram / launch_block_update must hold
size_t block_gram_partials();
// h[2 (k R + r) + {0, 1}] = <V_k, W_r> for k < J, h[2 (J R + r R + s) + {0, 1}] = <W_r, W_s> (real vectors: imaginary 0)
int launch_block_gram(int64_t n, bool complex_elements, const VecList &V, int J, const double *W, int64_t w_stride,
                      int R, double *partials, double *h, cudaStream_t s);
// W_r -= sum_{k < J} c_{kr} V_k (c[2 (k R + r) + {0, 1}] in device memory), nrm2[2 r] = |W_r|^2 after
int launch_block_update(int64_t n, bool complex_elements, const VecList &V, int J, const double *coef, double *W,
                        int64_t w_stride, int R, double *partials, double *nrm2, cudaStream_t s);
// in place V_j <- sum_{i < k} S_{ij} V_i for j < l <= k (S[2 (i l + j) + {0, 1}] in device memory); no second basis
int launch_block_rotate(int64_t n, bool complex_elements, const VecList &V, int k, int l, const double *S,
                        cudaStream_t s);
// out[2k + {0, 1}] = sum over b < blocks of partials[(b * width + k) * 2 + {0, 1}], in a fixed order (k_reduce_partials)
void launch_reduce_partials(int blocks, int width, const double *partials, double *out, cudaStream_t s);
// Kernels of dmv_lanczos_quadrature (dmv_solver.cu): G <= kMaxBlockRhs recurrences, vector g at offset g n elements.
// The recurrence of a vector breaks down at step t + 1 when beta_{t+1} = sqrt(b2_next) <= 1e-14 max(1, |alpha_t|) with
// alpha_t = dot / b2 (b2 = |r_t|^2): one expression, evaluated alike by the device and the host.
__host__ __device__ inline bool quad_breakdown(double b2_next, double dot, double b2) {
  return sqrt(b2_next) <= 1e-14 * fmax(1.0, fabs(dot / b2));
}
// doubles the `partials` buffer of launch_quad_dot / launch_quad_update must hold for G vectors
size_t quad_partials(int G);
// x[g n + i] = seeded start value of vector first + g at representative reps[i], g < G
int launch_quad_fill(int64_t n, bool complex_elements, const uint64_t *reps, uint64_t seed, int first, int G,
                     double *x, cudaStream_t s);
// out[2 g + {0, 1}] = <A_g, B_g> (A may equal B)
int launch_quad_dot(int64_t n, bool complex_elements, int G, const double *A, const double *B, double *partials,
                    double *out, cudaStream_t s);
// step j: P <- r_{j+1} from P = r_{j-1}, Q = r_j, W = H r_j and the stored dot / b2 of steps j - 1 and j;
// nrm2[2 g] = |r_{j+1}|^2
int launch_quad_update(int64_t n, bool complex_elements, int G, double *P, double *Q, const double *W,
                       const double *dot, const double *b2, int j, double *partials, double *nrm2, cudaStream_t s);
// Spin-spin Gram block of dmv_zz_correlations (dmv_observe.cu): gram[i * zz_gram_columns + j] = sum_b |x_b|^2 a_i s_j
// with s_j = +-1 for bit j of reps[b] and a = (s, 1); zz_gram_size doubles (rows padded to 16, columns to 8).
// `partials` must hold zz_gram_partials(n, n_sites) doubles.
int zz_gram_columns(int n_sites);
size_t zz_gram_size(int n_sites);
size_t zz_gram_partials(int64_t n, int n_sites);
void launch_zz_gram(int64_t n, bool complex_elements, int n_sites, const uint64_t *reps, const double *x,
                    double *partials, double *gram, cudaStream_t s);
int64_t launch_counter();
int planned_grid(int64_t rows, int row_split);
int choose_row_split(int64_t rows, int n_groups);
constexpr int kWarpsPerCta = 8;

// ---- launch helpers of every launcher (dmv_kernels.cu defines sm_count and check_launch) ----------------------------
#define CUDA_CHECK(expr)                                                                        \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e));            \
  } while (0)

// streaming multiprocessors of the current device (queried once per device ordinal)
int sm_count();
// after every launch: a launch error names the kernel, and the launch is counted once (launch_counter)
void check_launch(const char *what);

// `work_ctas` CTAs' worth of work, at least one (so that an empty launch still writes its partials), at most max_ctas
inline int capped_grid(int64_t work_ctas, int64_t max_ctas) {
  return (int)std::min<int64_t>(std::max<int64_t>(work_ctas, 1), max_ctas);
}

// let `kernel` have `smem` bytes of dynamic shared memory: launches above 48 KB need the opt-in
template <typename K>
void opt_in_smem(K kernel, size_t smem) {
  if (smem > 48 * 1024)
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      throw std::runtime_error("cannot opt in to " + std::to_string(smem) + " bytes of shared memory");
}

// CTAs of `kernel` (`threads` each, `smem` bytes of dynamic shared memory) that are resident on one SM at once
template <typename K>
int resident_ctas(K kernel, size_t smem = 0, int threads = 32 * kWarpsPerCta) {
  opt_in_smem(kernel, smem);
  int per_sm = 0;
  CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
  return per_sm;
}

// one wave of resident CTAs of `kernel` over `ctas` CTAs' worth of work
template <typename K>
int one_wave(K kernel, int64_t ctas, size_t smem = 0, int threads = 32 * kWarpsPerCta) {
  return capped_grid(ctas, (int64_t)sm_count() * std::max(resident_ctas(kernel, smem, threads), 1));
}

// f(std::integral_constant<bool, B>) for the runtime flag b
template <typename F>
auto with_bool(bool b, F &&f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}

// f(std::integral_constant<int, V>) for the V of the list equal to v; a value outside the list has no kernel instance
template <int V, int... Rest, typename F>
auto with_choice(int v, F &&f) {
  if (v == V) return f(std::integral_constant<int, V>{});
  if constexpr (sizeof...(Rest) > 0) return with_choice<Rest...>(v, f);
  else throw std::runtime_error("no kernel instance for the value " + std::to_string(v));
}

}  // namespace dmv
