/*
 * dmv_b200.h -- C ABI of libdmv_b200.so: the distributed matrix-free H.x hot path for Hopper (sm_90a).
 *
 * This is the drop-in boundary for the reference's hot path (SURVEY.md section 8b).  Plain pointers
 * and sizes only; no torch / C++ types.  Every entry point names the reference interface it replaces.
 * All functions returning int return 0 on success and a non-zero code on failure, with a message
 * available from dmv_last_error() (the reference halts instead: src/DistributedMatrixVector.chpl:116,
 * 1099-1102; the ls_chpl_* wrappers below abort() on failure to stay drop-in).
 *
 * Threading: one context per GPU; a context is not thread-safe; dmv_matvec() is collective over the
 * ranks of the communicator (like the reference's allLocalesBarrier use, DMV:895,954,1013).
 */
#ifndef DMV_B200_H
#define DMV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dmv_context dmv_context;

/* Element type of x / y.  The reference's vectors are real(64) (DMV:1095-1096); complex128 is the
 * extension BASELINE.json asks for. */
enum { DMV_F64 = 1, DMV_C128 = 2 };

/* Flat description of a spin basis: the visible part of `ls_hs_basis` (reference src/FFI.chpl:94-105)
 * plus the symmetry group the third-party library keeps opaque.  Group element g maps a state s to
 * g.s with (g.s) bit i = s bit perms[g*number_sites + i], followed by a global spin flip when
 * flips[g] != 0.  characters are interleaved (re, im).  group_order == 0: no projection. */
typedef struct {
  int32_t number_sites;      /* <= 64 (DMV:1099: numberWords == 1) */
  int32_t hamming_weight;    /* -1: not fixed */
  int32_t spin_inversion;    /* 0, +1, -1 */
  int32_t has_permutations;  /* basis.hasPermutationSymmetries(), src/ForeignTypes.chpl:96-98 */
  int64_t group_order;       /* all elements, including the inversion-doubled ones */
  const int32_t *perms;
  const uint8_t *flips;
  const double *characters;
} dmv_basis_desc;

/* Flat non-branching term tables: <beta|t|alpha> = v [alpha & m == r] (-1)^popcount(alpha & s),
 * beta = alpha ^ x (the content of `ls_hs_nonbranching_terms`, reference src/FFI.chpl:109-113, whose
 * tail is opaque there).  v interleaved (re, im).  Diagonal terms have x == 0 and carry no x array. */
typedef struct {
  int64_t n_off;
  const double *off_v;
  const uint64_t *off_m, *off_r, *off_x, *off_s;
  int64_t n_diag;
  const double *diag_v;
  const uint64_t *diag_m, *diag_r, *diag_s;
} dmv_operator_desc;

/* ---- library lifetime: replaces ls_chpl_init / ls_chpl_finalize (reference src/library.c:19-34) */
void ls_chpl_init(void);
void ls_chpl_finalize(void);
const char *dmv_last_error(void);
int dmv_version(void);
/* number of kernel launches issued by this library since load (evidence for bench.py's gpu_launches) */
int64_t dmv_launch_count(void);

/* ---- context: replaces the per-call setup of matrixVectorProduct (DMV:1077-1084: operator clone,
 * uncheckedSetRepresentatives) and of localOffDiagonalNoQueue (DMV:864-955: buffers, pointer wiring)
 * with a persistent object.  `device` is the CUDA device ordinal; rank / num_ranks define the hash
 * partition  owner(s) = hash64_01(s) % num_ranks  (reference src/StatesEnumeration.chpl:122-136). */
int dmv_context_create(const dmv_basis_desc *basis, const dmv_operator_desc *op, int device, int rank,
                       int num_ranks, dmv_context **out);
int dmv_context_destroy(dmv_context *ctx);
/* launch on `cuda_stream` (a cudaStream_t; NULL is the legacy default stream), or on the context's own
 * non-blocking stream when use_own_stream != 0 (the initial state) */
int dmv_set_stream(dmv_context *ctx, void *cuda_stream, int use_own_stream);
int dmv_synchronize(dmv_context *ctx);
/* options (a value outside those listed raises and leaves the option unchanged; every option also applies to the
 * whole-basis context of the replicated-x product, whether set before or after that context exists):
 *          "mode"     = -1 auto (row traversal on one rank when a row kernel applies -- k_gather: bit-parallel operator on a
 *                        basis without permutation symmetries; k_rows: real bit-parallel operator on a basis with
 *                        permutation symmetries and trivial characters -- else push) | 0 push: scatter with FP64
 *                        atomics, the reference's traversal (DMV:73-127) | 1 rows (k_gather / k_rows, else the queued
 *                        k_pull); one rank only
 *          "gather"   = -1 auto | 0 use the queued k_pull instead of k_gather when "mode" selects rows
 *          "rows"     = -1 auto | 0 use the queued k_pull instead of k_rows
 *          "rows_index" = -1 auto, 0 open-addressing table with the vector element in the slot | 1 dense table behind a
 *                        two-level perfect hash (5 bits per state; measured slower, kept for reference)
 *          "rows_table" = 1 (default) open-addressing table of k_rows laid out by key prefix, so that the look-ups of
 *                        neighbouring rows share L2 | 0 homes hashed over the whole table (the perfect hash's leftover
 *                        states always use hashed homes)
 *          "rows_table_bits" = 1 .. 14 (default 12): the ordered layout's directory has at most 2^bits blocks (4 bytes
 *                        each, staged in the shared memory of every CTA of k_rows: at 2^14 only two CTAs fit an SM on
 *                        the 6x6 square)
 *          "rows_table_buckets" = 2 | 4 | 8 (default 8): complex128 buckets per state of the ordered layout
 *          "rows_dense_order" = -1 auto (on wherever "rows_table" = 1) | 0 off | 1 on: instead of the ordered layout, the
 *                        dense ordered table -- one slot per state in key order at the granularity of the ordered
 *                        layout's blocks ("rows_table_bits"), found through a perfect hash per rank block of 40 states
 *                        (32 bytes each, L2-resident); "rows_index" = 1 takes precedence.  Info: "rows_dense_order_on"
 *                        whether it is built, "rows_dense_order_placed" the states its hash levels place ("rows_dense"
 *                        counts the states of the perfect-hash index only)
 *          "rows_l2" = 0 | 1 | 2 (default): L2 eviction priority of k_rows' accesses on the ordered layouts, per
 *                        instruction (nothing device-wide is set).  1: evict_first for the buckets / slots farther than
 *                        "rows_l2_window" = 0 .. 32 (default 2) MB of table from the row's own place, and for the row's
 *                        state, norm, x and y; 2: and evict_last for the nearer buckets / slots and the dense ordered
 *                        table's rank blocks; 0: none.  y does not depend on it
 *          "rows_ctas" = -1 auto (default) | 2 | 3 | 4 CTAs per SM k_rows is compiled for (k_rows_batch and the perfect-hash
 *                        index: always 2) (registers per thread 106-128 | 80 | 64).  Auto: 3 with the square-torus
 *                        forms of the orbit minimum, whose 3-CTA builds spill nothing more, when the occupancy query
 *                        finds 3 resident, else 2; 2 with the generic orbit walk, whose 3-CTA build spills ~100 bytes of
 *                        the pipeline state.  Info "rows_ctas_resident": the CTAs per SM the last k_rows launch had
 *                        resident (a build for more CTAs than fit runs with fewer, and slower)
 *          "rows_batch" = -1 auto, 1: dmv_matvec_batch on bases with permutation symmetries takes up to six doubles per
 *                        state (six real / three complex vectors) through k_rows_batch | 0 vector by vector;
 *                        "rows_batch_min" = doubles per state (vectors x element width, default 2) from which it is used
 *          "gather_walk" = 0 every lane walks its emitting groups from the top bit | 1 group-major warp-uniform walk
 *                        (measured slower; only at row split 1, else walk 0) | 2 from the bottom bit (round 1)
 *          "gather_split" = -1 auto (more lanes per row of k_gather on bases of fewer than 16 warps of rows per SM, never
 *                        more lanes than flip-mask groups) | 1, 2, 4, 8, 16 or 32 lanes per row, each walking every
 *                        S-th group.  Applies to the single, batched and replicated-x products
 *          "push_split" = -1 auto (the same rule over the scatter tables) | 1, 2, 4, 8, 16 or 32 lanes per source state
 *                        of k_generate, each taking every S-th flip-mask group (only slice 0 adds the diagonal).  Applies
 *                        to the scatter product and its counting pass (dmv_plan); a change re-plans.  The overlapped
 *                        rounds of the record exchange always run S = 1
 *          "index"    = -1 auto (identity / Lin tables / directory) | 0 directory + binary search | 2 combinadic rank
 *                        | 3 Lin tables (full fixed-Hamming bases)
 *          "bitparallel" = 1 | 0 walk the flip-mask groups one by one
 *          "canon"    = -1 auto (orbit minima through canonical forms: full space group of a torus, rotations x mirror x
 *                        flip of a chain) | 1 the round-1 forms (block rotations + coset chain; four run searches)
 *                        | 2 single-block LUT + independent networks | 0 walk the chain of group elements
 *          "exchange" = -1 auto (replicated x when the whole basis fits, else peer-direct records, else NCCL buckets)
 *                        | 0 NCCL send/recv of record buckets | 1 peer-direct records over NVLink | 2 replicated x
 *          "peer_gather" = -1 auto (replicated x: all-gather of x as peer-direct NVLink stores + flags) | 0 ncclAllGather
 *          "rounds"   = -1 auto (peer-direct records in 4 overlapped rounds for blocks of >= 2^18 states) | 0, 1 one shot
 *                        (generate everything, fence, accumulate) | R <= 64 rounds
 * dmv_get_info: "index_mode", "pull", "gather", "rows", "rows_ok", "projection", "n_groups", "orbit_n_q", "orbit_n_t",
 *               "canon_mode", "torus_mode", "peer_direct", "replicated", "replicated_block", "peer_gather", "rounds",
 *               "global_states", "complex_coefficients", "quadrature_group", "rows_tk" (side of the square-torus orbit minimum k_rows is
 *               compiled for with the current options: 4 | 6, 0 the generic walk), "gather_split" (lanes per row the next
 *               single-rank k_gather launch uses), "push_split" (lanes per source state the next k_generate launch and
 *               its plan use), ... (-1: unknown); "global.<key>" answers <key> for the whole-basis
 *               context of the replicated-x product (-1 while there is none) */
int dmv_set_option(dmv_context *ctx, const char *name, int64_t value);
int64_t dmv_get_info(const dmv_context *ctx, const char *name);

/* ---- basis
 * dmv_basis_build: replaces Basis.build() / enumerateStates for this rank (reference
 *   src/ForeignTypes.chpl:72, src/StatesEnumeration.chpl:516-603): enumerates on the GPU the ascending
 *   representatives owned by this rank and their norms, and installs them.
 * dmv_set_representatives: replaces Basis.uncheckedSetRepresentatives (src/ForeignTypes.chpl:74-77,
 *   DMV:1084).  `representatives` must be ascending and owned by this rank; `norms` may be NULL (they
 *   are then computed on the GPU when the basis needs them).  Host or device pointers.
 * dmv_get_representatives copies them out (host or device destination); pass NULL to query the count. */
int dmv_basis_build(dmv_context *ctx);
int dmv_set_representatives(dmv_context *ctx, const uint64_t *representatives, int64_t count,
                            const double *norms);
int64_t dmv_number_states(const dmv_context *ctx);
int dmv_get_representatives(dmv_context *ctx, uint64_t *representatives, double *norms);

/* ---- third-party kernels the path consumes, now on the GPU (host or device pointers)
 * dmv_state_index: ls_hs_state_index (reference src/FFI.chpl:173-175; call DMV:102); -1 when absent.
 * dmv_state_info:  ls_hs_state_info  (src/FFI.chpl:181-184; call src/BatchedOperator.chpl:188-194).
 * dmv_locale_idx_of: localeIdxOf     (src/StatesEnumeration.chpl:129-136). */
int dmv_state_index(dmv_context *ctx, int64_t count, const uint64_t *spins, int64_t *indices);
int dmv_state_info(dmv_context *ctx, int64_t count, const uint64_t *alphas, uint64_t *betas,
                   double *characters, double *norms);
int dmv_locale_idx_of(dmv_context *ctx, int64_t count, const uint64_t *states, int num_locales,
                      uint8_t *keys);

/* ---- BatchedOperator.computeOffDiag (reference src/BatchedOperator.chpl:82-213)
 * Generates, for alphas[0..count) with values xs, the flat list (betas, coeffs, keys) after
 * projection; *n receives the number of entries.  Output arrays must hold count * max_off_diag
 * entries (dmv_max_number_off_diag).  Entry ORDER is unspecified (the reference's is row-major;
 * consumers only bucket and accumulate).  coeffs interleaved complex128.  Host or device pointers. */
int64_t dmv_max_number_off_diag(const dmv_context *ctx);
int dmv_compute_off_diag(dmv_context *ctx, int64_t count, const uint64_t *alphas, const void *xs,
                         int elt, int64_t *n, uint64_t *betas, double *coeffs, uint8_t *keys);

/* ---- the hot path
 * dmv_local_matvec: localMatrixVector(matrix, x, y, representatives) (DMV:1055-1070) on this rank's
 *   block when num_ranks == 1.  y = D x + O x if the operator has diagonal terms, else y += O x
 *   (DMV:1062-1069: without diagonal terms y is not cleared).  x, y: host or device pointers of
 *   dmv_number_states() elements of type `elt`.
 * dmv_matvec: matrixVectorProduct (DMV:1072-1093), collective over the communicator: generation,
 *   hash bucketing, all-to-all exchange (peer-direct NVLink stores or NCCL) and owner-side search +
 *   accumulate -- or the replicated-x form below when it applies. */
int dmv_local_matvec(dmv_context *ctx, int elt, const void *x, void *y);
int dmv_matvec(dmv_context *ctx, int elt, const void *x, void *y);

/* ---- stepwise form of the distributed product, for hosts that own the exchange themselves (a Chapel
 * host with GASNet PUTs as in DMV:361-371, torch.distributed, or several logical ranks on one GPU):
 *   dmv_plan:      one counting pass; fills send_counts[num_ranks] (records this rank emits for each
 *                  destination in one product; the own entry is processed locally and reported too).
 *   dmv_generate:  y (+)= D x; emits all records; own bucket is searched + accumulated into y at once,
 *                  the others are left in the context's outgoing buckets.
 *   dmv_outgoing:  device pointers + count of the bucket for `dest` (valid until the next generate).
 *   dmv_accumulate: localProcess (DMV:73-127) on `count` received records (device or host pointers):
 *                  y[index(beta)] += coeff (* norm).  A record that is non-zero and not in the basis
 *                  is an error (DMV:115-118). */
int dmv_plan(dmv_context *ctx, int64_t *send_counts);
int dmv_generate(dmv_context *ctx, int elt, const void *x, void *y);
int dmv_outgoing(dmv_context *ctx, int dest, const uint64_t **betas, const double **coeffs,
                 int64_t *count);
int dmv_accumulate(dmv_context *ctx, int elt, int64_t count, const uint64_t *betas,
                   const double *coeffs, void *y);

/* ---- replicated-x form of the distributed product (alternative to the record exchange of DMV:313-436,
 * chosen automatically by dmv_matvec -- option "exchange" = -1 / 2 -- when the whole basis fits on one device): every
 * rank keeps the whole sorted basis, x is all-gathered (E bytes per state instead of 8 + E bytes per off-diagonal term
 * over NVLink) into slots of dmv_get_info(ctx, "replicated_block") elements per rank, and each rank computes ITS rows by
 * the row traversal (k_gather, or the queued k_pull for bases with permutation symmetries): no records, no atomics on y.
 * The hash partition of x, y and the representatives seen by the caller (SE:129-156) is unchanged.
 * Inside dmv_matvec the all-gather of x is one kernel of peer-direct NVLink stores into the CUDA-IPC-mapped gathered
 * vectors of all ranks plus release / acquire flags (option "peer_gather"; ncclAllGather when IPC mapping is impossible).
 * Bases with permutation symmetries run k_rows on a hash table over the whole basis, refilled from the gathered x.
 *   dmv_replicated_setup:   local set-up (whole basis, slot table); no communication.
 *   dmv_replicated_product: y <- rows of this rank applied to a caller-assembled gathered x (device pointers); for
 *                           hosts that own the all-gather themselves (several logical ranks on one GPU, tests). */
int dmv_replicated_setup(dmv_context *ctx);
int dmv_replicated_product(dmv_context *ctx, int elt, const void *x_cat, void *y);

/* ---- block <-> hashed redistribution of vectors (arrFromBlockToHashed, reference src/BlockToHashed.chpl:87-208;
 * arrFromHashedToBlock, src/HashedToBlock.chpl:67-153): how vectors in file (sorted-state) order enter and leave the
 * hash partition (test/TestMatrixVectorProduct.chpl:35,45).  "Block": the global array cut into contiguous chunks,
 * one per rank, with masks[i] = owner of element i (SE:138-156); "hashed": each rank holds the elements it owns,
 * ascending.  elt = 8-byte words per element (1: real(64) / uint(64), 2: complex128).  Host or device pointers.
 *   dmv_hashed_positions: positions[i] = slot of chunk element i in the ordering "grouped by owner, stable";
 *                         counts[r] = elements owned by r.  Building block of the two conversions.
 *   dmv_permute:          out[positions[i]] = in[i] (gather == 0) or out[i] = in[positions[i]] (gather != 0).
 *   dmv_block_to_hashed / dmv_hashed_to_block: the conversions, collective over the communicator (NCCL
 *                         all-to-all-v of the grouped chunks); with one rank they are the permutation alone. */
int dmv_hashed_positions(dmv_context *ctx, int64_t count, const uint8_t *masks, int num_ranks, int64_t *counts,
                         uint32_t *positions);
int dmv_permute(dmv_context *ctx, int elt, int64_t count, const uint32_t *positions, const void *in, void *out,
                int gather);
int dmv_block_to_hashed(dmv_context *ctx, int elt, int64_t chunk_count, const uint8_t *masks_chunk,
                        const void *block_chunk, void *hashed, int64_t hashed_count);
int dmv_hashed_to_block(dmv_context *ctx, int elt, int64_t chunk_count, const uint8_t *masks_chunk,
                        const void *hashed, int64_t hashed_count, void *block_chunk);

/* ---- communicator (NCCL over NVLink): 128-byte unique id made on rank 0, shared by the host */
int dmv_comm_unique_id(void *id128);
int dmv_comm_init(dmv_context *ctx, const void *id128);

/* ---- several vectors per call: numVectors > 1 of ls_chpl_matrix_vector_product, which the reference itself does not
 * implement (DMV:1101-1102 halts; its eigensolver loops over columns, src/Diagonalize.chpl:154-158).  x, y hold
 * num_vectors vectors of dmv_number_states elements one after the other (the [numVectors, N] layout of BlockVector).
 * On one rank: with device pointers and an operator k_gather applies to, four vectors at a time share the term walk and the
 * index look-ups; on bases with permutation symmetries (k_rows) up to six doubles per state -- six real or three complex
 * vectors -- share the orbit minimum and ONE 64-byte look-up per term (k_rows_batch; host vectors are staged a batch at a
 * time).  Everything else is the loop over dmv_local_matvec / dmv_matvec.  Semantics per vector as for a single product.
 * (The ls_chpl_* entry keeps the reference's behaviour and halts for numVectors != 1.) */
int dmv_matvec_batch(dmv_context *ctx, int elt, int num_vectors, const void *x, void *y);

/* ---- Lanczos ground state on the device ("next" row f3; the reference gives its product to PRIMME as the matvec
 * callback, src/Diagonalize.chpl:134-225).  Three-term recurrence with the vectors resident in HBM, dot products reduced
 * over the ranks with NCCL; converged when |beta_k s_k| <= tol * max(1, |theta|).  Collective when num_ranks > 1.
 * eigenvector (optional, host or device, dmv_number_states elements of type elt) is rebuilt in a second pass.
 * The start vector is a deterministic function of `seed`. */
int dmv_lanczos(dmv_context *ctx, int elt, int max_iters, double tol, uint64_t seed, double *eigenvalue,
                void *eigenvector, int *iterations, double *residual);

/* ---- time evolution on the device: y = exp(z H) x for a Hermitian H (every model the reference takes) by the Lanczos
 * approximation with adaptive sub-steps and full reorthogonalisation; the Krylov basis stays in HBM, dot products are
 * reduced over the ranks with NCCL and only a few scalars per step visit the host.  z = (z_re, z_im): real time is
 * z = -i t, imaginary time is z = -tau.  elt = DMV_C128 always; DMV_F64 only when z_im == 0 and the operator and
 * characters are real (info "complex_coefficients" == 0).  x, y: host or device pointers of dmv_number_states elements;
 * y may alias x.  krylov_dim: 0 = default (30), else 2..64; the basis is one context-owned allocation of
 * (krylov_dim + 1) * dmv_number_states elements, kept for later calls, and the call fails (naming the bytes needed)
 * when it does not fit.  tol > 0: bound on the estimated error per unit of z, relative to the norm of the vector each
 * sub-step starts from.  Collective when num_ranks > 1 (needs dmv_comm_init), like dmv_lanczos.
 * products (may be NULL): products of H applied; error_estimate (may be NULL): sum of the local estimates.
 * dmv_get_info "expm_dot_vectors" / "expm_combine_vectors": vectors read or written by the block kernels of the last
 * call (for bandwidth accounting). */
int dmv_expm_multiply(dmv_context *ctx, int elt, double z_re, double z_im, const void *x, void *y,
                      int krylov_dim, double tol, int *products, double *error_estimate);

/* ---- the nev lowest eigenpairs on the device (row f3: what src/Diagonalize.chpl asks PRIMME for) by block
 * Krylov-Schur with full reorthogonalisation; the basis stays in HBM, the products run through dmv_matvec_batch, dot
 * products are reduced over the ranks with NCCL and only small dense matrices visit the host.  Collective when
 * num_ranks > 1 (needs dmv_comm_init), like dmv_lanczos.
 * elt = DMV_C128 always; DMV_F64 only when info "complex_coefficients" == 0.  1 <= nev <= the global dimension.
 * block_size: 0 = auto (min(nev, 4) for DMV_F64, min(nev, 3) for DMV_C128: the vectors one batched product shares), else
 *   1..6, capped at the global dimension.  block_size 1 finds one copy of a degenerate eigenvalue at a time and can miss
 *   its other copies; block_size >= the multiplicity finds them all.
 * krylov_dim: basis size m; 0 = auto, min(65 - p, max(32, 2 nev + 4 p)) with p the block size; else nev + 2 p <= m and
 *   m + p <= 65.  m is capped at the global dimension n_global; when the capped m is n_global, nev + 2 p <= m is waived
 *   (the basis spans the whole space and every pair is exact after one Rayleigh-Ritz).  The basis is one context-owned
 *   allocation of (m + p) * dmv_number_states elements, shared with dmv_expm_multiply and kept for later calls; the call
 *   fails (naming the bytes needed) when it does not fit.
 * tol > 0: pair i is converged when its Krylov-Schur residual estimate |H y_i - theta_i y_i| <= tol * max(1, |theta_i|).
 * max_restarts >= 0: the call stops after that many restart cycles even if not every pair has converged (not an error).
 * seed: the start block is a deterministic function of it (k_fill, as dmv_lanczos).
 * eigenvalues (nev, ascending), residuals (nev, may be NULL): host memory.  eigenvectors (may be NULL): nev vectors of
 * dmv_number_states elements of type elt one after the other ([nev, n], the layout of dmv_matvec_batch), this rank's
 * hashed block, host or device memory; orthonormal over the ranks; within a degenerate eigenspace any orthonormal basis.
 * converged: pairs of the nev that met the criterion; products: single-vector applications of H; restarts: restart
 * cycles (each may be NULL).  dmv_get_info "eigsh_block_vectors" / "eigsh_rotate_vectors": vectors read or written by the
 * Gram / update kernels and by the in-place rotation k_block_rotate in the last call (for bandwidth accounting). */
int dmv_eigsh(dmv_context *ctx, int elt, int nev, int block_size, int krylov_dim, double tol, int max_restarts,
              uint64_t seed, double *eigenvalues, void *eigenvectors, double *residuals,
              int *converged, int *products, int *restarts);

/* ---- spin-spin correlations on the device (row f5; not in the reference): <x|σᶻᵢσᶻⱼ|x> / <x|x> and <x|σᶻᵢ> / <x|x>
 * for num_vectors vectors ([num_vectors, n] layout of dmv_matvec_batch, n = dmv_number_states, this rank's hashed block),
 * host or device x; σᶻ is +1 on a set bit.  x is a vector of the symmetry-adapted basis (the representatives and norms
 * the products use); the answer is the expectation value in the state it represents on the full space.  One pass over
 * x and the representatives per vector (k_zz_gram on the FP64 tensor cores) and an O(|G| N^2) group average on the
 * host.  correlations: num_vectors * N * N doubles (vector, i, j), magnetization: num_vectors * N doubles (may be NULL),
 * host or device.  Fails for a zero vector.  Collective when num_ranks > 1 (needs dmv_comm_init); every rank returns
 * the same matrices.  A repeated call is bit-identical. */
int dmv_zz_correlations(dmv_context *ctx, int elt, int num_vectors, const void *x, double *correlations,
                        double *magnetization);

/* ---- flip-flop correlations on the device (row f7; not in the reference): T_ij = <x|σ⁺ᵢσ⁻ⱼ|x> / <x|x> for num_vectors
 * vectors (the layout, the basis and the meaning of x are those of dmv_zz_correlations), host or device x.  σ⁺ turns a
 * 0 bit into a 1 bit (the convention of the operator expressions).  pm: num_vectors * N * N complex numbers (vector, i,
 * j), interleaved (re, im), 2 num_vectors N^2 doubles, host or device.  T is Hermitian; T_ii = (1 + m_i) / 2 with m
 * from dmv_zz_correlations.  For every basis, with or without a fixed Hamming weight, and i != j:
 *     <σˣᵢσˣⱼ + σʸᵢσʸⱼ> = 2 (T_ij + T_ji) = 4 Re T_ij,    <σᵢ·σⱼ> = C_ij + 4 Re T_ij   (C: dmv_zz_correlations),
 * and Im T_ij is the spin current of the bond (up to the sign convention of the current).
 * Method: x lies in a one-dimensional irrep of the group G of the basis, so σ⁺ᵢσ⁻ⱼ may be replaced by its G-average,
 * which the row formula of the product evaluates.  One walk over this rank's rows and their antiparallel pairs sums
 * conj(x_b) / n_b chi (n x)[rep(r_b ^ (1 << i | 1 << j))] over the rows with bit i set and bit j clear into one sum per
 * class (orbit under G) of ordered pairs; T_ij = S_c / (<x|x> |c|).  An element with a spin flip maps (i, j) to
 * (p(j), p(i)).  elt = DMV_F64 or DMV_C128, also with complex characters.  Fails for a zero vector.  Collective when
 * num_ranks > 1 (needs dmv_comm_init and the whole basis on every rank, as the replicated-x product); every rank
 * returns the same matrices.  Every reduction has a fixed order and there are no floating-point atomics: a repeated
 * call is bit-identical. */
int dmv_pm_correlations(dmv_context *ctx, int elt, int num_vectors, const void *x, double *pm);

/* ---- one-site operators between symmetry sectors on the device (row f8; not in the reference): the start vectors of
 * dynamical structure factors S(q, ω).  y = B_targetᴴ · O · B_source · x with O = Σ_j w_j o_j, o_j = 1, σᶻ_j, σ⁺_j or σ⁻_j
 * (kind), σᶻ = +1 on a set bit, σ⁺ turning a 0 bit into a 1 bit (the conventions of the expressions and of
 * dmv_pm_correlations); weights: N complex numbers, interleaved (re, im).  B is the symmetry-adapted basis of a context
 * (column k = P|r_k> / ‖P|r_k>‖, P = 1/|G| Σ_g conj χ(g) U_g).  So y is the projection of Oψ onto the target sector; it
 * is not assumed that Oψ lies wholly in that sector.
 * Accepted: both contexts on the same device with the same number of sites, rank and number of ranks; Hamming weights
 * equal for DMV_SPIN_ONE / DMV_SPIN_Z, target = source + 1 for DMV_SPIN_PLUS and source - 1 for DMV_SPIN_MINUS, or both
 * free (-1); the target group a subset of the source group, compared as sets of (permutation, flip) (characters may
 * differ; a target without symmetries is always allowed, and unfolds a symmetric state into the plain basis).  elt
 * applies to x and y; DMV_F64 only when the weights and the characters of both bases are real.  x: num_vectors source
 * vectors, y: num_vectors target vectors, [num_vectors, n] layout (n = dmv_number_states of each context, this rank's
 * hashed block), host or device.  Anything else fails with a message naming the reason, and nothing is written.
 * Method: with psi = B_source x in the source's irrep, P_target O psi = Σ_k K_k o'_k psi with
 *     K_k = 1/|G_t| Σ_{g in G_t} χ_t(g) conj χ_s(g) w_{p_g⁻¹(k)},
 * o'_k = o_k for elements without a flip; a flip turns σᶻ into -σᶻ and swaps σ⁺ and σ⁻ (free weight with spin inversion:
 * the row walks both its set and its clear bits).  One lane per target row (k_spin_rows) finds psi at the row's own
 * state or at its one-bit neighbours through the source's orbit minimum, character and look-up (k_rows' table refilled
 * from x when the source has trivial characters, else the index and the norms).  A source state outside the source
 * basis adds nothing when its projection vanishes and is an error otherwise.  One store per row and no atomics: a
 * repeated call is bit-identical.  Collective when num_ranks > 1 (needs dmv_comm_init on the source and its whole basis
 * on every rank, as dmv_pm_correlations); the rows are this rank's rows of the target basis. */
enum { DMV_SPIN_ONE = 0, DMV_SPIN_Z = 1, DMV_SPIN_PLUS = 2, DMV_SPIN_MINUS = 3 };
int dmv_apply_spin(dmv_context *target, dmv_context *source, int elt, int kind, const double *weights,
                   int num_vectors, const void *x, void *y);

/* ---- bipartite entanglement on the device (row f9; not in the reference): the reduced density matrix
 * ρ_A = Tr_B |ψ><ψ| of the normalised full-space state ψ = B x / ‖x‖ (B the basis of dmv_apply_spin, so
 * ψ(s) = χ n x[rep(s)] / ‖x‖), for a set A of n_a sites (1 <= n_a <= 16, distinct, in [0, N)).  Bit k of a local
 * configuration of A is site sites_a[k], so the order of the list matters; B is the complement, its sites ascending.
 * At a fixed Hamming weight W, ρ_A is block diagonal in the weight w of A: blocks w = max(0, W - (N - n_a)) ...
 * min(n_a, W), of dimension d_w = C(n_a, w), rows the local configurations of weight w in ascending numeric order.  At
 * free weight one block of dimension 2^n_a, rows 0 ... 2^n_a - 1.  dmv_rdm_layout gives the blocks (no device needed):
 * *num_blocks, *w_first (-1 at free weight; may be NULL) and dims (room for 17 entries; may be NULL), with the checks
 * of n_a and, when sites_a is not NULL, of the sites.
 * rho (host or device): num_vectors * Σ_w d_w² complex numbers, interleaved (re, im), every block row-major, one after
 * another in ascending w, vector after vector.  Hermitian by construction (the lower triangle mirrors the upper one, the
 * diagonal is real); real x with real characters gives imaginary parts of exactly 0.  Tr ρ = 1 to rounding (not
 * imposed).  x: num_vectors vectors [num_vectors, n] of this rank's hashed block, host or device; elt = DMV_C128 always,
 * DMV_F64 only when info "complex_coefficients" == 0.  Refused with a message, and nothing written: a zero vector,
 * duplicate sites or sites out of range, n_a outside 1..16, and a ρ whose blocks, work space and (for host rho) staging
 * copy do not fit in free device memory (the message names the bytes).
 * Method: per block, the columns b of B (combinadic order at a fixed weight) are cut into chunks of at most 2^24
 * amplitudes, a function of (N, W, A) alone.  k_rdm_fill writes Ψ[a, c] = ψ(embed_A(a) | embed_B(b_c)) of a chunk through
 * the orbit minimum and look-up of dmv_apply_spin; k_rdm_gram adds Ψ Ψᴴ on the FP64 tensor cores (tiles of 32 x 32 on or
 * above the diagonal, a fixed number of column slices summed in order, chunks added in order).  No floating-point
 * atomics: a repeated call is bit-identical.  Collective when num_ranks > 1 (needs dmv_comm_init and the whole basis on
 * every rank, as dmv_apply_spin): rank r takes chunks r, r + P, ...; the blocks are summed over the ranks and every rank
 * returns the same ρ.  dmv_get_info: "rdm_amplitudes" (amplitudes this rank filled in the last call) and
 * "rdm_gram_flops" (real FP64 multiply-adds its Gram ran, padded tiles included). */
int dmv_reduced_density_matrix(dmv_context *ctx, int elt, int num_vectors, const void *x, int n_a,
                               const int32_t *sites_a, double *rho);
int dmv_rdm_layout(int n_sites, int hamming_weight, int n_a, const int32_t *sites_a, int *num_blocks, int *w_first,
                   int32_t *dims);

/* ---- finite-temperature Lanczos on the device (row f6; not in the reference): the random-vector quadrature of the
 * finite-temperature Lanczos method (Jaklič & Prelovšek 1994), also called stochastic Lanczos quadrature.  For each of
 * num_vectors start vectors r, `steps` steps of the three-term recurrence (no reorthogonalisation, no stored basis) give
 * the tridiagonal T_M = Q diag(θ) Qᵀ and its Gauss quadrature: nodes θ_k and weights w_k = |r|² Q₀ₖ², so that
 *     <r|f(H)|r> ≈ Σ_k w_k f(θ_k)   (exact for polynomials of degree below 2 M),
 *     Tr_sector f(H) ≈ (1/R) Σ_r Σ_k w_rk f(θ_rk)   (unbiased when E[r r†] = 1).
 * The quadrature stays correct after orthogonality is lost: spurious copies of converged Ritz values carry the right
 * total weight.  Row r of nodes / weights (host memory, num_vectors * steps doubles each) holds vector r; Σ_k w_rk = |r|²
 * (the norm over all ranks).  Slots past steps_done[r] hold node 0 and weight 0.
 * steps: >= 1, capped at the global dimension.  A recurrence whose Krylov space is invariant (β_{j+1} <= 1e-14
 *   max(1, |α_j|), decided from the reduced scalars, so every rank takes the same step) stops at j + 1 steps and its vector
 *   is zeroed; steps_done[r] (may be NULL) says where.
 * start: NULL for seeded vectors, else num_vectors vectors [num_vectors, n] of type elt (this rank's hashed block, host or
 *   device memory; none may be zero).  Seeded entry s of vector r depends only on (seed, r, representative s), so one
 *   rank and P ranks start from the same vectors:
 *     h = hash64_01(s ^ hash64_01(seed + 0x9e3779b97f4a7c15 (r + 1)))   (arithmetic modulo 2^64)
 *     DMV_F64: +1 if bit 63 of h is clear, else -1;  DMV_C128: e^{iφ} with φ = 2π (h >> 11) 2^-53.
 *   Then |r|² = n_global (to rounding for DMV_C128) and E[r r†] = 1.
 * elt = DMV_C128 always; DMV_F64 only when info "complex_coefficients" == 0.
 * The recurrences run in groups of G start vectors that share one batched product per step (dmv_matvec_batch): G = 4 on
 * k_gather, 6 real or 3 complex vectors on k_rows_batch, 1 otherwise (and at most num_vectors); dmv_get_info
 * "quadrature_group" gives the G of the last call.  The 3 G vectors of a group are one context-owned allocation, kept for
 * later calls; the call fails (naming the bytes needed) when it does not fit.  Every reduction has a fixed order: a
 * repeated call on the same context gives bit-identical nodes and weights.  products (may be NULL): single-vector
 * applications of H.  Collective when num_ranks > 1 (needs dmv_comm_init), like dmv_lanczos. */
int dmv_lanczos_quadrature(dmv_context *ctx, int elt, int num_vectors, int steps, uint64_t seed, const void *start,
                           double *nodes, double *weights, int *steps_done, int *products);

/* ---- per-stage timings of the last product, in milliseconds (the reference's timing tree,
 * DMV:1028-1052).  names: see dmv_timing_name(i); returns the number of stages. */
int dmv_last_timings(dmv_context *ctx, double *ms, int capacity);
const char *dmv_timing_name(int i);
/* algorithmic counters of the last plan: number of emitted off-diagonal terms of this rank */
int64_t dmv_number_terms(const dmv_context *ctx);

/* ---- the reference's plugin surface (src/FFI.chpl:233-239, DMV:1095-1110).  `op` is the
 * ls_hs_operator* the Haskell library hands out; it must have been bound to a context with
 * dmv_bind_operator (see INTEGRATION.md for the shim that extracts the flat tables). */
int dmv_bind_operator(const void *ls_hs_operator_ptr, dmv_context *ctx);
void ls_chpl_matrix_vector_product(const void *ls_hs_operator_ptr, int num_vectors, double *x, double *y);

/* PRIMME's matrix-vector callback (reference src/Diagonalize.chpl:134-162: `primme.matrixMatvec = ls_chpl_primme_matvec`):
 * y[:, k] = H x[:, k] for k < *block_size, real(64) columns with leading dimensions *ldx, *ldy >= dmv_number_states.
 * The reference finds the operator through primme->matrix; here the primme_params pointer is the handle and must have
 * been bound with dmv_bind_operator(primme, ctx).  Host or device columns; collective when the context has several
 * ranks; sets *ierr = 0 and halts on failure like the reference. */
void ls_chpl_primme_matvec(void *x, int64_t *ldx, void *y, int64_t *ldy, int *block_size, void *primme, int *ierr);

/* The other three entries of `ls_chpl_kernels` (src/FFI.chpl:233-239).  Outputs are returned the way Chapel's
 * convertToExternalArray does (BO:232,265-272): allocated by the callee, released by the caller through `freer`.
 * Layout of chpl_external_array (Chapel runtime, chpl-external-array.h): {void *elts; uint64_t num_elts; void *freer}.
 *   ls_chpl_operator_apply_diag      BO:217-234: coeffs[i] = <alpha_i|H|alpha_i> (real(64)), no projection
 *   ls_chpl_operator_apply_off_diag  BO:236-275: CSR by row: betas / coeffs (complex128) hold count * T entries of
 *                                    which offsets[count] are used, offsets = row pointer; terms with the same flip
 *                                    mask are merged into one entry; within a row entries are ordered by flip-mask
 *                                    group (the third-party kernel's order is not specified in the reference tree)
 *   ls_chpl_enumerate_representatives SE:588-603: this rank's block of representatives; `handle` is the ls_hs_basis*
 *                                    (bound with dmv_bind_operator like an operator handle); bounds are ignored
 *                                    exactly as in the reference
 * dmv_apply_diag / dmv_apply_off_diag are the same kernels on caller-owned arrays (host or device pointers;
 * betas: count * dmv_max_number_off_diag entries, coeffs: twice that many doubles, offsets: count + 1). */
typedef struct {
  void *elts;
  uint64_t num_elts;
  void (*freer)(void *);
} dmv_external_array;
int dmv_apply_diag(dmv_context *ctx, int64_t count, const uint64_t *alphas, double *coeffs);
int dmv_apply_off_diag(dmv_context *ctx, int64_t count, const uint64_t *alphas, uint64_t *betas, double *coeffs,
                       int64_t *offsets);
void ls_chpl_operator_apply_diag(const void *ls_hs_operator_ptr, int64_t count, const uint64_t *alphas,
                                 dmv_external_array *coeffs, int64_t num_tasks);
void ls_chpl_operator_apply_off_diag(const void *ls_hs_operator_ptr, int64_t count, const uint64_t *alphas,
                                     dmv_external_array *betas, dmv_external_array *coeffs,
                                     dmv_external_array *offsets, int64_t num_tasks);
void ls_chpl_enumerate_representatives(const void *ls_hs_basis_ptr, uint64_t lower, uint64_t upper,
                                       dmv_external_array *dest);

/* ---- host-side pieces exposed for the CPU tests (no device needed; NOT on the product path).
 * dmv_debug_tridiagonal_lowest: lowest eigenpair of a symmetric tridiagonal matrix, the host half of dmv_lanczos.
 * dmv_debug_compile_group: compiles the symmetry group of `basis` into the device orbit program, verifies it against
 *   bit-by-bit permutation and evaluates the compiled program (the device functions themselves, compiled for the host)
 *   for `count` states: reps[k] = min_g g(s_k), stab[k] = |{g : g(s_k) = s_k}|.
 *   info[0..5] = {n_q, n_stages, n_t, n_left, n_right, has_flip}.
 * dmv_debug_torus_sq_rows: for a basis whose group is the full space group of a K x K torus (K = 4 or 6), evaluates
 *   the square-torus orbit minimum of s_k ^ x_f for every state k and flip mask f twice, with the device functions
 *   compiled for the host: rows[k n_flips + f] through the row form k_rows runs (the transposed state XORed with the
 *   transposed flip mask), single[...] through the single-state form.  Fails when the group has no square-torus form.
 * dmv_debug_ordered_table: builds the ordered layout of the k_rows table (complex128: one-slot buckets,
 *   `buckets_per_state` per state, at most 2^bits blocks) over the `n` ascending representatives `reps` with the device
 *   functions compiled for the host, inserts them in order and looks every one up again: block[k] = prefix block of
 *   reps[k], home[k] = its home bucket, probes[k] = buckets its look-up reads.  Fails when a state is not found.
 * dmv_debug_dense_order: builds the dense ordered table of k_rows (option rows_dense_order, at most 2^bits prefix blocks)
 *   over the `n` ascending representatives with the library's host builder, and looks every one up again with the
 *   device functions compiled for the host: block[k] = prefix block of reps[k], slot[k] = its slot, probes[k] = slots
 *   its look-up reads; info[0] = states the two perfect-hash levels place, info[1] = rank blocks.  Fails when two
 *   states share a slot or a state is not found. */
int dmv_debug_tridiagonal_lowest(int k, const double *diag, const double *offdiag, double *eigenvalue, double *vector);
/* dmv_debug_tridiagonal_expm: host half of dmv_expm_multiply, c = exp(z T) e_1 for the symmetric tridiagonal T
 *   (diag a[0..k), off-diag b[0..k-1)), c interleaved (re, im), 2k doubles */
int dmv_debug_tridiagonal_expm(int k, const double *a, const double *b, double z_re, double z_im, double *c);
/* dmv_debug_hermitian_eigen: host half of dmv_eigsh, the cyclic Jacobi eigensolver: a = k x k Hermitian matrix,
 *   row-major, interleaved (re, im) (2 k^2 doubles); eigenvalues ascending (k doubles); eigenvectors (may be NULL):
 *   2 k^2 doubles, component r of eigenvector i at [2 (r k + i)] */
int dmv_debug_hermitian_eigen(int k, const double *a, double *eigenvalues, double *eigenvectors);
/* dmv_debug_tridiagonal_quadrature: host half of dmv_lanczos_quadrature, the Gauss quadrature of the symmetric
 *   tridiagonal T (diag a[0..k), off-diag b[0..k-1)): nodes = its eigenvalues ascending, weights = the squared first
 *   components of its eigenvectors (k doubles each; they sum to 1) */
int dmv_debug_tridiagonal_quadrature(int k, const double *a, const double *b, double *nodes, double *weights);
/* dmv_debug_zz_symmetrize: host half of dmv_zz_correlations, the group average of a Gram block: gram is (N + 1) x N,
 *   row-major, gram[i][j] = sum_b |x_b|^2 s_i(r_b) s_j(r_b) for i < N and gram[N][j] = sum_b |x_b|^2 s_j(r_b)
 *   (gram[0][0] = <x|x> must be positive); correlations N x N, magnetization N (may be NULL).  The group is that of
 *   `basis`: its permutations and flips, {1, flip} for spin inversion alone, {1} without symmetries. */
int dmv_debug_zz_symmetrize(const dmv_basis_desc *basis, const double *gram, double *correlations,
                            double *magnetization);
/* dmv_debug_pm_classes: host half of dmv_pm_correlations.  class_of (N * N): class of the ordered pair (i, j), -1 on the
 *   diagonal, classes numbered in the row-major order of their first pair; class_size (room for N * N): pairs per class;
 *   *num_classes.  With sums (2 per class, interleaved), W = <x|x> > 0 and magnetization (N): pm (2 N^2 doubles) as
 *   dmv_pm_correlations finishes it.  The group is that of dmv_debug_zz_symmetrize. */
int dmv_debug_pm_classes(const dmv_basis_desc *basis, int32_t *class_of, int32_t *class_size, int32_t *num_classes,
                         const double *sums, double W, const double *magnetization, double *pm);
/* dmv_debug_spin_weights: host half of dmv_apply_spin, with its checks (sites, Hamming weights, subgroup, kind, elt and
 *   real weights / characters for DMV_F64).  k (4 N doubles, may be NULL): the complex coefficients of the set-bit
 *   walk, then of the clear-bit walk (DMV_SPIN_Z: K on the set bits and -K on the clear bits of the row's own state;
 *   DMV_SPIN_ONE: zero); c0 (2 doubles, may be NULL): the constant of the row factor (DMV_SPIN_ONE: Σ_k K_k);
 *   *walk (may be NULL): 0 the row's own state, 1 its clear bits, 2 its set bits, 3 both. */
int dmv_debug_spin_weights(const dmv_basis_desc *source, const dmv_basis_desc *target, int elt, int kind,
                           const double *weights, double *k, double *c0, int *walk);
int dmv_debug_compile_group(const dmv_basis_desc *basis, int64_t *info, int64_t count,
                            const uint64_t *states, uint64_t *reps, int32_t *stab);
int dmv_debug_ordered_table(const uint64_t *reps, int64_t n, int bits, int buckets_per_state, uint32_t *block,
                            uint32_t *home, uint32_t *probes);
int dmv_debug_dense_order(const uint64_t *reps, int64_t n, int bits, uint32_t *block, uint32_t *slot, uint32_t *probes,
                          int64_t *info);
int dmv_debug_torus_sq_rows(const dmv_basis_desc *basis, int64_t count, const uint64_t *states, int64_t n_flips,
                            const uint64_t *flips, uint64_t *rows, uint64_t *single);
/* The term store of the row kernel on bases with permutation symmetries (k_rows_stored, csrc/dmv_store.cu): the target
 *   index and a coefficient code of every term, built once per basis and rows, read in column blocks whose scaled x
 *   stays in L2.  It is chosen automatically; dmv_debug_rows_store overrides the choice for tests and measurements:
 *   mode -1 auto, 0 never, 1 whenever the store can be built; chunks 0 the cost model's column blocks, else 1 .. 64.
 *   The replicated-x product's whole-basis twin takes the same setting.  dmv_get_info keys: "rows_store" (1: the last
 *   rows product ran on the store), "rows_store_chunks", "rows_store_mb", "rows_store_terms", "rows_store_builds".
 * dmv_debug_rows_store_plan: the choice from sizes alone (no device): n_states targets, n_rows rows, about `terms`
 *   terms, element type, L2 and free bytes, mode and chunks as above.  out[5] = {use, column blocks, blocks per pass,
 *   states per block, bytes}; ms[2] = the model's milliseconds for the store and for k_rows.
 * dmv_debug_rows_store_coefficients: the coefficient dictionary of the store from a real look-up table of n values
 *   (and their negatives when any_s_out): *count codes written to coef (at most 16), or *count = -1 when the store
 *   cannot encode them (more than 16 distinct values, or any_generic). */
int dmv_debug_rows_store(dmv_context *ctx, int mode, int chunks);
int dmv_debug_rows_store_plan(int64_t n_states, int64_t n_rows, int64_t terms, int elt, int64_t l2_bytes,
                              int64_t free_bytes, int mode, int chunks, int64_t *out, double *ms);
int dmv_debug_rows_store_coefficients(const double *lut, int64_t n, int any_s_out, int any_generic, double *coef,
                                      int *count);
/* dmv_debug_solver_kernel: runs one launcher of the solver vector kernels (csrc/dmv_solver.cu) on the current device
 *   and a private stream, on host data, for the tests (needs a device, unlike the entries above).  kernel: "dot",
 *   "lanczos_update", "scale", "fill", "block_dot", "block_combine", "block_gram", "block_update", "block_rotate",
 *   "quad_fill", "quad_dot" or "quad_update"; elt: DMV_F64 | DMV_C128; n: elements of a vector (8-byte words for
 *   "scale" and "fill").  Every vector argument is a word offset into `arena` (arena_words doubles), which is copied
 *   to the device, run on, and copied back whole; offsets must be even for complex elements, -1 is null where the
 *   launcher takes null.  args (n_args), by kernel, with the small device inputs in `coef` and the small outputs in
 *   `out` (2 doubles per complex value):
 *     dot            {a, b}                              out[2] += <a, b>
 *     lanczos_update {w, v, u | -1}      coef {alpha, beta}            out[0] += |w|^2 after
 *     scale          {x, y, accumulate}  scalar = s
 *     fill           {x, seed, offset}
 *     block_dot      {J, w, V_0 .. V_{J-1}}                            out: h, 2 (J + 1)
 *     block_combine  {J, w | -1, out, V_0 .. V_{J-1}}  scalar = a, coef: c, 2 J    out: |out|^2, 2
 *     block_gram     {J, R, W, w_stride, V_0 .. V_{J-1}}               out: h, 2 (J R + R R)
 *     block_update   {J, R, W, w_stride, V_0 .. V_{J-1}}  coef: c, 2 J R  out: |W_r|^2, 2 R
 *     block_rotate   {k, l, V_0 .. V_{k-1}}              coef: S, 2 k l
 *     quad_fill      {x, seed, first, G}                 coef: n representatives (uint64 bits)
 *     quad_dot       {G, A, B}                                         out: 2 G
 *     quad_update    {G, P, Q, W, j, b2}   coef: dot from 0, b2 from word b2, 2 (j + 1) G each   out: |r_{j+1}|^2, 2 G
 *   The outputs of dot and lanczos_update are read first (the kernels add to them); every other output and the
 *   partials buffer (sized as the solvers size it) are NaN bytes before the launch.  *grid = CTAs of the main launch
 *   (0 when the launcher launched nothing).  The launchers' own checks apply (J <= 65, 1 <= R, G <= 6, 1 <= l <= k). */
int dmv_debug_solver_kernel(const char *kernel, int elt, int64_t n, const int64_t *args, int n_args, double scalar,
                            double *arena, int64_t arena_words, const double *coef, int64_t coef_words, double *out,
                            int64_t out_words, int *grid);

#ifdef __cplusplus
}
#endif
#endif /* DMV_B200_H */
