// dmv_store.cu -- the term store of k_rows_stored: the target and coefficient of every term k_rows accumulates, found
// once per basis, and the product that reads them in column blocks (RowsStoreView in dmv_host.h, kernels in
// dmv_kernels.cu).
//
// k_rows spends each product on two things that do not depend on x: the orbit minimum of every term (instruction issue)
// and the random look-up of its target in a table several times the size of L2 (one HBM sector per term).  The store
// keeps each term as 4 bytes -- the target's index within its column block and a code for its coefficient -- so a
// product streams the entries and gathers (n x) from the compact scaled x of one group of column blocks at a time,
// which L2 holds while the pass runs.  The blocks cost a partial sum per row between passes; rows_store_plan weighs
// that against the gathers (DESIGN §3).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

#include "dmv_context.h"
#include "../../include/dmv_b200.h"

namespace dmv { namespace host {

namespace {

// Rates of the cost model: the least-squares fit (in log time) to the sweep of one H100 SXM at 700 W
// (profiles/h100_rows_store_sweep.log: 6x6 square, chain_32_symm, chain_36_symm, complex128 and float64, C = 1 .. 64).
// They are effective rates, not hardware ones, and one set cannot fit every workload: the gathers of the chains have
// more locality than the torus' (chain_36_symm at C = 1, all misses: 76 G/s; the 6x6 square: 34 G/s, the rate of random
// HBM sectors), so the model is off by up to 41 % on the 6x6 square at C = 1 and 51 % on chain_36_symm in float64.
// Near each workload's best C it is within 20 %, and its choice is within 10 % of the best C measured.
constexpr double kRowsTermsPerS = 30.0e9;    // k_rows: measured 32.5 G terms/s on the 6x6 square, 25 on chain_32 and
                                             // 20 on chain_36 (there the model puts k_rows 37 % too fast)
constexpr double kL2GatherPerS = 125.0e9;    // random gathers that hit L2
constexpr double kMissGatherPerS = 60.0e9;   // gathers that miss L2, between the torus' 34 and the chains' 76 G/s
constexpr double kStreamBytesPerS = 3.0e12;  // entries, counts, row data and partial sums
constexpr double kL2Share = 0.25;            // share of L2 a pass's block of x keeps resident beside the streams
constexpr int64_t kStoreMinRows = 1 << 20;   // below this a product takes well under a millisecond: k_rows

int64_t store_bytes(int64_t n_states, int64_t n_rows, int64_t terms, int chunks) {
  const int64_t tiles = (n_rows + 31) / 32;
  return terms * 4 + (int64_t)chunks * n_rows + ((int64_t)chunks * tiles + 1) * 8 + n_rows * 8 + n_states * 16 +
         n_rows * 16;
}

// seconds of one product on a store of `chunks` blocks read `per_pass` blocks at a time, elements of E bytes
double store_seconds(int64_t n_states, int64_t n_rows, int64_t terms, int chunks, int per_pass, double E,
                     int64_t l2_bytes) {
  const int64_t block = (n_states + chunks - 1) / chunks;
  const double pass_bytes = (double)block * per_pass * E;
  const double hit = std::min(1.0, kL2Share * (double)l2_bytes / std::max(pass_bytes, 1.0));
  const int passes = (chunks + per_pass - 1) / per_pass;
  const double gather = (double)terms * (hit / kL2GatherPerS + (1.0 - hit) / kMissGatherPerS);
  const double stream = ((double)terms * 4 + (double)chunks * n_rows + (double)n_rows * (16 + 2 * E)) / kStreamBytesPerS;
  const double partial = (2.0 * passes - 2.0) * (double)n_rows * E / kStreamBytesPerS;
  const double fill = (double)n_states * (8 + 2 * E) / kStreamBytesPerS;
  return gather + stream + partial + fill;
}

}  // namespace

// blocks per pass: the model's blocks are sized for complex128, so float64 reads two at a time; blocks asked for
// through dmv_debug_rows_store are read one per pass
int store_per_pass(int chunks_asked, int elt, int chunks) {
  return std::min(chunks, chunks_asked == 0 && elt != DMV_C128 ? 2 : 1);
}

// The store for a product on `n_rows` rows of a basis of `n_states` states with about `terms` terms (an estimate from
// sizes before the store exists), elements of `elt` doubles, on a device with `l2_bytes` of L2 and `free_bytes` free.
// mode -1 auto, 0 never, 1 whenever it fits; chunks 0 the model's column blocks, else that many.  The column blocks
// depend on the sizes only, never on the element type: float64 reads two blocks per pass of the same store.
StorePlan rows_store_plan(int64_t n_states, int64_t n_rows, int64_t terms, int elt, int64_t l2_bytes, int64_t free_bytes,
                          int mode, int chunks) {
  StorePlan P;
  if (mode == 0) { P.why = "off"; return P; }
  if (n_states < 1 || n_rows < 1) { P.why = "empty"; return P; }
  if (chunks < 0 || chunks > kStoreMaxChunks) { P.why = "chunks"; return P; }
  const double E = elt == DMV_C128 ? 16.0 : 8.0;
  if (chunks == 0) {   // the model's blocks: the fewest with the least time for complex128
    double best = 0.0;
    for (int c = 1; c <= kStoreMaxChunks && c <= n_states; ++c) {
      const double t = store_seconds(n_states, n_rows, terms, c, 1, 16.0, l2_bytes);
      if (c == 1 || t < best * (1.0 - 1e-9)) { best = t; P.chunks = c; }
    }
  } else {
    P.chunks = (int)std::min<int64_t>(chunks, n_states);
  }
  P.block_states = (n_states + P.chunks - 1) / P.chunks;
  P.per_pass = store_per_pass(chunks, elt, P.chunks);
  P.bytes = store_bytes(n_states, n_rows, terms, P.chunks);
  P.ms_store = 1e3 * store_seconds(n_states, n_rows, terms, P.chunks, P.per_pass, E, l2_bytes);
  P.ms_rows = 1e3 * (double)terms / kRowsTermsPerS;
  if (P.block_states > (int64_t)1 << kStoreIndexBits) { P.why = "packing"; return P; }
  if ((double)P.bytes > 0.25 * (double)free_bytes) { P.why = "memory"; return P; }
  if (mode == -1) {
    if (n_rows < kStoreMinRows) { P.why = "small"; return P; }
    if (P.ms_store >= P.ms_rows) { P.why = "model"; return P; }
  }
  P.use = true;
  P.why = "store";
  return P;
}

// the dictionary of the coefficients pop_term returns on the bit-parallel path: the real look-up table and, when some
// group has an outside sign mask, its negatives; distinct as bit patterns, in order of first appearance.  False when a
// group takes the generic coefficient or the values need more than kStoreCodes codes.
bool store_coefficients(const HostTables &h, std::vector<double> &coef) {
  coef.clear();
  if (h.any_generic) return false;
  auto add = [&](double v) {
    for (double c : coef)
      if (std::memcmp(&c, &v, sizeof v) == 0) return true;
    if ((int)coef.size() == kStoreCodes) return false;
    coef.push_back(v);
    return true;
  };
  for (double v : h.lut_re) {
    if (!add(v)) return false;
    if (h.any_s_out && !add(v * -1.0)) return false;
  }
  return true;
}

namespace {

int64_t device_l2_bytes(const dmv_context *ctx) {
  int l2 = 0;
  CUDA_CHECK(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, ctx->device));
  return l2;
}

enum BuildResult { BUILT, REFUSED, OVERFLOW, NO_MEMORY };

// builds basis->store over the rows of p (see rows_store_product).  REFUSED: a target is missing with c != 0 (k_rows
// then reports it on every product) or a coefficient has no code -- neither changes while the basis and rows stay;
// OVERFLOW: a row has more than 255 entries in one of plan.chunks blocks; NO_MEMORY: the exact size breaks the memory
// rule (S.exact_terms keeps the term count, so a later attempt checks it without another count pass).
BuildResult rows_store_build(dmv_context *basis, const KernelParams &p0, int64_t n_rows, const StorePlan &plan,
                             const std::vector<double> &coef, int64_t free_bytes, cudaStream_t st) {
  RowsStore &S = basis->store;
  KernelParams p = p0;
  p.row_begin = 0;
  p.row_end = n_rows;
  RowsStoreView &V = S.view;
  V = RowsStoreView{};
  V.n_rows = n_rows;
  V.n_tiles = (n_rows + 31) / 32;
  V.chunks = plan.chunks;
  V.block_states = plan.block_states;
  for (int c = 0; c < kStoreCodes; ++c) V.coef[c] = c < (int)coef.size() ? coef[c] : 0.0;
  S.counts.alloc((size_t)V.chunks * n_rows);
  S.tile_off.alloc((size_t)V.chunks * V.n_tiles + 1);
  if (p.n_diag > 0) S.diag.alloc((size_t)n_rows);
  V.counts = S.counts.ptr;
  V.tile_off = S.tile_off.ptr;
  V.diag = p.n_diag > 0 ? S.diag.ptr : nullptr;
  DevBuf<unsigned long long> flags;
  flags.alloc(4);
  CUDA_CHECK(cudaMemsetAsync(flags.ptr, 0, 4 * sizeof(unsigned long long), st));
  launch_store_build(p, V, false, flags.ptr, st);
  launch_store_offsets(V, st);
  unsigned long long h_flags[4] = {0, 0, 0, 0};
  uint64_t total = 0;
  CUDA_CHECK(cudaMemcpyAsync(h_flags, flags.ptr, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  CUDA_CHECK(cudaMemcpyAsync(&total, S.tile_off.ptr + (size_t)V.chunks * V.n_tiles, 8, cudaMemcpyDeviceToHost, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  const int64_t bytes = store_bytes(basis->n_states, n_rows, (int64_t)total, V.chunks);
  const BuildResult why = (h_flags[0] || h_flags[2]) ? REFUSED : h_flags[1] ? OVERFLOW
                          : (double)bytes > 0.25 * (double)free_bytes ? NO_MEMORY : BUILT;
  if (why != BUILT) {
    S.release_buffers();
    if (why == NO_MEMORY) S.exact_terms = (int64_t)total;
    return why;
  }
  S.entries.alloc((size_t)std::max<uint64_t>(total, 1));
  S.xs.alloc((size_t)basis->n_states * 2);
  S.partial.alloc((size_t)n_rows * 2);
  V.entries = S.entries.ptr;
  launch_store_build(p, V, true, flags.ptr, st);
  CUDA_CHECK(cudaStreamSynchronize(st));
  S.built = true;
  S.terms = (int64_t)total;
  S.bytes = bytes;
  ++S.builds;
  return BUILT;
}

}  // namespace

// y[rows of p] through k_rows_stored when the store applies (see rows_product for the arguments); false: k_rows' turn.
// The rows are p.row_states (the replicated-x product: this rank's block, p.row_end of them) or the basis itself, of
// which p may name a range (the row chunks of a product into host memory).
// The choice is made once per product, by the call that refills x (fill); the later row chunks of the same product
// follow it.  Free memory is only asked before a store is built: once one exists for these rows and this setting
// (mode, chunks), every product runs on it, so neither the path nor the order of a row's sum depends on what else
// holds device memory at the time.
bool rows_store_product(dmv_context *basis, KernelParams &p, int elt, const void *x_all, const uint32_t *pos,
                        cudaStream_t stream, bool fill, dmv_context *timer) {
  RowsStore &S = basis->store;
  const bool ce = elt == DMV_C128;
  auto passes = [&]() {
    const int C = S.view.chunks;
    for (int k0 = 0; k0 < C; k0 += S.per_pass)
      launch_rows_stored(p, S.view, S.xs.ptr, S.partial.ptr, k0, std::min(C, k0 + S.per_pass), ce, stream);
  };
  if (!fill) {   // a later row chunk: the decision of the product's first chunk stands
    if (!S.active) return false;
    passes();
    return true;
  }
  S.active = false;
  const int mode = basis->opt.rows_store, chunks = basis->opt.rows_store_chunks;
  if (mode == 0 || basis->n_states < 1) return false;
  const int64_t n_rows = p.row_states ? p.row_end : basis->n_states;
  const bool same_rows = S.rows_of == p.row_states && S.n_rows == n_rows;
  if (!same_rows || (S.built && (S.mode != mode || S.chunks_asked != chunks))) {
    CUDA_CHECK(cudaStreamSynchronize(stream));   // (queued products may still read the old store)
    S.release();
    S.rows_of = p.row_states;
    S.n_rows = n_rows;
  }
  if (!S.built) {
    if (S.refused) return false;
    std::vector<double> coef;
    if (!store_coefficients(basis->h_pull, coef)) { S.refused = true; return false; }
    // terms from sizes: about half of the row's flip-mask groups emit (a Heisenberg bond flips an antiparallel pair);
    // the plan, its column blocks included, is a function of the sizes alone
    const int64_t terms_estimate = n_rows * std::max<int64_t>(1, (int64_t)basis->h_pull.groups.size() / 2);
    size_t free_b = 0, total_b = 0;
    CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    const StorePlan plan = rows_store_plan(basis->n_states, n_rows, terms_estimate, elt, device_l2_bytes(basis),
                                           (int64_t)free_b, mode, chunks);
    if (!plan.use || plan.chunks == S.overflow_chunks) return false;
    if (S.exact_terms > 0 &&
        (double)store_bytes(basis->n_states, n_rows, S.exact_terms, plan.chunks) > 0.25 * (double)free_b)
      return false;   // (still short of memory: no second count pass)
    const BuildResult r = rows_store_build(basis, p, n_rows, plan, coef, (int64_t)free_b, stream);
    if (r == REFUSED) S.refused = true;
    if (r == OVERFLOW) S.overflow_chunks = plan.chunks;
    if (r != BUILT) return false;
    S.mode = mode;
    S.chunks_asked = chunks;
  }
  S.per_pass = store_per_pass(chunks, elt, S.view.chunks);
  CUDA_CHECK(cudaEventRecord(timer->ev_fill[0], stream));
  launch_table_fill(basis->n_states, ce, x_all, basis->d_norms.ptr, pos, nullptr, nullptr, nullptr, nullptr, stream,
                    S.xs.ptr);
  CUDA_CHECK(cudaEventRecord(timer->ev_fill[1], stream));
  timer->fill_timed = true;
  passes();
  S.active = true;
  return true;
}

} }  // namespace dmv::host

extern "C" {

int dmv_debug_rows_store_plan(int64_t n_states, int64_t n_rows, int64_t terms, int elt, int64_t l2_bytes,
                              int64_t free_bytes, int mode, int chunks, int64_t *out, double *ms) {
  const dmv::host::StorePlan P = dmv::host::rows_store_plan(n_states, n_rows, terms, elt, l2_bytes, free_bytes, mode,
                                                            chunks);
  if (out) {
    out[0] = P.use ? 1 : 0;
    out[1] = P.chunks;
    out[2] = P.per_pass;
    out[3] = P.block_states;
    out[4] = P.bytes;
  }
  if (ms) { ms[0] = P.ms_store; ms[1] = P.ms_rows; }
  return 0;
}

int dmv_debug_rows_store_coefficients(const double *lut, int64_t n, int any_s_out, int any_generic, double *coef,
                                      int *count) {
  dmv::host::HostTables h;
  if (lut && n > 0) h.lut_re.assign(lut, lut + n);
  h.any_s_out = any_s_out != 0;
  h.any_generic = any_generic != 0;
  std::vector<double> c;
  const bool ok = dmv::host::store_coefficients(h, c);
  if (count) *count = ok ? (int)c.size() : -1;
  if (ok && coef) std::copy(c.begin(), c.end(), coef);
  return 0;
}

}  // extern "C"
