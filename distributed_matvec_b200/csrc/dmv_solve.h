// dmv_solve.h -- the host frame of the device solvers (dmv_lanczos, dmv_expm_multiply, dmv_eigsh, dmv_zz_correlations,
// dmv_pm_correlations, dmv_lanczos_quadrature): entry checks, reductions over the ranks, products and work space.  The rules every rank must
// follow live here once: decisions come from all-reduced scalars, a work space is never shrunk silently to what fits,
// and a product's output is cleared first only when the operator has no diagonal (include/dmv_b200.h, dmv_local_matvec:
// y = D x + O x with diagonal terms, else y += O x).
#pragma once
#include "dmv_context.h"

namespace dmv { namespace host {

struct SolverRun {
  dmv_context *ctx;
  const char *name;   // the entry point, for error messages
  int elt, P;
  int64_t n;          // states of this rank
  size_t words;       // 8-byte words of one vector
  bool ce;            // complex elements
  cudaStream_t st;

  // real_operator_only: real vectors (DMV_F64) are refused when the operator or its characters are complex
  SolverRun(dmv_context *c, int elt_, const char *name_, bool real_operator_only) : ctx(c), name(name_), elt(elt_) {
    use_device(ctx);
    require_states(ctx);
    if (elt != DMV_F64 && elt != DMV_C128) throw std::runtime_error("elt must be DMV_F64 or DMV_C128");
    if (real_operator_only && elt == DMV_F64 && ctx->complex_coefficients)
      throw std::runtime_error("the operator or its characters are complex: use complex vectors (DMV_C128)");
    P = ctx->num_ranks;
    if (P > 1 && !ctx->comm) throw std::runtime_error(std::string(name) + " on several ranks needs dmv_comm_init");
    n = ctx->n_states;
    words = (size_t)n * elt;
    ce = elt == DMV_C128;
    st = ctx->stream;
  }

  // sum `count` doubles at device address d over the ranks, in place
  void all_reduce(double *d, size_t count) const {
    if (P > 1) NCCL_CHECK(nccl().AllReduce(d, d, count, ncclDouble, ncclSum, ctx->comm, st));
  }

  // the dimension of the whole space: every rank stops at it alike (all-reduced on first use, in its own scratch slot)
  int64_t global_states() {
    if (n_global >= 0) return n_global;
    n_global = n;
    if (P > 1) {
      ctx->solver_scalars.alloc(kScratch);
      double *d = ctx->solver_scalars.ptr;
      const double mine = (double)n;
      CUDA_CHECK(cudaMemcpyAsync(d, &mine, sizeof(double), cudaMemcpyHostToDevice, st));
      all_reduce(d, 1);
      double g = 0.0;
      CUDA_CHECK(cudaMemcpyAsync(&g, d, sizeof(double), cudaMemcpyDeviceToHost, st));
      CUDA_CHECK(cudaStreamSynchronize(st));
      n_global = (int64_t)std::llround(g);
    }
    return n_global;
  }

  // out = H in for nv vectors of this rank, `words` apart
  void product(const double *in, double *out, int nv = 1) {
    if (ctx->h_diag_kept == 0) CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)nv * words * 8, st));
    const int rc = nv > 1    ? dmv_matvec_batch(ctx, elt, nv, in, out)
                   : P == 1 ? dmv_local_matvec(ctx, elt, in, out)
                            : dmv_matvec(ctx, elt, in, out);
    if (rc) throw std::runtime_error(g_last_error);
  }

  // `count` vectors of this rank (one element at least) in the context's work space, shared by the solvers and kept
  // between calls.  It only grows; a space that does not fit in free memory is an error naming the bytes, never a
  // smaller space.  Message: "<name>: <what> <count> vectors of <n> elements needs ... bytes ...<hint>".
  double *vectors(size_t count, const std::string &what, const std::string &hint = "") {
    DevBuf<double> &b = ctx->solver_vectors;
    const size_t need_words = count * std::max<size_t>(words, 1);
    if (b.count < need_words) {
      b.release();
      size_t free_b = 0, total_b = 0;
      CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
      const size_t need = need_words * sizeof(double);
      if (need > free_b)
        throw std::runtime_error(std::string(name) + ": " + what + " " + std::to_string(count) + " vectors of " +
                                 std::to_string(n) + " elements needs " + std::to_string(need) + " bytes, but only " +
                                 std::to_string(free_b) + " bytes are free on the device" + hint);
      b.alloc(need_words);
    }
    return b.ptr;
  }

  // the small device arrays of a solver (its own layout) and the per-CTA partials of the fixed-order reductions;
  // both grow only and are kept between calls
  double *scalars(size_t count) {
    ctx->solver_scalars.alloc(kScratch + count);
    return ctx->solver_scalars.ptr + kScratch;
  }
  double *partials(size_t count) {
    ctx->solver_partials.alloc(count);
    return ctx->solver_partials.ptr;
  }

 private:
  // global_states' slot ahead of the scalars; 32 doubles keep the scalars at the allocation's 256-byte alignment (the
  // warp-uniform coefficient loads of k_block_rotate touch more 32-byte sectors when they are shifted)
  static constexpr size_t kScratch = 32;
  int64_t n_global = -1;
};

} }  // namespace dmv::host
