// dmv_krylov.cu -- dmv_expm_multiply: y = exp(z H) x for a Hermitian H by the Lanczos approximation with adaptive
// sub-steps (Saad 1992; Hochbruck & Lubich 1997).  Every vector stays in HBM; the Krylov basis is orthogonalised in
// full with the fused block kernels of dmv_solver.cu, and only the reduced scalars of each step visit the host, where
// the small tridiagonal problem is solved.
#include <cfloat>
#include <complex>

#include "dmv_dense.h"
#include "dmv_solve.h"

extern "C" {

// ---- y = exp(z H) x on the device (DESIGN.md section 3, "dmv_expm_multiply").  Per sub-step of length h (a fraction of z):
// Lanczos with full (DGKS) reorthogonalisation builds V_0 .. V_{k-1} and T_k from w / |w|; on the host,
// c = exp(h z T_k) e_1 and the error estimate  beta * beta_k * |h z| * |e_k^T phi_1(h z T_k) e_1|  (Saad's corrected
// estimate: the norm of the next term of the Krylov expansion); h is halved until the estimate is <= tol * h * beta, and
// w <- beta * sum_j c_j V_j.  The Krylov space is built once per sub-step: shrinking h costs host arithmetic only.
int dmv_expm_multiply(dmv_context *ctx, int elt, double z_re, double z_im, const void *x, void *y, int krylov_dim,
                      double tol, int *products, double *error_estimate) {
  API_BEGIN
  if (products) *products = 0;
  if (error_estimate) *error_estimate = 0.0;
  SolverRun run(ctx, elt, "dmv_expm_multiply", true);
  if (krylov_dim != 0 && (krylov_dim < 2 || krylov_dim > kMaxBlockVectors - 1))
    throw std::runtime_error("krylov_dim must be 0 (default 30) or between 2 and 64");
  if (!(tol > 0.0) || !std::isfinite(tol)) throw std::runtime_error("tol must be positive and finite");
  if (!std::isfinite(z_re) || !std::isfinite(z_im)) throw std::runtime_error("z must be finite");
  if (elt == DMV_F64 && z_im != 0.0)
    throw std::runtime_error("a complex z needs complex vectors (DMV_C128)");
  if (!x || !y) throw std::runtime_error("x and y must not be null");
  const int m = krylov_dim == 0 ? 30 : krylov_dim;
  const int64_t n = run.n;
  const size_t words = run.words;
  const bool ce = run.ce;
  const cplx z(z_re, z_im);
  cudaStream_t st = run.st;
  ctx->kr_dot_vectors = ctx->kr_combine_vectors = 0;
  if (z == cplx(0.0, 0.0)) {   // exp(0) = 1: x itself, bit for bit
    if (x != y && words) CUDA_CHECK(cudaMemcpyAsync(y, x, words * 8, cudaMemcpyDefault, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
  }
  double *const basis = run.vectors(m + 1, "the Krylov basis of krylov_dim + 1 =", "; use a smaller krylov_dim");
  // scalars: [0, 2 * 66) block dot results, [132, 134) |out|^2 of a combine, [136, 136 + 2 * 65) host coefficients
  constexpr int kNrm = 2 * (kMaxBlockVectors + 1), kCoef = kNrm + 4;
  double *scal = run.scalars(kCoef + 2 * kMaxBlockVectors);
  double *partials = run.partials((size_t)block_partials_grid(n, ce) * (kMaxBlockVectors + 1) * 2);
  std::vector<double *> vp(m + 1);
  for (int k = 0; k <= m; ++k) vp[k] = basis + (size_t)k * words;
  VecList list{};
  auto set_list = [&](int J) { for (int k = 0; k < J; ++k) list.p[k] = vp[k]; };
  auto fetch = [&](double *h, const double *d, int count) {
    CUDA_CHECK(cudaMemcpyAsync(h, d, sizeof(double) * count, cudaMemcpyDeviceToHost, st));
  };
  // Krylov space exhausted at the GLOBAL dimension: every rank takes the same decision (as dmv_lanczos)
  const int64_t n_global = run.global_states();
  // w = x (host or device; y may alias x: x is read in full before y is written)
  if (words) CUDA_CHECK(cudaMemcpyAsync(vp[0], x, words * 8, cudaMemcpyDefault, st));
  std::vector<double> hh(kNrm + 2), h2(kNrm + 2);
  launch_block_dot(n, ce, list, 0, vp[0], partials, scal, st);
  ctx->kr_dot_vectors += 1;
  run.all_reduce(scal, 2);
  fetch(hh.data(), scal, 2);
  CUDA_CHECK(cudaStreamSynchronize(st));
  double beta = std::sqrt(std::max(0.0, hh[0]));
  double remaining = 1.0, err_sum = 0.0;
  int prods = 0;
  std::vector<double> alpha, betas, coef(2 * kMaxBlockVectors);
  std::vector<cplx> c;
  while (remaining > 0.0 && beta > 0.0 && std::isfinite(beta)) {
    launch_scale((int64_t)words, 1.0 / beta, vp[0], vp[0], false, st);   // V_0 = w / beta
    alpha.clear();
    betas.clear();
    int k = 0;
    double beta_k = 0.0;
    bool exact = false;
    for (int j = 0; j < m; ++j) {
      double *u = vp[j + 1];
      run.product(vp[j], u);
      ++prods;
      const int J = j + 1;
      set_list(J);
      // h = V^H u (and |u|^2), reduced over the ranks on the device; u -= V h reads h from there: no host round trip
      launch_block_dot(n, ce, list, J, u, partials, scal, st);
      run.all_reduce(scal, 2 * (J + 1));
      launch_block_combine(n, ce, 1.0, u, list, J, scal, u, partials, scal + kNrm, st);
      run.all_reduce(scal + kNrm, 2);
      ctx->kr_dot_vectors += J + 1;
      ctx->kr_combine_vectors += J + 2;
      fetch(hh.data(), scal, 2 * (J + 1));
      fetch(hh.data() + kNrm, scal + kNrm, 2);
      CUDA_CHECK(cudaStreamSynchronize(st));
      const double before = std::sqrt(std::max(0.0, hh[2 * J]));
      double after = std::sqrt(std::max(0.0, hh[kNrm]));
      double a_j = hh[2 * j];
      if (after < 0.7 * before) {   // DGKS: the pass cancelled most of u, so orthogonalise once more
        launch_block_dot(n, ce, list, J, u, partials, scal, st);
        run.all_reduce(scal, 2 * (J + 1));
        launch_block_combine(n, ce, 1.0, u, list, J, scal, u, partials, scal + kNrm, st);
        run.all_reduce(scal + kNrm, 2);
        ctx->kr_dot_vectors += J + 1;
        ctx->kr_combine_vectors += J + 2;
        fetch(h2.data(), scal, 2 * (J + 1));
        fetch(h2.data() + kNrm, scal + kNrm, 2);
        CUDA_CHECK(cudaStreamSynchronize(st));
        a_j += h2[2 * j];
        after = std::sqrt(std::max(0.0, h2[kNrm]));
      }
      alpha.push_back(a_j);
      k = J;
      beta_k = after;
      // happy breakdown: H V_j lies in the span (to rounding), or the space is the whole basis -- the step is exact
      if (after <= 1e-14 * before || (int64_t)k >= n_global) { exact = true; break; }
      if (J < m) {
        betas.push_back(after);
        launch_scale((int64_t)words, 1.0 / after, u, u, false, st);
      }
    }
    const dmv::host::TridiagonalEigen T(alpha, betas);
    double h = remaining, err = 0.0;
    if (!exact) {
      for (int halvings = 0;; ++halvings) {
        err = beta * beta_k * std::abs(h * z) * std::abs(T.phi1_last(h * z));
        if (err <= tol * h * beta) break;
        if (halvings == 200)
          throw std::runtime_error("dmv_expm_multiply: no sub-step of at least 2^-200 of z meets tol; raise "
                                   "krylov_dim or tol");
        h *= 0.5;
      }
    }
    T.exp_e1(h * z, c);
    for (int i = 0; i < k; ++i) { coef[2 * i] = -beta * c[i].real(); coef[2 * i + 1] = -beta * c[i].imag(); }
    CUDA_CHECK(cudaMemcpyAsync(scal + kCoef, coef.data(), sizeof(double) * 2 * k, cudaMemcpyHostToDevice, st));
    set_list(k);
    launch_block_combine(n, ce, 0.0, nullptr, list, k, scal + kCoef, vp[m], partials, scal + kNrm, st);
    ctx->kr_combine_vectors += k + 1;
    run.all_reduce(scal + kNrm, 2);
    fetch(hh.data() + kNrm, scal + kNrm, 2);
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::swap(vp[0], vp[m]);   // w = beta sum_j c_j V_j becomes the start of the next sub-step
    beta = std::sqrt(std::max(0.0, hh[kNrm]));
    err_sum += err;
    remaining = h == remaining ? 0.0 : remaining - h;
  }
  if (words) CUDA_CHECK(cudaMemcpyAsync(y, vp[0], words * 8, cudaMemcpyDefault, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  if (products) *products = prods;
  if (error_estimate) *error_estimate = err_sum;
  check_status(ctx);
  API_END
}

// host-only self-check entry for the tridiagonal exponential behind dmv_expm_multiply (no device needed)
int dmv_debug_tridiagonal_expm(int k, const double *a, const double *b, double z_re, double z_im, double *c) {
  API_BEGIN
  if (k < 1) throw std::runtime_error("empty matrix");
  std::vector<double> av(a, a + k), bv(b, b + (k - 1));
  const dmv::host::TridiagonalEigen T(av, bv);
  std::vector<dmv::host::cplx> out;
  T.exp_e1(dmv::host::cplx(z_re, z_im), out);
  for (int i = 0; i < k; ++i) { c[2 * i] = out[i].real(); c[2 * i + 1] = out[i].imag(); }
  API_END
}

}  // extern "C"
