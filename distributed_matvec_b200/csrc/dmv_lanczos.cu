// dmv_lanczos.cu -- dmv_lanczos: ground state by Lanczos with all vectors resident in HBM (the consumer of the product;
// the reference hands its product to PRIMME, src/Diagonalize.chpl:134-225).
#include "dmv_dense.h"
#include "dmv_solve.h"

extern "C" {

// ---- Lanczos ground-state solver on the device ("next" row f3): the consumer of the product.  The reference hands its
// matvec to PRIMME (src/Diagonalize.chpl:134-225); here the three-term recurrence, its dot products (NCCL all-reduce
// across ranks) and the Ritz-vector accumulation all stay in HBM, only alpha_j / beta_j (two doubles) visit the host.
int dmv_lanczos(dmv_context *ctx, int elt, int max_iters, double tol, uint64_t seed, double *eigenvalue,
                void *eigenvector, int *iterations, double *residual) {
  API_BEGIN
  SolverRun run(ctx, elt, "dmv_lanczos", false);
  if (max_iters < 1) throw std::runtime_error("max_iters must be positive");
  const int64_t n = run.n;
  const size_t words = run.words;
  const bool ce = run.ce;
  double *const vecs = run.vectors(4, "the work space of");   // v, v_prev, w and the Ritz vector
  double *scal = run.scalars(8);
  cudaStream_t st = run.st;
  auto reduce = [&]() {   // sum scal[0] over the ranks, bring it to the host
    run.all_reduce(scal, 1);
    double h = 0.0;
    CUDA_CHECK(cudaMemcpyAsync(&h, scal, sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    return h;
  };
  auto start_vector = [&](double *v) {
    launch_fill((int64_t)words, seed, (uint64_t)ctx->rank << 40, v, st);
    CUDA_CHECK(cudaMemsetAsync(scal, 0, 8 * sizeof(double), st));
    launch_dot(n, ce, v, v, scal, st);
    const double nrm = std::sqrt(reduce());
    if (!(nrm > 0.0)) throw std::runtime_error("empty basis");
    launch_scale((int64_t)words, 1.0 / nrm, v, v, false, st);
  };
  std::vector<double> alphas, betas, ritz;
  double theta = 0.0, res = 0.0;
  // every rank must take the same stopping decision: the Krylov space is exhausted at the GLOBAL dimension
  const int64_t n_global = run.global_states();
  {
    double *v = vecs, *u = vecs + words, *w = vecs + 2 * words;
    start_vector(v);
    double beta_prev = 0.0;
    for (int j = 0; j < max_iters; ++j) {
      run.product(v, w);
      CUDA_CHECK(cudaMemsetAsync(scal, 0, 8 * sizeof(double), st));
      launch_dot(n, ce, v, w, scal, st);
      const double alpha = reduce();
      const double coef[2] = {alpha, beta_prev};
      CUDA_CHECK(cudaMemcpyAsync(scal + 4, coef, sizeof(coef), cudaMemcpyHostToDevice, st));
      CUDA_CHECK(cudaMemsetAsync(scal, 0, sizeof(double), st));
      launch_lanczos_update(n, ce, w, v, j > 0 ? u : nullptr, scal + 4, scal, st);
      const double beta = std::sqrt(std::max(0.0, reduce()));
      alphas.push_back(alpha);
      theta = tridiagonal_lowest(alphas, betas, ritz);
      res = std::fabs(beta * ritz.back());
      const bool done = res <= tol * std::max(1.0, std::fabs(theta)) || beta <= 1e-14 * std::max(1.0, std::fabs(alpha)) ||
                        (int64_t)alphas.size() >= n_global;
      if (done || j + 1 == max_iters) break;
      betas.push_back(beta);
      launch_scale((int64_t)words, 1.0 / beta, w, w, false, st);
      double *t = u; u = v; v = w; w = t;   // v_prev <- v, v <- w / beta, old v_prev becomes scratch
      beta_prev = beta;
    }
  }
  if (eigenvalue) *eigenvalue = theta;
  if (iterations) *iterations = (int)alphas.size();
  if (residual) *residual = res;
  if (eigenvector) {
    // second pass with the stored alpha / beta (no dot products): Ritz vector = sum_j s_j v_j
    double *v = vecs, *u = vecs + words, *w = vecs + 2 * words, *acc = vecs + 3 * words;
    start_vector(v);
    CUDA_CHECK(cudaMemsetAsync(acc, 0, words * 8, st));
    const int k = (int)alphas.size();
    for (int j = 0; j < k; ++j) {
      launch_scale((int64_t)words, ritz[j], v, acc, true, st);
      if (j + 1 == k) break;
      run.product(v, w);
      const double coef[2] = {alphas[j], j > 0 ? betas[j - 1] : 0.0};
      CUDA_CHECK(cudaMemcpyAsync(scal + 4, coef, sizeof(coef), cudaMemcpyHostToDevice, st));
      launch_lanczos_update(n, ce, w, v, j > 0 ? u : nullptr, scal + 4, scal, st);
      CUDA_CHECK(cudaStreamSynchronize(st));   // coef lives on the host stack
      launch_scale((int64_t)words, 1.0 / betas[j], w, w, false, st);
      double *t = u; u = v; v = w; w = t;
    }
    CUDA_CHECK(cudaMemcpyAsync(eigenvector, acc, words * 8, cudaMemcpyDefault, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
  }
  check_status(ctx);
  API_END
}

// host-only self-check entry for the tridiagonal solver behind dmv_lanczos (no device needed)
int dmv_debug_tridiagonal_lowest(int k, const double *diag, const double *offdiag, double *eigenvalue, double *vector) {
  API_BEGIN
  if (k < 1) throw std::runtime_error("empty matrix");
  std::vector<double> a(diag, diag + k), b(offdiag, offdiag + (k - 1)), v;
  *eigenvalue = tridiagonal_lowest(a, b, v);
  if (vector) std::copy(v.begin(), v.end(), vector);
  API_END
}

}  // extern "C"
