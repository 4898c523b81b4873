// dmv_thermal.cu -- dmv_lanczos_quadrature: the finite-temperature Lanczos method (Jaklic & Prelovsek 1994), also known
// as stochastic Lanczos quadrature.  For each start vector r, M steps of the three-term recurrence give the tridiagonal
// T_M; its Gauss quadrature (nodes theta_k, weights |r|^2 Q_0k^2) estimates <r|f(H)|r> = sum_k w_k f(theta_k), exact for
// polynomials of degree below 2M.  The recurrences of a group of G start vectors share one batched product per step;
// their scalars stay on the device until the group is done, and only then visit the host, where each T_M is solved.
#include "dmv_dense.h"
#include "dmv_solve.h"

extern "C" {

// ---- finite-temperature Lanczos on the device (DESIGN.md section 3, "dmv_lanczos_quadrature").  No normalised copies:
// P = r_{j-1}, Q = r_j = beta_j v_j and W = H r_j (one dmv_matvec_batch over the G vectors of Q); k_quad_dot gives
// <r_j, W> = alpha_j beta_j^2, k_quad_update writes r_{j+1} over P together with |r_{j+1}|^2, then P and Q swap roles.
int dmv_lanczos_quadrature(dmv_context *ctx, int elt, int num_vectors, int steps, uint64_t seed, const void *start,
                           double *nodes, double *weights, int *steps_done, int *products) {
  API_BEGIN
  if (products) *products = 0;
  SolverRun run(ctx, elt, "dmv_lanczos_quadrature", true);
  if (num_vectors < 1) throw std::runtime_error("num_vectors must be positive");
  if (steps < 1) throw std::runtime_error("steps must be positive");
  if (!nodes || !weights) throw std::runtime_error("nodes and weights must not be null");
  const int P = run.P;
  const int64_t n = run.n;
  const size_t words = run.words;
  const bool ce = run.ce;
  cudaStream_t st = run.st;
  // group width G: the vectors one batched product shares (dmv_matvec_batch): four on k_gather, six doubles per state
  // on k_rows_batch, else one
  int width = 1;
  if (P == 1 && use_pull(ctx) && use_gather(ctx)) width = 4;
  else if (P == 1 && use_pull(ctx) && use_rows_batch(ctx)) width = kMaxBlockRhs / elt;
  const int G = std::min(width, num_vectors);
  double *partials = run.partials(quad_partials(G));
  // steps cap at the GLOBAL dimension (every rank takes the same decision, as dmv_lanczos)
  const int64_t n_global = run.global_states();
  if (n_global < 1) throw std::runtime_error("the basis is empty");
  const int M = (int)std::min<int64_t>(steps, n_global);
  // per step t and vector g: dot[2 (t G + g)] = <r_t, H r_t>, b2[2 (t G + g)] = |r_t|^2 (odd slots: imaginary parts)
  double *hist_dot = run.scalars((size_t)2 * G * (2 * (size_t)M + 1)), *hist_b2 = hist_dot + (size_t)2 * G * M;
  // the three vectors of every recurrence of a group
  double *const vecs = run.vectors(3 * G, "the work space of a group of " + std::to_string(G) + " recurrences, 3 G =");
  ctx->qd_group = G;
  const char *start_bytes = static_cast<const char *>(start);
  std::fill(nodes, nodes + (size_t)num_vectors * steps, 0.0);
  std::fill(weights, weights + (size_t)num_vectors * steps, 0.0);
  std::vector<double> hdot, hb2, a, b, nd, wt;
  int64_t prods = 0;
  for (int r0 = 0; r0 < num_vectors; r0 += G) {
    const int g = std::min(G, num_vectors - r0);   // this group's width: the step stride of the scalars too
    double *Pb = vecs, *Qb = Pb + (size_t)G * words, *Wb = Pb + (size_t)2 * G * words;
    auto dot_of = [&](int t) { return hist_dot + (size_t)2 * t * g; };
    auto b2_of = [&](int t) { return hist_b2 + (size_t)2 * t * g; };
    if (start) {
      if (words)
        CUDA_CHECK(cudaMemcpyAsync(Qb, start_bytes + (size_t)r0 * words * 8, (size_t)g * words * 8, cudaMemcpyDefault,
                                   st));
    } else {
      launch_quad_fill(n, ce, ctx->d_reps.ptr, seed, r0, g, Qb, st);
    }
    launch_quad_dot(n, ce, g, Qb, Qb, partials, b2_of(0), st);
    run.all_reduce(b2_of(0), 2 * g);
    if (start) {   // a zero start vector is an error: one synchronisation per group, before its recurrence
      hb2.resize((size_t)2 * g);
      CUDA_CHECK(cudaMemcpyAsync(hb2.data(), b2_of(0), sizeof(double) * 2 * g, cudaMemcpyDeviceToHost, st));
      CUDA_CHECK(cudaStreamSynchronize(st));
      for (int v = 0; v < g; ++v)
        if (!(hb2[2 * v] > 0.0))
          throw std::runtime_error("start vector " + std::to_string(r0 + v) + " is a zero vector");
    }
    for (int j = 0; j < M; ++j) {
      run.product(Qb, Wb, g);
      launch_quad_dot(n, ce, g, Qb, Wb, partials, dot_of(j), st);
      run.all_reduce(dot_of(j), 2 * g);
      if (j + 1 == M) break;
      launch_quad_update(n, ce, g, Pb, Qb, Wb, hist_dot, hist_b2, j, partials, b2_of(j + 1), st);
      run.all_reduce(b2_of(j + 1), 2 * g);
      std::swap(Pb, Qb);
    }
    prods += (int64_t)g * M;
    // the group's scalars come to the host once; every vector's T is read off them with the device's breakdown rule
    hdot.resize((size_t)2 * g * M);
    hb2.resize((size_t)2 * g * (M + 1));
    CUDA_CHECK(cudaMemcpyAsync(hdot.data(), hist_dot, sizeof(double) * hdot.size(), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(hb2.data(), hist_b2, sizeof(double) * hb2.size(), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    for (int v = 0; v < g; ++v) {
      a.clear();
      b.clear();
      for (int j = 0; j < M; ++j) {
        const double bj2 = hb2[2 * ((size_t)j * g + v)], dj = hdot[2 * ((size_t)j * g + v)];
        a.push_back(dj / bj2);
        if (j + 1 == M) break;
        const double bn2 = hb2[2 * ((size_t)(j + 1) * g + v)];
        if (!(bn2 > 0.0) || quad_breakdown(bn2, dj, bj2)) break;   // invariant Krylov space: T is exact
        b.push_back(std::sqrt(bn2));
      }
      tridiagonal_quadrature(a, b, nd, wt);
      const double norm2 = hb2[2 * v];
      const size_t row = (size_t)(r0 + v) * steps;
      for (size_t k = 0; k < nd.size(); ++k) {
        nodes[row + k] = nd[k];
        weights[row + k] = norm2 * wt[k];
      }
      if (steps_done) steps_done[r0 + v] = (int)a.size();
    }
  }
  if (products) *products = (int)std::min<int64_t>(prods, 2147483647);
  check_status(ctx);
  API_END
}

// host-only self-check entry for the Gauss quadrature behind dmv_lanczos_quadrature (no device needed): nodes ascending,
// weights = squared first components of the eigenvectors of T (they sum to 1)
int dmv_debug_tridiagonal_quadrature(int k, const double *a, const double *b, double *nodes, double *weights) {
  API_BEGIN
  if (k < 1) throw std::runtime_error("empty matrix");
  std::vector<double> av(a, a + k), bv(b, b + (k - 1)), nd, wt;
  dmv::host::tridiagonal_quadrature(av, bv, nd, wt);
  std::copy(nd.begin(), nd.end(), nodes);
  std::copy(wt.begin(), wt.end(), weights);
  API_END
}

}  // extern "C"
