// dmv_eigsh.cu -- dmv_eigsh: the nev lowest eigenpairs of a Hermitian H by block Krylov-Schur (Stewart 2001; Zhou & Saad
// 2008), the solver the reference asks PRIMME for (src/Diagonalize.chpl).  Every vector stays in HBM: the products run
// through dmv_matvec_batch, the orthogonalisation through the block kernels of dmv_solver.cu, and only the reduced
// scalars visit the host, where the small dense Rayleigh-Ritz problem is solved by cyclic Jacobi.
#include <cfloat>
#include <complex>

#include "dmv_dense.h"
#include "dmv_solve.h"

extern "C" {

// ---- the nev lowest eigenpairs on the device (DESIGN.md section 3, "dmv_eigsh").  A cycle expands the basis a block
// of p vectors at a time until m vectors have products: one dmv_matvec_batch per block, the new block orthogonalised
// against the whole basis (block Gram + update kernels, DGKS second pass) and among itself (CholQR2), the coefficients
// kept in the dense projected matrix T = V^H H V.  Rayleigh-Ritz on T[:m, :m] (cyclic Jacobi) gives the Ritz pairs and
// their residual norms |B s_i| (B = the p rows of T below m); a restart keeps l Ritz vectors (k_block_rotate in place)
// and the residual block.
int dmv_eigsh(dmv_context *ctx, int elt, int nev, int block_size, int krylov_dim, double tol, int max_restarts,
              uint64_t seed, double *eigenvalues, void *eigenvectors, double *residuals, int *converged,
              int *products, int *restarts) {
  using dmv::host::cplx;
  API_BEGIN
  if (converged) *converged = 0;
  if (products) *products = 0;
  if (restarts) *restarts = 0;
  SolverRun run(ctx, elt, "dmv_eigsh", true);
  if (nev < 1) throw std::runtime_error("nev must be positive");
  if (!(tol > 0.0) || !std::isfinite(tol)) throw std::runtime_error("tol must be positive and finite");
  if (block_size < 0 || block_size > kMaxBlockRhs)
    throw std::runtime_error("block_size must be 0 (auto) or between 1 and " + std::to_string(kMaxBlockRhs));
  if (krylov_dim < 0 || krylov_dim > kMaxBlockVectors - 1)
    throw std::runtime_error("krylov_dim must be 0 (auto) or between 1 and " + std::to_string(kMaxBlockVectors - 1));
  if (max_restarts < 0) throw std::runtime_error("max_restarts must not be negative");
  if (!eigenvalues) throw std::runtime_error("eigenvalues must not be null");
  const int64_t n = run.n;
  const size_t words = run.words;
  const bool ce = run.ce;
  cudaStream_t st = run.st;
  // scalars: [kH, kH + 2 * (65 * 6 + 36)) Gram results, [kN, kN + 12) norms of an update, [kC, ...) coefficients of an
  // update (J x R complex), [kS, ...) the coefficient matrix of a rotation (k x l complex)
  constexpr int kH = 0, kN = 1024, kC = 1040, kS = kC + 2 * kMaxBlockVectors * kMaxBlockRhs;
  double *scal = run.scalars(kS + 2 * kMaxBlockVectors * kMaxBlockVectors);
  double *partials = run.partials(block_gram_partials());
  const int64_t n_global = run.global_states();   // every rank takes its decisions from the GLOBAL dimension
  if (nev > n_global)
    throw std::runtime_error("nev = " + std::to_string(nev) + " exceeds the dimension of the space, " +
                             std::to_string(n_global));
  // block size p (auto: the vectors one k_gather / k_rows_batch launch shares) and basis size m
  const int p = (int)std::min<int64_t>(block_size ? block_size : std::min(nev, ce ? 3 : 4), n_global);
  if (krylov_dim && krylov_dim + p > kMaxBlockVectors)
    throw std::runtime_error("krylov_dim + block_size must be at most " + std::to_string(kMaxBlockVectors));
  const int m_req = krylov_dim ? krylov_dim : std::min(kMaxBlockVectors - p, std::max(32, 2 * nev + 4 * p));
  const int m = (int)std::min<int64_t>(m_req, n_global);
  if (m < n_global && nev + 2 * p > m)
    throw std::runtime_error("krylov_dim = " + std::to_string(m) + " is too small: it needs at least nev + 2 * "
                             "block_size = " + std::to_string(nev + 2 * p) + " (and krylov_dim + block_size <= " +
                             std::to_string(kMaxBlockVectors) + ")");
  const int mp = m + p;
  double *const basis = run.vectors(mp, "the Krylov basis of krylov_dim + block_size =",
                                    "; use a smaller krylov_dim or block_size");
  ctx->eg_block_vectors = ctx->eg_rotate_vectors = 0;
  auto slot = [&](int k) { return basis + (size_t)k * words; };
  auto list_of = [&](int first, int count) {
    VecList l{};
    for (int k = 0; k < count; ++k) l.p[k] = slot(first + k);
    return l;
  };
  std::vector<double> hbuf(2 * (kMaxBlockVectors * kMaxBlockRhs + kMaxBlockRhs * kMaxBlockRhs));
  // <V_k, W_r> (k < J) and <W_r, W_s> for the q vectors W at slots [w, w + q), summed over the ranks
  auto gram = [&](int J, int w, int q) {
    const int width = J * q + q * q;
    launch_block_gram(n, ce, list_of(0, J), J, slot(w), n, q, partials, scal + kH, st);
    ctx->eg_block_vectors += J + q;
    run.all_reduce(scal + kH, 2 * width);
    CUDA_CHECK(cudaMemcpyAsync(hbuf.data(), scal + kH, sizeof(double) * 2 * width, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::vector<cplx> h(width);
    for (int t = 0; t < width; ++t) h[t] = cplx(hbuf[2 * t], hbuf[2 * t + 1]);
    return h;
  };
  // W_r -= sum_{k < J} c[k q + r] V_k; returns |W_r|^2 after, summed over the ranks
  auto update = [&](int J, int w, int q, const std::vector<cplx> &c) {
    std::vector<double> cd(2 * (size_t)J * q);
    for (int t = 0; t < J * q; ++t) { cd[2 * t] = c[t].real(); cd[2 * t + 1] = c[t].imag(); }
    if (J) CUDA_CHECK(cudaMemcpyAsync(scal + kC, cd.data(), sizeof(double) * cd.size(), cudaMemcpyHostToDevice, st));
    launch_block_update(n, ce, list_of(0, J), J, scal + kC, slot(w), n, q, partials, scal + kN, st);
    ctx->eg_block_vectors += J + 2 * q;
    run.all_reduce(scal + kN, 2 * q);
    double nb[2 * kMaxBlockRhs];
    CUDA_CHECK(cudaMemcpyAsync(nb, scal + kN, sizeof(double) * 2 * q, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::vector<double> nrm(q);
    for (int r = 0; r < q; ++r) nrm[r] = std::max(0.0, nb[2 * r]);
    return nrm;
  };
  // slots [first, first + l) <- slots [first, first + k) * S (S: k x l, row-major)
  auto rotate = [&](int first, int k, int l, const std::vector<cplx> &S) {
    std::vector<double> sd(2 * (size_t)k * l);
    for (size_t t = 0; t < (size_t)k * l; ++t) { sd[2 * t] = S[t].real(); sd[2 * t + 1] = S[t].imag(); }
    CUDA_CHECK(cudaMemcpyAsync(scal + kS, sd.data(), sizeof(double) * sd.size(), cudaMemcpyHostToDevice, st));
    launch_block_rotate(n, ce, list_of(first, k), k, l, scal + kS, st);
    ctx->eg_rotate_vectors += k + l;
  };
  int draws = 0;
  // a fresh direction at slot s, orthonormal to slots [0, s); zero once the basis spans the whole space
  auto fresh = [&](int s) {
    if ((int64_t)s >= n_global) {
      CUDA_CHECK(cudaMemsetAsync(slot(s), 0, words * 8, st));
      return;
    }
    for (int attempt = 0;; ++attempt) {
      if (attempt == 8) throw std::runtime_error("dmv_eigsh: no fresh direction orthogonal to the basis");
      launch_fill((int64_t)words, seed + 1 + (uint64_t)draws++, (uint64_t)ctx->rank << 40, slot(s), st);
      const double before = std::sqrt(std::real(gram(0, s, 1)[0]));
      double after = before;
      for (int pass = 0; pass < 2; ++pass) {
        std::vector<cplx> h = gram(s, s, 1);
        h.resize(s);
        after = std::sqrt(update(s, s, 1, h)[0]);
      }
      if (after > 1e-8 * before) {
        launch_scale((int64_t)words, 1.0 / after, slot(s), slot(s), false, st);
        return;
      }
    }
  };
  // Orthonormalise the q vectors at slots [J, J + q) against slots [0, J) and among themselves.  Returns coef
  // ((J + q) x q, row-major) with W_c(in) = sum_r coef[r q + c] V_r: column c of T for the vector W_c is the product of.
  auto orthonormalise = [&](int J, int q) {
    std::vector<cplx> coef((size_t)(J + q) * q, cplx(0.0, 0.0));
    std::vector<cplx> h = gram(J, J, q);
    std::vector<double> before(q);
    for (int c = 0; c < q; ++c) before[c] = std::sqrt(std::max(0.0, h[J * q + c * q + c].real()));
    if (J > 0) {
      bool again = false;
      for (int pass = 0; pass < 2 && (pass == 0 || again); ++pass) {
        if (pass) h = gram(J, J, q);
        h.resize((size_t)J * q);
        for (int t = 0; t < J * q; ++t) coef[t] += h[t];
        const std::vector<double> after = update(J, J, q, h);
        again = false;   // DGKS: a second pass when a vector lost most of its norm
        for (int c = 0; c < q; ++c) again |= after[c] < 0.49 * before[c] * before[c];
      }
    }
    // CholQR2: G = W^H W = R^H R, W <- W R^-1, twice.  A pivot below 1e-4 of its column's norm (an ill-conditioned or
    // rank-deficient block) sends the block to the column-by-column path below instead.
    std::vector<cplx> rtot((size_t)q * q, cplx(0.0, 0.0));
    for (int c = 0; c < q; ++c) rtot[c * q + c] = 1.0;
    bool by_column = false;
    for (int pass = 0; pass < 2 && !by_column; ++pass) {
      const std::vector<cplx> g = gram(0, J, q);
      std::vector<cplx> R((size_t)q * q, cplx(0.0, 0.0));
      for (int j = 0; j < q && !by_column; ++j) {
        double d = g[j * q + j].real();
        for (int i = 0; i < j; ++i) d -= std::norm(R[i * q + j]);
        const double rjj = std::sqrt(std::max(d, 0.0));
        if (!(rjj > 1e-4 * std::sqrt(std::max(g[j * q + j].real(), 0.0))) || !(rjj > 1e-12 * before[j])) {
          by_column = true;
          break;
        }
        R[j * q + j] = rjj;
        for (int l = j + 1; l < q; ++l) {
          cplx s = g[j * q + l];
          for (int i = 0; i < j; ++i) s -= std::conj(R[i * q + j]) * R[i * q + l];
          R[j * q + l] = s / rjj;
        }
      }
      if (by_column) break;
      std::vector<cplx> Ri((size_t)q * q, cplx(0.0, 0.0));   // R^-1, upper triangular
      for (int j = 0; j < q; ++j) {
        Ri[j * q + j] = 1.0 / R[j * q + j];
        for (int i = j - 1; i >= 0; --i) {
          cplx s(0.0, 0.0);
          for (int t = i + 1; t <= j; ++t) s += R[i * q + t] * Ri[t * q + j];
          Ri[i * q + j] = -s / R[i * q + i];
        }
      }
      rotate(J, q, q, Ri);
      std::vector<cplx> nt((size_t)q * q, cplx(0.0, 0.0));   // rtot <- R rtot
      for (int i = 0; i < q; ++i)
        for (int j = 0; j < q; ++j)
          for (int t = 0; t < q; ++t) nt[i * q + j] += R[i * q + t] * rtot[t * q + j];
      rtot = nt;
    }
    if (!by_column) {
      for (int i = 0; i < q; ++i)
        for (int c = 0; c < q; ++c) coef[(size_t)(J + i) * q + c] = rtot[i * q + c];
      return coef;
    }
    // column by column (the first CholQR pass, if it ran, was a change of basis within the block: undo it in coef by
    // tracking W(in) = V coef + W rtot, then treat the columns of W one at a time with two full passes each)
    std::vector<cplx> wcoef = rtot;   // current W_c(in) = sum_r coef[r q + c] V_r + sum_i W_i(now) wcoef[i q + c]
    for (int c = 0; c < q; ++c) {
      const int s = J + c;
      const double ref = before[c] > 0.0 ? before[c] : 1.0;
      double nu = 0.0;
      std::vector<cplx> hc;
      for (int pass = 0; pass < 2; ++pass) {
        hc = gram(s, s, 1);
        hc.resize(s);
        // W_c(now) = sum_{r < s} hc_r V_r + W_c(new)
        for (int r = 0; r < s; ++r)
          for (int cc = 0; cc < q; ++cc) coef[(size_t)r * q + cc] += hc[r] * wcoef[c * q + cc];
        nu = std::sqrt(update(s, s, 1, hc)[0]);
      }
      double scale_norm = 0.0;   // norm of this column relative to the input it came from
      for (int cc = 0; cc < q; ++cc) scale_norm = std::max(scale_norm, std::abs(wcoef[c * q + cc]) * before[cc]);
      if (nu > 1e-12 * std::max(ref, scale_norm)) {
        launch_scale((int64_t)words, 1.0 / nu, slot(s), slot(s), false, st);
        for (int cc = 0; cc < q; ++cc) coef[(size_t)s * q + cc] += nu * wcoef[c * q + cc];
      } else {
        fresh(s);   // deflation: the coupling to this direction is 0
      }
    }
    return coef;
  };

  // ---- start block: p deterministic vectors from `seed`
  launch_fill((int64_t)words * p, seed, (uint64_t)ctx->rank << 40, slot(0), st);
  orthonormalise(0, p);
  std::vector<cplx> T((size_t)mp * mp, cplx(0.0, 0.0));
  int cur = 0, prods = 0, rst = 0, nconv = 0;
  std::vector<double> theta, res;
  std::vector<cplx> S;   // m x m Ritz vectors of the last Rayleigh-Ritz
  for (;;) {
    // expand: products of the block at [cur, cur + q) land at [cur + p, cur + p + q)
    while (cur < m) {
      const int q = std::min(p, m - cur), J = cur + p;
      run.product(slot(cur), slot(J), q);
      prods += q;
      const std::vector<cplx> coef = orthonormalise(J, q);
      for (int r = 0; r < J + q; ++r)
        for (int c = 0; c < q; ++c) T[(size_t)r * mp + cur + c] = coef[(size_t)r * q + c];
      cur += q;
    }
    // Rayleigh-Ritz on T[:m, :m]; residual of pair i: |B s_i| with B = T[m : m + p, :m]
    std::vector<cplx> A((size_t)m * m);
    for (int r = 0; r < m; ++r)
      for (int c = 0; c < m; ++c) A[(size_t)r * m + c] = T[(size_t)r * mp + c];
    const dmv::host::HermitianEigen E(m, A);
    theta = E.lam;
    S = E.q;
    std::vector<cplx> BS((size_t)p * m, cplx(0.0, 0.0));
    for (int r = 0; r < p; ++r)
      for (int c = 0; c < m; ++c) {
        const cplx b = T[(size_t)(m + r) * mp + c];
        if (b == cplx(0.0, 0.0)) continue;
        for (int i = 0; i < m; ++i) BS[(size_t)r * m + i] += b * S[(size_t)c * m + i];
      }
    res.assign(m, 0.0);
    for (int i = 0; i < m; ++i) {
      double s2 = 0.0;
      for (int r = 0; r < p; ++r) s2 += std::norm(BS[(size_t)r * m + i]);
      res[i] = std::sqrt(s2);
    }
    nconv = 0;
    for (int i = 0; i < nev; ++i) nconv += res[i] <= tol * std::max(1.0, std::fabs(theta[i]));
    if (nconv == nev || rst == max_restarts || m < nev + 2 * p) break;   // (m < nev + 2p: the whole space)
    // restart: keep l Ritz vectors, the middle of nev + p <= l <= m - p (half the spare Ritz vectors, half the space
    // for new directions), and the residual block behind them
    const int l = nev + p + (m - nev - 2 * p) / 2;
    std::vector<cplx> Sl((size_t)m * l);
    for (int r = 0; r < m; ++r)
      for (int i = 0; i < l; ++i) Sl[(size_t)r * l + i] = S[(size_t)r * m + i];
    rotate(0, m, l, Sl);
    CUDA_CHECK(cudaMemcpyAsync(slot(l), slot(m), (size_t)p * words * 8, cudaMemcpyDeviceToDevice, st));
    std::fill(T.begin(), T.end(), cplx(0.0, 0.0));
    for (int i = 0; i < l; ++i) T[(size_t)i * mp + i] = theta[i];
    for (int r = 0; r < p; ++r)
      for (int i = 0; i < l; ++i) T[(size_t)(l + r) * mp + i] = BS[(size_t)r * m + i];
    cur = l;
    ++rst;
  }
  // the wanted Ritz vectors into the first nev slots
  std::vector<cplx> Sn((size_t)m * nev);
  for (int r = 0; r < m; ++r)
    for (int i = 0; i < nev; ++i) Sn[(size_t)r * nev + i] = S[(size_t)r * m + i];
  rotate(0, m, nev, Sn);
  if (eigenvectors && words)
    CUDA_CHECK(cudaMemcpyAsync(eigenvectors, slot(0), (size_t)nev * words * 8, cudaMemcpyDefault, st));
  CUDA_CHECK(cudaStreamSynchronize(st));
  for (int i = 0; i < nev; ++i) {
    eigenvalues[i] = theta[i];
    if (residuals) residuals[i] = res[i];
  }
  if (converged) *converged = nconv;
  if (products) *products = prods;
  if (restarts) *restarts = rst;
  check_status(ctx);
  API_END
}

// host-only self-check entry for the dense Hermitian eigensolver behind dmv_eigsh (no device needed)
int dmv_debug_hermitian_eigen(int k, const double *a, double *eigenvalues, double *eigenvectors) {
  API_BEGIN
  if (k < 1) throw std::runtime_error("empty matrix");
  std::vector<dmv::host::cplx> A((size_t)k * k);
  for (size_t t = 0; t < A.size(); ++t) A[t] = dmv::host::cplx(a[2 * t], a[2 * t + 1]);
  const dmv::host::HermitianEigen E(k, A);
  for (int i = 0; i < k; ++i) eigenvalues[i] = E.lam[i];
  if (eigenvectors)
    for (size_t t = 0; t < A.size(); ++t) { eigenvectors[2 * t] = E.q[t].real(); eigenvectors[2 * t + 1] = E.q[t].imag(); }
  API_END
}

}  // extern "C"
