// dmv_dense.h -- the small dense eigensolvers the device solvers run on the host: the symmetric tridiagonal ones of
// dmv_lanczos (dmv_lanczos.cu), dmv_expm_multiply (dmv_krylov.cu) and dmv_lanczos_quadrature (dmv_thermal.cu), and the
// Hermitian one of dmv_eigsh (dmv_eigsh.cu).  Host code only.
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <complex>
#include <numeric>
#include <stdexcept>
#include <vector>

namespace dmv { namespace host {

using cplx = std::complex<double>;

// Eigen-decomposition T = Q diag(lam) Q^T of the symmetric tridiagonal T (diagonal a[0..k), off-diagonal b[0..k-1)) by
// the implicit QL method with Wilkinson shifts; q[r * k + i] = component r of eigenvector i.  With first_row_only the
// rotations are applied to row 0 of Q alone (q holds k values): the Golub-Welsch quadrature needs no more, and that costs
// O(k^2) instead of O(k^3).  The rows of Q evolve independently, so row 0 is the same in both modes.
struct TridiagonalEigen {
  int k = 0, rows = 0;
  std::vector<double> lam, q;
  TridiagonalEigen(const std::vector<double> &a, const std::vector<double> &b, bool first_row_only = false) {
    k = (int)a.size();
    rows = first_row_only ? std::min(k, 1) : k;
    lam = a;
    std::vector<double> e(k, 0.0);
    for (int i = 0; i + 1 < k; ++i) e[i] = b[i];
    q.assign((size_t)rows * k, 0.0);
    for (int i = 0; i < rows; ++i) q[(size_t)i * k + i] = 1.0;
    std::vector<double> &d = lam;
    for (int l = 0; l < k; ++l) {
      for (int iter = 0;; ++iter) {
        int m = l;
        for (; m + 1 < k; ++m)   // the first negligible off-diagonal element at or below l splits the matrix
          if (std::fabs(e[m]) <= DBL_EPSILON * (std::fabs(d[m]) + std::fabs(d[m + 1]))) break;
        if (m == l) break;
        if (iter == 200) throw std::runtime_error("tridiagonal eigensolver did not converge");
        double g = (d[l + 1] - d[l]) / (2.0 * e[l]);   // Wilkinson shift from the leading 2 x 2 block
        double r = std::hypot(g, 1.0);
        g = d[m] - d[l] + e[l] / (g + std::copysign(r, g));
        double s = 1.0, c = 1.0, p = 0.0;
        bool underflow = false;
        for (int i = m - 1; i >= l; --i) {   // chase the bulge up with plane rotations
          double f = s * e[i];
          const double bb = c * e[i];
          r = std::hypot(f, g);
          e[i + 1] = r;
          if (r == 0.0) { d[i + 1] -= p; e[m] = 0.0; underflow = true; break; }
          s = f / r;
          c = g / r;
          g = d[i + 1] - p;
          r = (d[i] - g) * s + 2.0 * c * bb;
          p = s * r;
          d[i + 1] = g + p;
          g = c * r - bb;
          for (int t = 0; t < rows; ++t) {
            double *row = &q[(size_t)t * k];
            f = row[i + 1];
            row[i + 1] = s * row[i] + c * f;
            row[i] = c * row[i] - s * f;
          }
        }
        if (underflow) continue;
        d[l] -= p;
        e[l] = g;
        e[m] = 0.0;
      }
    }
  }
  // c = exp(w T) e_1 (needs every row)
  void exp_e1(cplx w, std::vector<cplx> &c) const {
    c.assign(k, cplx(0.0, 0.0));
    for (int i = 0; i < k; ++i) {
      const cplx f = std::exp(w * lam[i]) * q[i];   // q[0 * k + i]: first component of eigenvector i
      for (int r = 0; r < k; ++r) c[r] += q[(size_t)r * k + i] * f;
    }
  }
  // e_k^T phi_1(w T) e_1 with phi_1(x) = (e^x - 1) / x (needs every row)
  cplx phi1_last(cplx w) const {
    cplx s(0.0, 0.0);
    for (int i = 0; i < k; ++i) s += q[(size_t)(k - 1) * k + i] * q[i] * phi1(w * lam[i]);
    return s;
  }
  static cplx phi1(cplx x) {
    if (std::abs(x) >= 0.5) return (std::exp(x) - 1.0) / x;
    cplx s(1.0, 0.0);   // Taylor series sum_j x^j / (j + 1)!, Horner form; |x| < 0.5: the term j = 17 is < 1e-22
    for (int j = 17; j >= 1; --j) s = 1.0 + s * x / (double)(j + 1);
    return s;
  }
};

// Gauss quadrature of T (Golub & Welsch 1969): nodes = eigenvalues of T ascending, weights = squared first components
// of its eigenvectors (they sum to 1).
inline void tridiagonal_quadrature(const std::vector<double> &a, const std::vector<double> &b, std::vector<double> &nodes,
                                   std::vector<double> &weights) {
  const TridiagonalEigen T(a, b, true);
  std::vector<int> order(T.k);
  for (int i = 0; i < T.k; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return T.lam[x] < T.lam[y]; });
  nodes.resize(T.k);
  weights.resize(T.k);
  for (int i = 0; i < T.k; ++i) {
    nodes[i] = T.lam[order[i]];
    weights[i] = T.q[order[i]] * T.q[order[i]];
  }
}

// Lowest eigenpair of a symmetric tridiagonal matrix (diagonal a[0..k), off-diagonal b[0..k-1)): Sturm bisection for
// the eigenvalue, inverse iteration for the vector.  Host side of dmv_lanczos; k is at most a few hundred.
inline double tridiagonal_lowest(const std::vector<double> &a, const std::vector<double> &b, std::vector<double> &vec) {
  const int k = (int)a.size();
  double lo = a[0], hi = a[0];
  for (int i = 0; i < k; ++i) {
    const double r = (i > 0 ? std::fabs(b[i - 1]) : 0.0) + (i + 1 < k ? std::fabs(b[i]) : 0.0);
    lo = std::min(lo, a[i] - r);
    hi = std::max(hi, a[i] + r);
  }
  auto below = [&](double x) {   // number of eigenvalues < x
    int count = 0;
    double q = a[0] - x;
    for (int i = 0;; ++i) {
      if (q < 0.0) ++count;
      if (i + 1 == k) break;
      if (std::fabs(q) < 1e-300) q = q < 0 ? -1e-300 : 1e-300;
      q = a[i + 1] - x - b[i] * b[i] / q;
    }
    return count;
  };
  for (int it = 0; it < 200 && hi - lo > 4e-16 * std::max(1.0, std::max(std::fabs(lo), std::fabs(hi))); ++it) {
    const double mid = 0.5 * (lo + hi);
    if (below(mid) >= 1) hi = mid; else lo = mid;
  }
  const double theta = 0.5 * (lo + hi);
  // inverse iteration on (T - shift I): LU of a tridiagonal matrix with partial pivoting (the dgttrf / dgttrs scheme)
  vec.assign(k, 1.0 / std::sqrt((double)k));
  const double scale = std::max(1.0, std::max(std::fabs(lo), std::fabs(hi)));
  const double shift = theta - 1e-13 * scale;
  if (k > 1) {
    std::vector<double> dl(k - 1), d(k), du(k - 1), du2(k > 2 ? k - 2 : 0, 0.0);
    std::vector<int> piv(k - 1);
    for (int i = 0; i < k; ++i) d[i] = a[i] - shift;
    for (int i = 0; i + 1 < k; ++i) { dl[i] = b[i]; du[i] = b[i]; }
    const double tiny = 1e-300;
    for (int i = 0; i + 1 < k; ++i) {
      if (std::fabs(d[i]) >= std::fabs(dl[i])) {
        if (std::fabs(d[i]) < tiny) d[i] = tiny;
        const double f = dl[i] / d[i];
        dl[i] = f;
        d[i + 1] -= f * du[i];
        piv[i] = i;
      } else {
        const double f = d[i] / dl[i];
        d[i] = dl[i];
        dl[i] = f;
        const double t = du[i];
        du[i] = d[i + 1];
        d[i + 1] = t - f * d[i + 1];
        if (i + 2 < k) { du2[i] = du[i + 1]; du[i + 1] = -f * du[i + 1]; }
        piv[i] = i + 1;
      }
    }
    if (std::fabs(d[k - 1]) < tiny) d[k - 1] = tiny;
    for (int rep = 0; rep < 4; ++rep) {
      std::vector<double> x = vec;
      for (int i = 0; i + 1 < k; ++i) {
        if (piv[i] == i) x[i + 1] -= dl[i] * x[i];
        else { const double t = x[i]; x[i] = x[i + 1]; x[i + 1] = t - dl[i] * x[i]; }
      }
      x[k - 1] /= d[k - 1];
      if (k > 1) x[k - 2] = (x[k - 2] - du[k - 2] * x[k - 1]) / d[k - 2];
      for (int i = k - 3; i >= 0; --i) x[i] = (x[i] - du[i] * x[i + 1] - du2[i] * x[i + 2]) / d[i];
      double nrm = 0.0;
      for (double v : x) nrm += v * v;
      nrm = std::sqrt(nrm);
      if (!(nrm > 0.0) || !std::isfinite(nrm)) break;
      for (int i = 0; i < k; ++i) vec[i] = x[i] / nrm;
    }
  }
  if (k == 1) vec[0] = 1.0;
  return theta;
}

// Eigen-decomposition A = Q diag(lam) Q^H of a Hermitian k x k matrix (row-major; (A + A^H) / 2 is used) by the cyclic
// Jacobi method with complex rotations; lam ascending, q[r * k + i] = component r of eigenvector i.
struct HermitianEigen {
  int k = 0;
  std::vector<double> lam;
  std::vector<cplx> q;
  HermitianEigen(int n, const std::vector<cplx> &a_in) : k(n) {
    std::vector<cplx> a((size_t)n * n);
    double frob = 0.0;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        a[(size_t)i * n + j] = 0.5 * (a_in[(size_t)i * n + j] + std::conj(a_in[(size_t)j * n + i]));
        frob += std::norm(a[(size_t)i * n + j]);
      }
    for (int i = 0; i < n; ++i) a[(size_t)i * n + i] = a[(size_t)i * n + i].real();
    frob = std::sqrt(frob);
    std::vector<cplx> v((size_t)n * n, cplx(0.0, 0.0));
    for (int i = 0; i < n; ++i) v[(size_t)i * n + i] = 1.0;
    for (int sweep = 0;; ++sweep) {
      double off = 0.0;
      for (int p = 0; p < n; ++p)
        for (int r = p + 1; r < n; ++r) off += std::norm(a[(size_t)p * n + r]);
      if (off == 0.0 || std::sqrt(off) <= 1e-300 + 1e-22 * frob) break;
      if (sweep == 100) throw std::runtime_error("Hermitian Jacobi eigensolver did not converge");
      for (int p = 0; p < n; ++p)
        for (int r = p + 1; r < n; ++r) {
          const cplx apr = a[(size_t)p * n + r];
          const double g = std::abs(apr);
          if (g == 0.0) continue;
          const double app = a[(size_t)p * n + p].real(), arr = a[(size_t)r * n + r].real();
          if (sweep > 3 && std::fabs(app) + 100.0 * g == std::fabs(app) && std::fabs(arr) + 100.0 * g == std::fabs(arr)) {
            a[(size_t)p * n + r] = a[(size_t)r * n + p] = 0.0;   // negligible next to both diagonal elements
            continue;
          }
          // G = diag(1, conj(u)) * real rotation, u = a_pr / |a_pr|: G^H A G zeroes a_pr
          const cplx u = apr / g, cu = std::conj(u);
          const double theta = (arr - app) / (2.0 * g);
          const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::hypot(theta, 1.0));
          const double c = 1.0 / std::hypot(t, 1.0), s = t * c;
          for (int i = 0; i < n; ++i) {   // columns p, r of A and of V: A G
            cplx &x = a[(size_t)i * n + p], &y = a[(size_t)i * n + r];
            const cplx xp = x, yp = y;
            x = c * xp - s * cu * yp;
            y = s * xp + c * cu * yp;
            cplx &vx = v[(size_t)i * n + p], &vy = v[(size_t)i * n + r];
            const cplx vxp = vx, vyp = vy;
            vx = c * vxp - s * cu * vyp;
            vy = s * vxp + c * cu * vyp;
          }
          for (int j = 0; j < n; ++j) {   // rows p, r: G^H (A G)
            cplx &x = a[(size_t)p * n + j], &y = a[(size_t)r * n + j];
            const cplx xp = x, yp = y;
            x = c * xp - s * u * yp;
            y = s * xp + c * u * yp;
          }
          a[(size_t)p * n + r] = a[(size_t)r * n + p] = 0.0;
          a[(size_t)p * n + p] = a[(size_t)p * n + p].real();
          a[(size_t)r * n + r] = a[(size_t)r * n + r].real();
        }
    }
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(),
                     [&](int x, int y) { return a[(size_t)x * n + x].real() < a[(size_t)y * n + y].real(); });
    lam.resize(n);
    q.resize((size_t)n * n);
    for (int i = 0; i < n; ++i) {
      lam[i] = a[(size_t)order[i] * n + order[i]].real();
      for (int r = 0; r < n; ++r) q[(size_t)r * n + i] = v[(size_t)r * n + order[i]];
    }
  }
};

} }  // namespace dmv::host
