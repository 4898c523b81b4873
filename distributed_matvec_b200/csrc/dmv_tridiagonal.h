// dmv_tridiagonal.h -- the host eigensolver of a symmetric tridiagonal matrix shared by dmv_expm_multiply
// (dmv_krylov.cu) and dmv_lanczos_quadrature (dmv_thermal.cu).  Host code only.
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <complex>
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

} }  // namespace dmv::host
