// TEST INFRASTRUCTURE ONLY — fp64 restatement of the reference's boxed-LCP solve chain.
//   BoxedLcpConstraintSolver::solveLcp        dart/constraint/BoxedLcpConstraintSolver.cpp:352-789
//   LCPUtils::{isLCPSolutionValid, guessSolution, reduce, mergeLCPColumns, removeFriction, dropLCPColumn}
//                                             dart/constraint/LCPUtils.cpp:12-80, 86-140, 144-201, 346-444, 208-247, 452-533
//   PgsBoxedLcpSolver::solve                  dart/constraint/PgsBoxedLcpSolver.cpp:79-278 (defaults PgsBoxedLcpSolver.hpp:55-60)
//   ConstrainedGroupGradientMatrices::{constructMatrices, opportunisticallyStandardizeResults}
//                                             dart/neural/ConstrainedGroupGradientMatrices.cpp:482-872, 218-339
//   Dantzig: oracle/dantzig_serial.hpp (serial restatement, pinned against the reference's own dSolveLCP, tests/test_lcp.py)
// Eigen's completeOrthogonalDecomposition().solve (third-party, not part of the reference) is restated as the
// minimum-norm least-squares solution computed from a one-sided Jacobi SVD with Eigen's default rank threshold
// (eps * max(rows, cols) relative to the largest singular value / pivot).
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

#include "dantzig_serial.hpp"

namespace orc {

typedef std::vector<double> Vec;
struct Mat {
  int r = 0, c = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int r_, int c_) : r(r_), c(c_), a((size_t)r_ * c_, 0.0) {}
  double& operator()(int i, int j) { return a[(size_t)i * c + j]; }
  double operator()(int i, int j) const { return a[(size_t)i * c + j]; }
};

enum { NOT_CLAMPING = -1, CLAMPING = -2, ILLEGAL = -3, IRRELEVANT = -4 };  // ConstrainedGroupGradientMatrices.hpp:33-39

// min-norm least squares x = Q^+ b for a general m x n matrix (Hestenes one-sided Jacobi SVD on Q^T)
inline Vec pinv_solve(const Mat& Q, const Vec& b) {
  const int m = Q.r, n = Q.c;
  if (m == 0 || n == 0) return Vec(n, 0.0);
  // work on U = Q (m x n) columns; V accumulates rotations (n x n):  Q V = U, columns of U orthogonal at the end
  Mat U = Q, V(n, n);
  for (int i = 0; i < n; i++) V(i, i) = 1.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = 0.0;
    for (int p = 0; p < n - 1; p++) for (int q = p + 1; q < n; q++) {
      double alpha = 0, beta = 0, gamma = 0;
      for (int i = 0; i < m; i++) { alpha += U(i, p) * U(i, p); beta += U(i, q) * U(i, q); gamma += U(i, p) * U(i, q); }
      if (gamma == 0.0) continue;
      off = std::max(off, std::fabs(gamma) / std::sqrt(std::max(alpha * beta, 1e-300)));
      if (std::fabs(gamma) <= 1e-15 * std::sqrt(alpha * beta)) continue;
      double zeta = (beta - alpha) / (2.0 * gamma);
      double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
      double cs = 1.0 / std::sqrt(1.0 + t * t), sn = cs * t;
      for (int i = 0; i < m; i++) { double up = U(i, p), uq = U(i, q); U(i, p) = cs * up - sn * uq; U(i, q) = sn * up + cs * uq; }
      for (int i = 0; i < n; i++) { double vp = V(i, p), vq = V(i, q); V(i, p) = cs * vp - sn * vq; V(i, q) = sn * vp + cs * vq; }
    }
    if (off < 1e-15) break;
  }
  Vec sig(n);
  double smax = 0;
  for (int j = 0; j < n; j++) { double s = 0; for (int i = 0; i < m; i++) s += U(i, j) * U(i, j); sig[j] = std::sqrt(s); smax = std::max(smax, sig[j]); }
  const double thresh = smax * 2.220446049250313e-16 * std::max(m, n);
  // x = V diag(1/sig) (U/sig)^T b
  Vec x(n, 0.0);
  for (int j = 0; j < n; j++) {
    if (sig[j] <= thresh || sig[j] == 0) continue;
    double coef = 0;
    for (int i = 0; i < m; i++) coef += U(i, j) * b[i];
    coef /= (sig[j] * sig[j]);
    for (int i = 0; i < n; i++) x[i] += V(i, j) * coef;
  }
  return x;
}

inline bool lcp_valid(const Mat& A, const Vec& x, const Vec& b, const Vec& hi, const Vec& lo, const std::vector<int>& fi,
                      bool ignoreFriction) {
  const int n = (int)x.size();
  for (int i = 0; i < n; i++) {
    double v = -b[i];
    for (int j = 0; j < n; j++) v += A(i, j) * x[j];
    double up = hi[i], low = lo[i];
    if (fi[i] != -1) {
      if (ignoreFriction) { if (x[i] != 0) return false; continue; }
      up *= x[fi[i]]; low *= x[fi[i]];
    }
    const double tol = 1e-5;
    if (std::fabs(low) < tol && std::fabs(up) < tol && std::fabs(x[i]) < tol) {}
    else if (std::fabs(x[i] - low) < tol) { if (v < -tol) return false; }
    else if (std::fabs(x[i] - up) < tol) { if (v > tol) return false; }
    else if (x[i] > low && x[i] < up) { if (std::fabs(v) > tol) return false; }
    else return false;
  }
  return true;
}

inline Vec guess_solution(const Mat& A, const Vec& b, const std::vector<int>& fi) {
  const int n = (int)b.size();
  std::vector<int> cl;
  for (int i = 0; i < n; i++) { if (fi[i] == -1) { if (b[i] > 0) cl.push_back(i); } else cl.push_back(i); }
  const int nc = (int)cl.size();
  if (nc == n) return pinv_solve(A, b);
  if (nc == 0) return Vec(n, 0.0);
  Mat rA(nc, nc); Vec rb(nc);
  for (int r = 0; r < nc; r++) { rb[r] = b[cl[r]]; for (int c = 0; c < nc; c++) rA(r, c) = A(cl[r], cl[c]); }
  Vec rx = pinv_solve(rA, rb), x(n, 0.0);
  for (int i = 0; i < nc; i++) x[cl[i]] = rx[i];
  return x;
}

struct Problem { Mat A; Vec x, b, hi, lo; std::vector<int> fi; Mat mapOut; };

inline void merge_cols(Problem& P, int colA, int colB) {
  const int n = P.A.c;
  Mat newACols(n, n - 1), newMap(P.mapOut.r, n - 1);
  Vec nx(n - 1, 0), nb(n - 1, 0), nhi(n - 1, 0), nlo(n - 1, 0);
  std::vector<int> nfi(n - 1, 0);
  for (int i = 0; i < n; i++) {
    if (i == colB) { for (int r = 0; r < P.mapOut.r; r++) newMap(r, colA) += P.mapOut(r, i); }
    else {
      int ni = i > colB ? i - 1 : i;
      for (int r = 0; r < n; r++) newACols(r, ni) = P.A(r, i) * (i == colA ? 2.0 : 1.0);
      nx[ni] = P.x[i]; nb[ni] = P.b[i]; nhi[ni] = P.hi[i]; nlo[ni] = P.lo[i];
      if (P.fi[i] < colB) nfi[ni] = P.fi[i]; else if (P.fi[i] == colB) nfi[ni] = colA; else nfi[ni] = P.fi[i] - 1;
      for (int r = 0; r < P.mapOut.r; r++) newMap(r, ni) += P.mapOut(r, i);
    }
  }
  Mat nA(n - 1, n - 1);
  for (int i = 0; i < n; i++) { if (i == colB) continue; int ni = i > colB ? i - 1 : i; for (int c = 0; c < n - 1; c++) nA(ni, c) = newACols(i, c); }
  P.A = nA; P.x = nx; P.b = nb; P.hi = nhi; P.lo = nlo; P.fi = nfi; P.mapOut = newMap;
}
inline void drop_col(Problem& P, int col) {
  const int n = P.A.c;
  Mat newACols(n, n - 1), newMap(P.mapOut.r, n - 1);
  Vec nx(n - 1, 0), nb(n - 1, 0), nhi(n - 1, 0), nlo(n - 1, 0);
  std::vector<int> nfi(n - 1, 0);
  for (int i = 0; i < n; i++) {
    if (i == col) continue;
    int ni = i > col ? i - 1 : i;
    for (int r = 0; r < n; r++) newACols(r, ni) = P.A(r, i);
    nx[ni] = P.x[i]; nb[ni] = P.b[i]; nhi[ni] = P.hi[i]; nlo[ni] = P.lo[i];
    if (P.fi[i] < col) nfi[ni] = P.fi[i]; else if (P.fi[i] > col) nfi[ni] = P.fi[i] - 1;
    for (int r = 0; r < P.mapOut.r; r++) newMap(r, ni) += P.mapOut(r, i);
  }
  Mat nA(n - 1, n - 1);
  for (int i = 0; i < n; i++) { if (i == col) continue; int ni = i > col ? i - 1 : i; for (int c = 0; c < n - 1; c++) nA(ni, c) = newACols(i, c); }
  P.A = nA; P.x = nx; P.b = nb; P.hi = nhi; P.lo = nlo; P.fi = nfi; P.mapOut = newMap;
}
inline void reduce(Problem& P) {  // LCPUtils::reduce, MERGE_THRESHOLD 1e-4
  const int n0 = P.A.r;
  P.mapOut = Mat(n0, n0);
  for (int i = 0; i < n0; i++) P.mapOut(i, i) = 1.0;
  while (true) {
    const int n = P.A.c;
    bool found = false;
    for (int a = 0; a < n - 1 && !found; a++) for (int b = a + 1; b < n; b++) {
      double d2 = 0;
      for (int r = 0; r < n; r++) { double d = P.A(r, a) - P.A(r, b); d2 += d * d; }
      if (d2 < 1e-4 && std::fabs(P.b[a] - P.b[b]) < 1e-4 && P.fi[a] == P.fi[b] && P.hi[a] == P.hi[b] && P.lo[a] == P.lo[b]) {
        merge_cols(P, a, b); found = true; break;
      }
    }
    if (!found) break;
  }
}
inline void remove_friction(Problem& P) {
  const int n0 = P.A.r;
  P.mapOut = Mat(n0, n0);
  for (int i = 0; i < n0; i++) P.mapOut(i, i) = 1.0;
  std::vector<int> fi0 = P.fi;
  for (int i = (int)fi0.size() - 1; i >= 0; i--) if (fi0[i] != -1) drop_col(P, i);
}
inline Vec map_out(const Problem& P, const Vec& xr) {
  Vec x(P.mapOut.r, 0.0);
  for (int r = 0; r < P.mapOut.r; r++) for (int c = 0; c < P.mapOut.c; c++) x[r] += P.mapOut(r, c) * xr[c];
  return x;
}

inline bool run_dantzig(Problem& P, bool early) {  // clobbers P like the reference clobbers A,b,lo,hi
  const int n = (int)P.x.size();
  if (n == 0) return true;
  std::vector<double> A(P.A.a), L((size_t)n * n, 0.0), d(n, 0), w(n, 0), dx(n, 0), dw(n, 0), Dell(n, 0), ell(n, 0), tmp(n, 0);
  std::vector<int> p(n), C(n);
  std::vector<unsigned char> st(n);
  nb2::DantzigWork W{A.data(), P.x.data(), P.b.data(), w.data(), P.lo.data(), P.hi.data(), L.data(), d.data(), dx.data(), dw.data(),
                     Dell.data(), ell.data(), tmp.data(), P.fi.data(), p.data(), C.data(), st.data()};
  return nb2::dantzig_solve(W, n, early) == 1;
}

// PgsBoxedLcpSolver::solve with the default Option(30, 1e-6, 1e-3, 1e-9, false); A, b are clobbered
inline bool run_pgs(Problem& P) {
  const int n = (int)P.x.size();
  Mat& A = P.A; Vec& x = P.x; Vec& b = P.b;
  const int maxIter = 30; const double dxTol = 1e-6, relTol = 1e-3, epsDiv = 1e-9;
  std::vector<int> order;
  bool term = true;
  for (int i = 0; i < n; i++) {
    if (A(i, i) < epsDiv) { x[i] = 0.0; continue; }
    order.push_back(i);
    const double old_x = x[i];
    double nx = b[i];
    for (int j = 0; j < i; j++) nx -= A(i, j) * x[j];
    for (int j = i + 1; j < n; j++) nx -= A(i, j) * x[j];
    nx /= A(i, i);
    double hi_t = P.hi[i], lo_t = P.lo[i];
    if (P.fi[i] >= 0) { hi_t = P.hi[i] * x[P.fi[i]]; lo_t = -hi_t; }
    x[i] = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
    if (term && std::fabs(x[i] - old_x) > dxTol) term = false;
  }
  if (term) return true;
  for (int idx : order) { const double dm = 1.0 / A(idx, idx); b[idx] *= dm; for (int j = 0; j < n; j++) A(idx, j) *= dm; }
  for (int iter = 1; iter < maxIter; iter++) {
    term = true;
    for (int idx : order) {
      double nx = b[idx];
      const double old_x = x[idx];
      for (int j = 0; j < idx; j++) nx -= A(idx, j) * x[j];
      for (int j = idx + 1; j < n; j++) nx -= A(idx, j) * x[j];
      double hi_t = P.hi[idx], lo_t = P.lo[idx];
      if (P.fi[idx] >= 0) { hi_t = P.hi[idx] * x[P.fi[idx]]; lo_t = -hi_t; }
      x[idx] = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
      if (term && std::fabs(x[idx]) > epsDiv) { if (std::fabs((x[idx] - old_x) / x[idx]) > relTol) term = false; }
    }
    if (term) break;
  }
  return term;
}

// ------------------------------------------------------------------ classification + standardisation
struct Classifier {
  // registered LCP (ConstrainedGroupGradientMatrices::registerLCPResults)
  Mat A; Vec x, hi, lo, b, colNorms; std::vector<int> fi; double cfm = 0; bool ignoreFriction = false;
  Vec restitution;  // per row
  // outputs
  std::vector<int> mapping, clampIdx, ubIdx;
  bool standardized = false;

  void construct() {
    const int m = (int)x.size();
    mapping = fi; clampIdx.assign(m, -1); ubIdx.assign(m, -1);
    int nCl = 0, nUb = 0;
    for (int j = 0; j < m; j++) {
      if (colNorms[j] < 1e-9) { mapping[j] = NOT_CLAMPING; continue; }
      const double force = x[j];
      double up = hi[j], low = lo[j];
      const int fp = fi[j];
      if (fp != -1) { up *= x[fp]; low *= x[fp]; }
      if (std::fabs(force) < 1e-6) {  // CLAMPING_THRESHOLD
        if (fp != -1) {
          if (std::fabs(x[fp]) < 1e-6) mapping[j] = NOT_CLAMPING;
          else if (ignoreFriction) mapping[j] = NOT_CLAMPING;
          else { mapping[j] = CLAMPING; clampIdx[j] = nCl++; }
        } else mapping[j] = NOT_CLAMPING;
        continue;
      }
      const double tie = 1e-5;
      if ((x[j] > low + tie && x[j] < up - tie) || (low - x[j] > 1e-2 || x[j] - up > 1e-2)) { mapping[j] = CLAMPING; clampIdx[j] = nCl++; }
      else if (low - x[j] > 1e-2 || x[j] - up > 1e-2) { mapping[j] = ILLEGAL; }
      else if (fp != -1 && std::fabs(x[fp]) > 1e-9 && colNorms[fp] > 1e-9 && ((fp > j) || mapping[fp] == CLAMPING)) { mapping[j] = fp; ubIdx[j] = nUb++; }
      else mapping[j] = NOT_CLAMPING;
    }
    standardize();
  }

  void standardize() {
    standardized = true;
    const int m = (int)x.size();
    if (m == 0) return;
    int nCl = 0, nUb = 0;
    for (int j = 0; j < m; j++) { if (clampIdx[j] >= 0) nCl++; if (ubIdx[j] >= 0) nUb++; }
    if (nCl == 0) {
      Vec zero(m, 0.0);
      if (lcp_valid(A, zero, b, hi, lo, fi, ignoreFriction)) { x = zero; return; }
      standardized = false; return;
    }
    std::vector<int> cl(nCl), ub(nUb);
    for (int j = 0; j < m; j++) { if (clampIdx[j] >= 0) cl[clampIdx[j]] = j; if (ubIdx[j] >= 0) ub[ubIdx[j]] = j; }
    // E (nUb x nCl): +hi or +lo of the row, whichever bound x sits on (ConstrainedGroupGradientMatrices.cpp:800-846)
    Mat E(nUb, nCl);
    for (int u = 0; u < nUb; u++) {
      const int j = ub[u], fp = mapping[j];
      const double up = x[fp] * hi[j], low = x[fp] * lo[j];
      E(u, clampIdx[fp]) = (std::fabs(x[j] - up) < std::fabs(x[j] - low)) ? hi[j] : lo[j];
    }
    // Q = A[cl,cl] + A[cl,ub] E   (== A_c^T M^-1 (A_c + A_ub E) + cfm I, the registered A already carries the cfm)
    Mat Q(nCl, nCl);
    Vec bc(nCl), orig(nCl);
    for (int r = 0; r < nCl; r++) {
      bc[r] = b[cl[r]]; orig[r] = x[cl[r]];
      for (int c = 0; c < nCl; c++) {
        double q = A(cl[r], cl[c]);
        for (int u = 0; u < nUb; u++) q += A(cl[r], ub[u]) * E(u, c);
        Q(r, c) = q;
      }
    }
    Vec fc = pinv_solve(Q, bc);
    bool anyNewlyNotClamping = false;
    Vec nx(m, 0.0);
    for (int i = 0; i < m; i++) {
      if (clampIdx[i] != -1) {
        nx[i] = fc[clampIdx[i]];
        if (std::fabs(fc[clampIdx[i]]) < 1e-6 && std::fabs(x[i]) > 1e-6 && fi[i] == -1) anyNewlyNotClamping = true;
      }
      if (ubIdx[i] != -1) {
        const int fp = fi[i];
        const double origMult = orig[clampIdx[fp]] / x[i];
        const double clean = (std::fabs(origMult - hi[i]) < std::fabs(origMult - lo[i])) ? hi[i] : lo[i];
        nx[i] = fc[clampIdx[fp]] * clean;
      }
    }
    if (lcp_valid(A, nx, b, hi, lo, fi, ignoreFriction)) {
      x = nx;
      if (anyNewlyNotClamping) construct();
      return;
    }
    standardized = false;
  }
};

struct ChainResult {
  Vec x;
  std::vector<int> mapping;
  int status = 0;  // bit0 short-circuit used, bit1 dantzig ran, bit2 dantzig failed/invalid, bit3 pgs used, bit4 pgs failed -> friction dropped, bit5 NaN reset, bit6 final not standardized
  double cfm = 0;
};

// BoxedLcpConstraintSolver::solveLcp.  A: m x m (no cfm), x0: warm start (previous x if same size, else guess)
inline ChainResult solve_chain(const Mat& A_in, const Vec& b, const Vec& lo, const Vec& hi, const std::vector<int>& fi,
                               const Vec& x0, const Vec& restitution, double fallback_cfm) {
  const int n = (int)b.size();
  ChainResult R;
  Mat Agrad = A_in, Aback = A_in;
  Vec colNorms(n, 0.0);
  for (int c = 0; c < n; c++) for (int r = 0; r < n; r++) colNorms[c] += A_in(r, c) * A_in(r, c);
  double cfm = 0.0;
  Vec x = x0;
  bool success = false, shortCircuit = false, ignoredFriction = false;
  Classifier K;
  {
    K.A = Agrad; K.x = x; K.hi = hi; K.lo = lo; K.fi = fi; K.b = b; K.colNorms = colNorms; K.cfm = cfm; K.ignoreFriction = false; K.restitution = restitution;
    K.construct();
    success = K.standardized;
    if (success) x = K.x;
    shortCircuit = success;
    if (success) R.status |= 1;
  }
  if (!success) {
    R.status |= 2;
    Problem P; P.A = A_in; P.x = x; P.b = b; P.hi = hi; P.lo = lo; P.fi = fi;
    reduce(P);
    if (P.A.c < n) R.status |= 512;  // columns merged (informational)
    Problem Psolve = P;
    success = run_dantzig(Psolve, true);
    if (success) {
      x = map_out(P, Psolve.x);
      if (!lcp_valid(Agrad, x, b, hi, lo, fi, false)) success = false;
    }
    if (!success) R.status |= 4;
  }
  bool hasNaN = false;
  for (double v : x) if (std::isnan(v)) hasNaN = true;
  if (hasNaN) { success = false; for (double& v : x) v = 0; R.status |= 32; }
  if (!success) {
    cfm = fallback_cfm;
    for (int i = 0; i < n; i++) { Aback(i, i) += cfm; Agrad(i, i) += cfm; }
    R.status |= 8;
    Problem P; P.A = Aback; P.x = x0; P.b = b; P.hi = hi; P.lo = lo; P.fi = fi;  // mXBackup = x at entry
    reduce(P);
    if (P.A.c < n) R.status |= 512;
    Problem Psolve = P;
    success = run_pgs(Psolve);
    if (success) {
      x = map_out(P, Psolve.x);
      if (!lcp_valid(Agrad, x, b, hi, lo, fi, false)) success = false;
    }
  }
  if (!success) {
    ignoredFriction = true;
    R.status |= 16;
    Problem P; P.A = Aback; P.x = x0; P.b = b; P.hi = hi; P.lo = lo; P.fi = fi;
    remove_friction(P);
    for (double& v : P.x) v = 0;
    Problem Psolve = P;
    success = run_pgs(Psolve);
    x = map_out(P, Psolve.x);
  }
  hasNaN = false;
  for (double v : x) if (std::isnan(v)) hasNaN = true;
  if (hasNaN) { for (double& v : x) v = 0; R.status |= 32; }
  if (!shortCircuit) {
    K = Classifier();
    K.A = Agrad; K.x = x; K.hi = hi; K.lo = lo; K.fi = fi; K.b = b; K.colNorms = colNorms; K.cfm = cfm; K.ignoreFriction = ignoredFriction; K.restitution = restitution;
    K.construct();
    if (K.standardized) x = K.x; else R.status |= 64;
  }
  R.x = x; R.mapping = K.mapping; R.cfm = cfm;
  return R;
}

}  // namespace orc
