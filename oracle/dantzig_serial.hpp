// TEST INFRASTRUCTURE ONLY — serial restatement of the reference's vendored ODE boxed Dantzig LCP solver, used by the oracle.
//   dSolveLCP   dart/external/odelcpsolver/lcp.cpp:780-1114   (driver loop, ratio test, cmd 1..6)
//   dLCP        lcp.cpp:362-775 (index sets C / N kept contiguous by physically permuting the problem, friction rows moved to the
//               end :491-501, lo/hi of friction rows fixed when the first one is reached :856-873)
// Pinned against the REAL reference code: tests/test_lcp.py compares it with dSolveLCP (oracle/_ref/libodelcp.so, or
// its answers recorded in tests/golden/dantzig_seeded.npz) on random and literal LCP instances.  The product has its OWN, warp-cooperative implementation
// (nimblephysics_b200/csrc/nb2_cw.cuh dantzig_solve) which is compared against this one through the solve chain — the two share
// no code.  Dense linear algebra: full symmetric A, L D L^T of A[C,C] appended row by row, rebuilt when an index leaves C.
#pragma once
#include <math.h>

#ifndef NB2_HD
#define NB2_HD inline
#endif

namespace nb2 {

#ifndef NB2_LCP_MAX
#define NB2_LCP_MAX 48  // max LCP dimension handled per world (16 contacts x 3 rows)
#endif

// strided pointer: element i of a per-world array lives at p[i * ST].  On the device the LCP workspace of the 32 worlds
// of a warp is interleaved [word][lane] (ST = 32) so that the warp-uniform parts of the pipeline touch one 256-byte line
// per access; the host builds (oracle, tests) use ST = 1.
template <class T, int ST> struct SP {
  T* p;
  NB2_HD T& operator[](int i) const { return p[(size_t)i * ST]; }
  NB2_HD T& operator[](size_t i) const { return p[i * ST]; }
  NB2_HD SP operator+(int k) const { SP r; r.p = p + (size_t)k * ST; return r; }
  NB2_HD SP operator+(size_t k) const { SP r; r.p = p + k * ST; return r; }
};

template <class PD, class PI, class PB>
struct DantzigWorkT {
  // all arrays of length n (or n*n) in fp64; caller allocates
  PD A;     // n*n, row-major, full symmetric; permuted in place
  PD x;     // n   (out)
  PD b;     // n
  PD w;     // n   (out)
  PD lo;    // n
  PD hi;    // n
  PD L;     // n*n
  PD d;     // n
  PD delta_x;
  PD delta_w;
  PD Dell;
  PD ell;
  PD tmp;
  PI findex;   // n
  PI p;        // n
  PI C;        // n
  PB state;    // n
};
typedef DantzigWorkT<double*, int*, unsigned char*> DantzigWork;

template <class DW> NB2_HD void dz_swap_problem(const DW& W, int n, int i1, int i2) {
  if (i1 == i2) return;
  // rows then columns; four elements per batch with all loads issued before the stores (in-order issue: "load, store,
  // load, store" would keep a single load in flight)
  for (int k0 = 0; k0 < n; k0 += 4) {
    double ta[4], tb[4];
#pragma unroll
    for (int u = 0; u < 4; u++) if (k0 + u < n) { ta[u] = W.A[i1 * n + k0 + u]; tb[u] = W.A[i2 * n + k0 + u]; }
#pragma unroll
    for (int u = 0; u < 4; u++) if (k0 + u < n) { W.A[i1 * n + k0 + u] = tb[u]; W.A[i2 * n + k0 + u] = ta[u]; }
  }
  for (int k0 = 0; k0 < n; k0 += 4) {
    double ta[4], tb[4];
#pragma unroll
    for (int u = 0; u < 4; u++) if (k0 + u < n) { ta[u] = W.A[(k0 + u) * n + i1]; tb[u] = W.A[(k0 + u) * n + i2]; }
#pragma unroll
    for (int u = 0; u < 4; u++) if (k0 + u < n) { W.A[(k0 + u) * n + i1] = tb[u]; W.A[(k0 + u) * n + i2] = ta[u]; }
  }
#define NB2_SW(arr, T) { T t = W.arr[i1]; W.arr[i1] = W.arr[i2]; W.arr[i2] = t; }
  NB2_SW(x, double) NB2_SW(b, double) NB2_SW(w, double) NB2_SW(lo, double) NB2_SW(hi, double)
  NB2_SW(p, int) NB2_SW(state, unsigned char) NB2_SW(findex, int)
#undef NB2_SW
}

// L D L^T of A[C,C] (C in factor order); d holds the reciprocals like ODE's m_d
template <class DW> NB2_HD void dz_factor(const DW& W, int n, int nC) {
  for (int i = 0; i < nC; i++) {
    const auto Ai = W.A + (size_t)W.C[i] * n;
    for (int j = 0; j <= i; j++) {
      double s = Ai[W.C[j]];
#pragma unroll 4
      for (int k = 0; k < j; k++) s -= W.L[i * n + k] * W.L[j * n + k] / W.d[k];
      if (j < i) W.L[i * n + j] = s * W.d[j];
      else W.d[i] = 1.0 / s;
    }
  }
}

// append index (physical slot i, about to be swapped into slot nC) to the factor using the ell/Dell of the latest
// dz_solve1(.., i, ..) — exactly what transfer_i_to_C does (lcp.cpp:503-535); O(nC) instead of a refactorisation
template <class DW> NB2_HD void dz_append_from_solve1(const DW& W, int n, int nC, int i) {
  double s = W.A[(size_t)i * n + i];
  for (int j = 0; j < nC; j++) { W.L[nC * n + j] = W.ell[j]; s -= W.ell[j] * W.Dell[j]; }
  W.d[nC] = 1.0 / s;
}

// solve1 (lcp.cpp:703-753): Dell = L \ A[C,i] ; ell = Dell .* d ; a[C] = -dir * L^T \ ell
template <class DW, class PA> NB2_HD void dz_solve1(const DW& W, int n, int nC, PA a, int i, int dir, bool only_transfer) {
  if (nC <= 0) return;
  const auto Ai = W.A + (size_t)i * n;
  for (int j = 0; j < nC; j++) {
    double s = Ai[W.C[j]];
#pragma unroll 4
    for (int k = 0; k < j; k++) s -= W.L[j * n + k] * W.Dell[k];
    W.Dell[j] = s;
  }
  for (int j = 0; j < nC; j++) W.ell[j] = W.Dell[j] * W.d[j];
  if (only_transfer) return;
  for (int j = 0; j < nC; j++) W.tmp[j] = W.ell[j];
  for (int j = nC - 1; j >= 0; j--) {
    double s = W.tmp[j];
#pragma unroll 4
    for (int k = j + 1; k < nC; k++) s -= W.L[k * n + j] * W.tmp[k];
    W.tmp[j] = s;
  }
  if (dir > 0) for (int j = 0; j < nC; j++) a[W.C[j]] = -W.tmp[j];
  else for (int j = 0; j < nC; j++) a[W.C[j]] = W.tmp[j];
}

// returns 1 on success, 0 on early termination (s <= 0), -1 when the iteration cap is hit
template <class DW> NB2_HD int dantzig_solve(const DW& W, int n, bool early_termination) {
  const double INF = HUGE_VAL;
  int nC = 0, nN = 0;
  for (int k = 0; k < n; k++) { W.x[k] = 0.0; W.w[k] = 0.0; W.p[k] = k; W.state[k] = 0; }
  // (no unbounded rows in contact problems: nub stays 0; an unbounded row would be lo=-inf & hi=+inf & findex<0)
  int nub = 0;
  for (int k = 0; k < n; k++) {
    if (W.findex[k] >= 0) continue;
    if (W.lo[k] == -INF && W.hi[k] == INF) { dz_swap_problem(W, n, nub, k); nub++; }
  }
  if (nub > 0) {
    for (int k = 0; k < nub; k++) W.C[k] = k;
    dz_factor(W, n, nub);
    // x = A[0:nub,0:nub] \ b
    for (int j = 0; j < nub; j++) { double s = W.b[j]; for (int k = 0; k < j; k++) s -= W.L[j * n + k] * W.tmp[k]; W.tmp[j] = s; }
    for (int j = 0; j < nub; j++) W.tmp[j] *= W.d[j];
    for (int j = nub - 1; j >= 0; j--) { double s = W.tmp[j]; for (int k = j + 1; k < nub; k++) s -= W.L[k * n + j] * W.tmp[k]; W.tmp[j] = s; W.x[j] = s; }
    nC = nub;
  }
  // move friction rows to the end (lcp.cpp:491-501)
  {
    int num_at_end = 0;
    for (int k = n - 1; k >= nub; k--) {
      if (W.findex[k] >= 0) { dz_swap_problem(W, n, k, n - 1 - num_at_end); num_at_end++; }
    }
  }
  bool hit_first_friction_index = false;
  long iter_cap = 200L * n + 1000;
  for (int i = nub; i < n; i++) {
    if (!hit_first_friction_index && W.findex[i] >= 0) {
      for (int j = 0; j < n; j++) W.delta_w[W.p[j]] = W.x[j];
      for (int k = i; k < n; k++) {
        const double wfk = W.delta_w[W.findex[k]];
        if (wfk == 0) { W.hi[k] = 0; W.lo[k] = 0; }
        else { W.hi[k] = fabs(W.hi[k] * wfk); W.lo[k] = -W.hi[k]; }
      }
      hit_first_friction_index = true;
    }
    {
      const auto Ai = W.A + (size_t)i * n;
      double s = 0.0;
#pragma unroll 4
      for (int k = 0; k < nC; k++) s += Ai[k] * W.x[k];
      double s2 = 0.0;
#pragma unroll 4
      for (int k = 0; k < nN; k++) s2 += Ai[nC + k] * W.x[nC + k];
      W.w[i] = s + s2 - W.b[i];
    }
    if (W.lo[i] == 0 && W.w[i] >= 0) { nN++; W.state[i] = 0; }
    else if (W.hi[i] == 0 && W.w[i] <= 0) { nN++; W.state[i] = 1; }
    else if (W.w[i] == 0) {
      dz_solve1(W, n, nC, W.delta_x, i, 0, true);
      dz_append_from_solve1(W, n, nC, i);
      dz_swap_problem(W, n, nC, i);
      W.C[nC] = nC; nC++;
    } else {
      for (;;) {
        if (--iter_cap < 0) return -1;
        int dir; double dirf;
        if (W.w[i] <= 0) { dir = 1; dirf = 1.0; } else { dir = -1; dirf = -1.0; }
        dz_solve1(W, n, nC, W.delta_x, i, dir, false);
        // delta_w(N) = A(N,C) delta_x(C) + dir * A(N,i) ; delta_w(i) = A(i,C) delta_x(C) + A(i,i) dirf
        for (int k = 0; k < nN; k++) {
          const auto Ak = W.A + (size_t)(nC + k) * n;
          double s = 0.0;
#pragma unroll 4
          for (int j = 0; j < nC; j++) s += Ak[j] * W.delta_x[j];
          W.delta_w[nC + k] = s;
        }
        {
          const auto Ai = W.A + (size_t)i * n;
          if (dir > 0) for (int k = 0; k < nN; k++) W.delta_w[nC + k] += Ai[nC + k];
          else for (int k = 0; k < nN; k++) W.delta_w[nC + k] -= Ai[nC + k];
          double s = 0.0;
#pragma unroll 4
          for (int j = 0; j < nC; j++) s += Ai[j] * W.delta_x[j];
          W.delta_w[i] = s + Ai[i] * dirf;
        }
        int cmd = 1, si = 0;
        double s = -W.w[i] / W.delta_w[i];
        if (dir > 0) {
          if (W.hi[i] < INF) { double s2 = (W.hi[i] - W.x[i]) * dirf; if (s2 < s) { s = s2; cmd = 3; } }
        } else {
          if (W.lo[i] > -INF) { double s2 = (W.lo[i] - W.x[i]) * dirf; if (s2 < s) { s = s2; cmd = 2; } }
        }
        for (int k = 0; k < nN; k++) {
          const int ik = nC + k;
          if (!W.state[ik] ? W.delta_w[ik] < 0 : W.delta_w[ik] > 0) {
            if (W.lo[ik] == 0 && W.hi[ik] == 0) continue;
            double s2 = -W.w[ik] / W.delta_w[ik];
            if (s2 < s) { s = s2; cmd = 4; si = ik; }
          }
        }
        for (int k = nub; k < nC; k++) {
          if (W.delta_x[k] < 0 && W.lo[k] > -INF) { double s2 = (W.lo[k] - W.x[k]) / W.delta_x[k]; if (s2 < s) { s = s2; cmd = 5; si = k; } }
          if (W.delta_x[k] > 0 && W.hi[k] < INF) { double s2 = (W.hi[k] - W.x[k]) / W.delta_x[k]; if (s2 < s) { s = s2; cmd = 6; si = k; } }
        }
        if (s <= 0.0) {
          if (early_termination) return 0;
          for (int k = i; k < n; k++) { W.x[k] = 0; W.w[k] = 0; }
          goto unpermute;  // the reference reports success in this case (lcp.cpp:1044-1050, 1113)
        }
        for (int k = 0; k < nC; k++) W.x[k] += s * W.delta_x[k];
        W.x[i] += s * dirf;
        for (int k = 0; k < nN; k++) W.w[nC + k] += s * W.delta_w[nC + k];
        W.w[i] += s * W.delta_w[i];
        switch (cmd) {
          case 1: W.w[i] = 0; dz_append_from_solve1(W, n, nC, i); dz_swap_problem(W, n, nC, i); W.C[nC] = nC; nC++; break;
          case 2: W.x[i] = W.lo[i]; W.state[i] = 0; nN++; break;
          case 3: W.x[i] = W.hi[i]; W.state[i] = 1; nN++; break;
          case 4:  // transfer_i_from_N_to_C (lcp.cpp:538-590): its own forward solve, then append
            W.w[si] = 0;
            dz_solve1(W, n, nC, W.delta_x, si, 0, true);
            dz_append_from_solve1(W, n, nC, si);
            dz_swap_problem(W, n, nC, si); W.C[nC] = nC; nN--; nC++;
            break;
          case 5:
          case 6: {
            if (cmd == 5) { W.x[si] = W.lo[si]; W.state[si] = 0; } else { W.x[si] = W.hi[si]; W.state[si] = 1; }
            // transfer_i_from_C_to_N (lcp.cpp:602-646): drop si from the factor order, rename the slot nC-1 -> si
            int j = 0, last_idx = -1;
            for (; j < nC; j++) {
              if (W.C[j] == nC - 1) last_idx = j;
              if (W.C[j] == si) {
                int k;
                if (last_idx == -1) { for (k = j + 1; k < nC; k++) if (W.C[k] == nC - 1) break; }
                else k = last_idx;
                W.C[k] = W.C[j];
                for (int m = j; m < nC - 1; m++) W.C[m] = W.C[m + 1];
                break;
              }
            }
            dz_swap_problem(W, n, si, nC - 1);
            nN++; nC--;
            dz_factor(W, n, nC);
            break;
          }
        }
        if (cmd <= 3) break;
      }
    }
  }
unpermute:
  for (int j = 0; j < n; j++) W.tmp[j] = W.x[j];
  for (int j = 0; j < n; j++) W.x[W.p[j]] = W.tmp[j];
  for (int j = 0; j < n; j++) W.tmp[j] = W.w[j];
  for (int j = 0; j < n; j++) W.w[W.p[j]] = W.tmp[j];
  return 1;
}

}  // namespace nb2
