// Constrained forward dynamics with bilateral contacts, batched (DESIGN.md §6o).  k contacts (1 <= k <= NB2_MAX_CONTACT_BODIES), each a
// point p_i on a canonical body, constrain the rows of the point's world Jacobian J_i (nb2_jac.cuh): all six [omega ; pdot] rows, or the
// three linear rows of a point contact.  J [m, n] stacks them (m = 6k or 3k), Jdot the same rows of the Jacobian's time derivative, and
//   M qdd + h = tau + J^T lam ,   J qdd + Jdot qdot = -rho lam      (h: the bias, spring and damping forces of forward dynamics, §6k)
// so that  lam = -(J M^-1 J^T + rho I)^-1 (J qdd_free + Jdot qdot)  and  qdd = FD(tau + J^T lam).  lam_i is [torque about p_i ; force].
//
// ONE WARP PER WORLD, one world per block.  The program of a world is cfd_world below, a sequence of stages; `stage(f)` runs f(lane, nl) on
// every lane and then separates the stages (the kernels: a __syncwarp; the host build: the lanes one after the other, in any order).
// Working set (arithmetic type R, stride 1), after the dense-Jacobian kernel's (nb2_djac.cuh dj_layout with ST row slots):
//   J, Jdot, Y = (M^-1 J^T)^T [m][n]; the Cholesky factor [m][m]; c -> lam, mu, lambar [m]; the points p_i and pbar_i [4][3]; tau' [n];
//   the backward's seed qddbar [n], [dL/dq ; dL/dqdot] [2n], u = dL/dtau [n], offset gradients [2][4][3]; one node's seed block [6][n];
//   the point-Jacobian stages' scratch; the singular flag.
// Columns of M^-1 J^T: each row slot runs the B1 / B2 sweeps of the FD backward (fd_backward_stage stages 1-4) seeded with J_r^T, which
// leave M^-1 J_r^T in its lambda words, the row rounds of k_dj.
//
// Backward (L(qdd, w)): with the factor of J M^-1 J^T + rho I,
//   mu = (J M^-1 J^T + rho I)^-1 (lambar + Y qddbar),   g = qddbar - J^T mu,   u = M^-1 g = dL/dtau,
// and the FD backward seeded with g on the saved stream of FD(tau + J^T lam) gives its part of dL/dq, dL/dqdot and the inertia gradient.
// The rest comes from the point-Jacobian VJPs with rank-one seeds (u, lam, mu, qdd fixed):
//   dL/dq += d<lam, J u>/dq - d<mu, J qdd + Jdot qdot>/dq  (jpb_* with lam u^T - mu qdd^T, jpdb_* with -mu qdot^T),
//   dL/dqdot += -Jdot^T mu - d<mu, Jdot qdot>/dqdot|_Jdot (jpdb_*),   dL/do_i from both.
// A 6-D output is the wrench about the world origin, [lam_a + p x lam_l ; lam_l]; its seed wbar becomes lambar = [wbar_a ; wbar_l +
// wbar_a x p] and adds pbar = lam_l x wbar_a to the point, which jpdb_reduce carries to q and the offset with the point's own adjoint.
//
// Dense Jacobians (cfdj_world, §6p): the forward of cfd_world once, then the backward above per seed e_i, in rounds of ST seeds.
#pragma once
#include <math.h>

#include "nb2_djac.cuh"
#include "nb2_jac.cuh"

#define NB2_CFD_PIVOT_C 64  // a Cholesky pivot <= NB2_CFD_PIVOT_C * eps_R * max diagonal marks the world singular

namespace nb2 {

// the contacts of one call: canonical body, body <- node transform (R row-major 9, p 3), and whether they are point contacts (3 rows)
template <class R> struct CfdNodes {
  int k, point;
  int body[NB2_MAX_CONTACT_BODIES];
  R T[NB2_MAX_CONTACT_BODIES][12];
};
// k contacts from the host's canonical bodies and body <- node transforms [k][12] (fp64); unused entries -1 / 0
template <class R> inline CfdNodes<R> cfd_nodes(int k, int point, const int32_t* body, const double* T) {
  CfdNodes<R> N;
  N.k = k; N.point = point;
  for (int e = 0; e < NB2_MAX_CONTACT_BODIES; e++) {
    N.body[e] = e < k ? body[e] : -1;
    for (int c = 0; c < 12; c++) N.T[e][c] = e < k ? (R)T[12 * e + c] : R(0);
  }
  return N;
}
// one world's rows.  Forward: state [2n], tau [n], offsets ([k][3], or NULL), qdd [n], wrench [k][6 or 3].  Backward adds the seeds gqdd
// [n] and gw [k][6 or 3] and writes gstate [2n], gtau [n], goff [k][3] (or NULL) and gI (word-major [10 nb][wiB], or NULL).
template <class R> struct CfdRows {
  const R* state; const R* tau; const R* off; R* qdd; R* wrench;
  const R* gqdd; const R* gw; R* gstate; R* gtau; R* goff; double* gI;
  const double* wi; size_t wiB;
  R rho;
};

struct CfdLayout { DjLayout D; int m, oJ, oJd, oY, oA, oC, oMu, oLb, oP, oPb, oTau, oQb, oG, oU, oGo, oGb, oK, oFlag, total; };
NB2_HD CfdLayout cfd_layout(int nb, int n, int nslots, int nfree, int m, int st) {
  CfdLayout L;
  L.D = dj_layout(nb, n, nslots, nfree, true, st);
  L.m = m;
  L.oJ = L.D.total; L.oJd = L.oJ + m * n; L.oY = L.oJd + m * n; L.oA = L.oY + m * n;
  L.oC = L.oA + m * m; L.oMu = L.oC + m; L.oLb = L.oMu + m; L.oP = L.oLb + m; L.oPb = L.oP + 12;
  L.oTau = L.oPb + 12; L.oQb = L.oTau + n; L.oG = L.oQb + n; L.oU = L.oG + 2 * n; L.oGo = L.oU + n; L.oGb = L.oGo + 24;
  L.oK = L.oGb + 6 * n;
  int k = jpd_layout(n).total;
  if (jpb_layout(nb, n).total > k) k = jpb_layout(nb, n).total;
  if (jpdb_layout(nb, n).total > k) k = jpdb_layout(nb, n).total;
  L.oFlag = L.oK + ((k + 3) & ~3);
  L.total = L.oFlag + 4;
  return L;
}
template <class R> NB2_HD CfdLayout cfd_layout(const Nb2ModelDev<R>& M, int m, int st) { return cfd_layout(M.nb, M.ndof, M.nslots, M.nfree, m, st); }

template <class R> NB2_HD R cfd_nan() { return R(NAN); }

// row slot t of a round: the FD backward's B1 / B2 seeded with J_r^T (r < m), which leave M^-1 J_r^T in the slot's lambda words.  The slot's
// scratch is its own, so one thread sweeps every lane of the schedule in order.
template <class R, int ST>
NB2_HD void cfd_column(const Nb2ModelDev<R>& M, const CfdLayout& L, R* ws, const R* state, int r, int t, const double* wi, size_t wiB) {
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof;
  R* rb = ws + L.D.oB + t;
  for (int d = 0; d < 2 * n; d++) rb[(size_t)(BL.oSt + d) * ST] = state[d];
  for (int d = 0; d < n; d++) rb[(size_t)(BL.oGV + d) * ST] = ws[L.oJ + r * n + d];
  for (int sg = 1; sg <= 4; sg++)
    for (int l = 0; l < M.lanes; l++) fd_backward_stage<R, ST>(M, rb, ws + L.D.oS, 1, l, sg, nullptr, wi, wiB, nullptr, 0);
}

// Cholesky of A = J Y^T + rho I in place (lower triangle, row-major [m][m]); false when a pivot is at or below the threshold
template <class R> NB2_HD bool cfd_cholesky(R* A, int m) {
  R dmax = R(0);
  for (int i = 0; i < m; i++) dmax = A[i * m + i] > dmax ? A[i * m + i] : dmax;
  const R tol = R(NB2_CFD_PIVOT_C) * (sizeof(R) == 8 ? R(2.220446049250313e-16) : R(1.1920929e-07)) * dmax;
  for (int j = 0; j < m; j++) {
    R d = A[j * m + j];
    for (int c = 0; c < j; c++) d -= A[j * m + c] * A[j * m + c];
    if (!(d > tol)) return false;
    const R ljj = nb2_sqrt(d);
    A[j * m + j] = ljj;
    for (int i = j + 1; i < m; i++) {
      R s = A[i * m + j];
      for (int c = 0; c < j; c++) s -= A[i * m + c] * A[j * m + c];
      A[i * m + j] = s / ljj;
    }
  }
  return true;
}
// x <- (L L^T)^-1 x
template <class R> NB2_HD void cfd_solve(const R* A, int m, R* x) {
  for (int i = 0; i < m; i++) {
    R s = x[i];
    for (int c = 0; c < i; c++) s -= A[i * m + c] * x[c];
    x[i] = s / A[i * m + i];
  }
  for (int i = m - 1; i >= 0; i--) {
    R s = x[i];
    for (int c = i + 1; c < m; c++) s -= A[c * m + i] * x[c];
    x[i] = s / A[i * m + i];
  }
}

// the forward stages 1 .. NB2_FWD_STAGES - 2 of FD on the lanes of the model's schedule, after dj_load (qdd in the action words, the saved
// stream written)
template <class R, class Stage> NB2_HD void cfd_fd_forward(const Nb2ModelDev<R>& M, R* ws, const double* wi, size_t wiB, Stage&& stage) {
  for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++) stage([&](int lane, int) { dj_forward_stage<R, true>(M, ws, lane, sg, wi, wiB); });
}

// contact i's wrench seed gw (its 6 or 3 entries) in point form: lambar lb and the point adjoint pb.  lb may be gw (every entry is read
// before any is written).
template <class R> NB2_HD void cfd_point_form(const CfdNodes<R>& N, const CfdLayout& L, const R* ws, int i, const R* gw, R* lb, R* pb) {
  if (N.point) {
    for (int j = 0; j < 3; j++) { lb[j] = gw[j]; pb[j] = R(0); }
    return;
  }
  const V3<R> ga = mk3<R>(gw[0], gw[1], gw[2]), p = mk3<R>(ws[L.oP + 3 * i], ws[L.oP + 3 * i + 1], ws[L.oP + 3 * i + 2]);
  const R* lam = ws + L.oC + 6 * i;
  const V3<R> gl = mk3<R>(gw[3], gw[4], gw[5]) + cross(ga, p), pbar = cross(mk3<R>(lam[3], lam[4], lam[5]), ga);
  lb[0] = ga.x; lb[1] = ga.y; lb[2] = ga.z; lb[3] = gl.x; lb[4] = gl.y; lb[5] = gl.z;
  pb[0] = pbar.x; pb[1] = pbar.y; pb[2] = pbar.z;
}

// one seed's point-Jacobian VJPs, added to its [dL/dq ; dL/dqdot] G: J with lam u^T - mu qdd^T, then Jdot with -mu qdot^T and the points'
// own adjoints pb, and -Jdot^T mu.  The offset gradients land in the go words.  The walks are seed-free, but jpdb_terms overwrites its
// walk's screws and velocities in place, so each seed walks again.
template <class R, class Stage>
NB2_HD void cfd_point_vjps(const Nb2ModelDev<R>& M, const CfdNodes<R>& N, const CfdRows<R>& io, const CfdLayout& L, R* ws, const R* mu,
                           const R* u, const R* pb, R* G, Stage&& stage) {
  const int n = M.ndof, k = N.k, rpc = N.point ? 3 : 6, r0c = N.point ? 3 : 0, m = k * rpc;
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const R* s = io.state;
  const R* qd = s + n;
  R* K = ws + L.oK;
  R* gb = ws + L.oGb;
  for (int deriv = 0; deriv < 2; deriv++) {
    if (deriv) stage([&](int lane, int nl) { jpdb_init<R>(M, K, lane, nl); });
    else stage([&](int lane, int nl) { jpb_init<R>(M, K, lane, nl); });
    for (int i = 0; i < k; i++) {
      const int b = N.body[i];
      const R* o = io.off ? io.off + 3 * i : nullptr;
      R* go = ws + L.oGo + 12 * deriv + 3 * i;
      stage([&](int lane, int nl) {
        for (int idx = lane; idx < 6 * n; idx += nl) {
          const int row = idx / n, d = idx - row * n, j = row - r0c;
          R g = R(0);
          if (j >= 0) {
            const int r = i * rpc + j;
            g = deriv ? -mu[r] * qd[d] : ws[L.oC + r] * u[d] - mu[r] * ws[F.oAct + d];
          }
          gb[idx] = g;
        }
      });
      if (deriv) {
        stage([&](int lane, int) { jpdb_walk<R>(M, s, qd, b, N.T[i], o, K, lane); });
        stage([&](int lane, int nl) { jpdb_terms<R>(M, b, gb, K, lane, nl); });
        stage([&](int lane, int) {
          if (lane == 0) for (int c = 0; c < 3; c++) K[jpdb_layout(M.nb, n).oPP + 3 + c] += pb[3 * i + c];
        });
        stage([&](int lane, int) { jpdb_reduce<R>(M, s, qd, b, K, go, lane); });
      } else {
        stage([&](int lane, int) { jpb_walk<R>(M, s, b, N.T[i], o, K, lane); });
        stage([&](int lane, int nl) { jpb_terms<R>(M, b, gb, K, lane, nl); });
        stage([&](int lane, int) { jpb_reduce<R>(M, s, b, K, go, lane); });
      }
    }
    stage([&](int lane, int nl) {
      for (int d = lane; d < n; d += nl) {
        if (deriv) {
          R v = K[jpdb_layout(M.nb, n).oGq + n + d];
          for (int r = 0; r < m; r++) v -= ws[L.oJd + r * n + d] * mu[r];
          G[d] += K[jpdb_layout(M.nb, n).oGq + d];
          G[n + d] += v;
        } else {
          G[d] += K[jpb_layout(M.nb, n).oGq + d];
        }
      }
    });
  }
}

// The program of one world.  BWD: the backward recomputes the forward (nothing is kept between the calls) and continues.
template <class R, int ST, bool BWD, class Stage>
NB2_HD void cfd_world(const Nb2ModelDev<R>& M, const CfdNodes<R>& N, const CfdRows<R>& io, R* ws, Stage&& stage) {
  const int n = M.ndof, k = N.k, rpc = N.point ? 3 : 6, r0c = N.point ? 3 : 0, m = k * rpc;
  const CfdLayout L = cfd_layout(M, m, ST);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const R* s = io.state;
  const R* qd = s + n;
  // ---- free accelerations, J, Jdot and the points
  stage([&](int lane, int nl) { dj_load<R>(M, ws, s, io.tau, lane, nl); });
  cfd_fd_forward<R>(M, ws, io.wi, io.wiB, stage);
  for (int i = 0; i < k; i++) {
    const int b = N.body[i];
    const R* o = io.off ? io.off + 3 * i : nullptr;
    R* K = ws + L.oK;
    for (int deriv = 0; deriv < 2; deriv++) {
      stage([&](int lane, int nl) { jp_zero<R>(M, K, lane, nl); });
      if (deriv) stage([&](int lane, int) { jpd_walk<R>(M, s, qd, b, N.T[i], o, K, lane); });
      else stage([&](int lane, int) { jp_walk<R>(M, s, b, N.T[i], o, K, lane); });
      if (deriv) stage([&](int lane, int nl) { jpd_columns<R>(M, b, K, lane, nl); });
      else stage([&](int lane, int nl) { jp_columns<R>(M, b, K, lane, nl); });
      stage([&](int lane, int nl) {
        R* dst = ws + (deriv ? L.oJd : L.oJ) + i * rpc * n;
        for (int idx = lane; idx < rpc * n; idx += nl) dst[idx] = K[r0c * n + idx];
        if (!deriv && lane == 0) for (int c = 0; c < 3; c++) ws[L.oP + 3 * i + c] = K[jp_layout(n).oP + c];
      });
    }
  }
  // c = J qdd_free + Jdot qdot; the columns of M^-1 J^T in rounds of ST row slots
  stage([&](int lane, int nl) {
    for (int r = lane; r < m; r += nl) {
      R c = R(0);
      for (int d = 0; d < n; d++) c += ws[L.oJ + r * n + d] * ws[F.oAct + d] + ws[L.oJd + r * n + d] * qd[d];
      ws[L.oC + r] = c;
    }
  });
  for (int q0 = 0; q0 < m; q0 += ST) {
    const int nrows = (m - q0 < ST) ? m - q0 : ST;
    stage([&](int lane, int) { if (lane < nrows) cfd_column<R, ST>(M, L, ws, s, q0 + lane, lane, io.wi, io.wiB); });
    stage([&](int lane, int nl) {
      const int lam = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree).oLam;
      for (int idx = lane; idx < nrows * n; idx += nl) {
        const int d = idx / nrows, t = idx - d * nrows;
        ws[L.oY + (q0 + t) * n + d] = ws[L.D.oB + t + (size_t)(lam + d) * ST];
      }
    });
  }
  // A = J M^-1 J^T + rho I (lower triangle), its factor, lam
  stage([&](int lane, int nl) {
    for (int idx = lane; idx < m * m; idx += nl) {
      const int r = idx / m, c = idx - r * m;
      if (c > r) continue;
      R a = r == c ? io.rho : R(0);
      for (int d = 0; d < n; d++) a += ws[L.oJ + r * n + d] * ws[L.oY + c * n + d];
      ws[L.oA + idx] = a;
    }
  });
  stage([&](int lane, int) {
    if (lane != 0) return;
    const bool ok = cfd_cholesky<R>(ws + L.oA, m);
    ws[L.oFlag] = ok ? R(0) : R(1);
    if (!ok) return;
    for (int r = 0; r < m; r++) ws[L.oC + r] = -ws[L.oC + r];
    cfd_solve<R>(ws + L.oA, m, ws + L.oC);
  });
  // qdd = FD(tau + J^T lam), which also writes the saved stream the backward sweeps read
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R t = io.tau[d];
      for (int r = 0; r < m; r++) t += ws[L.oJ + r * n + d] * ws[L.oC + r];
      ws[L.oTau + d] = t;
    }
  });
  stage([&](int lane, int nl) { dj_load<R>(M, ws, s, ws + L.oTau, lane, nl); });
  cfd_fd_forward<R>(M, ws, io.wi, io.wiB, stage);
  if (!BWD) {
    stage([&](int lane, int nl) {
      const bool bad = ws[L.oFlag] != R(0);
      for (int d = lane; d < n; d += nl) io.qdd[d] = bad ? cfd_nan<R>() : ws[F.oAct + d];
      for (int idx = lane; idx < m; idx += nl) {
        const int i = idx / rpc, j = idx - i * rpc;
        const R* lam = ws + L.oC + i * rpc;
        R v = lam[j];
        if (!N.point && j < 3) {
          const V3<R> t = cross(mk3<R>(ws[L.oP + 3 * i], ws[L.oP + 3 * i + 1], ws[L.oP + 3 * i + 2]), mk3<R>(lam[3], lam[4], lam[5]));
          v += j == 0 ? t.x : j == 1 ? t.y : t.z;
        }
        io.wrench[idx] = bad ? cfd_nan<R>() : v;
      }
    });
    return;
  }
  // ---- backward: the seeds in point form, mu, g = qddbar - J^T mu
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) ws[L.oQb + d] = io.gqdd[d];
    for (int i = lane; i < k; i += nl) {
      const R* gw = io.gw + i * rpc;
      R* lb = ws + L.oLb + i * rpc;
      R* pb = ws + L.oPb + 3 * i;
      if (N.point) {
        for (int j = 0; j < 3; j++) { lb[j] = gw[j]; pb[j] = R(0); }
        continue;
      }
      const V3<R> ga = mk3<R>(gw[0], gw[1], gw[2]), p = mk3<R>(ws[L.oP + 3 * i], ws[L.oP + 3 * i + 1], ws[L.oP + 3 * i + 2]);
      const R* lam = ws + L.oC + 6 * i;
      const V3<R> gl = mk3<R>(gw[3], gw[4], gw[5]) + cross(ga, p), pbar = cross(mk3<R>(lam[3], lam[4], lam[5]), ga);
      lb[0] = ga.x; lb[1] = ga.y; lb[2] = ga.z; lb[3] = gl.x; lb[4] = gl.y; lb[5] = gl.z;
      pb[0] = pbar.x; pb[1] = pbar.y; pb[2] = pbar.z;
    }
  });
  stage([&](int lane, int nl) {
    for (int r = lane; r < m; r += nl) {
      R v = ws[L.oLb + r];
      for (int d = 0; d < n; d++) v += ws[L.oY + r * n + d] * ws[L.oQb + d];
      ws[L.oMu + r] = v;
    }
  });
  stage([&](int lane, int) { if (lane == 0 && ws[L.oFlag] == R(0)) cfd_solve<R>(ws + L.oA, m, ws + L.oMu); });
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  R* rb = ws + L.D.oB;  // row slot 0
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R g = ws[L.oQb + d];
      for (int r = 0; r < m; r++) g -= ws[L.oJ + r * n + d] * ws[L.oMu + r];
      rb[(size_t)(BL.oGV + d) * ST] = g;
      rb[(size_t)(BL.oSt + d) * ST] = s[d];
      rb[(size_t)(BL.oSt + n + d) * ST] = s[n + d];
    }
  });
  // the FD backward at tau + J^T lam, seeded with g, on the lanes of the schedule
  for (int sg = 1; sg < NB2_BWD_STAGES - 1; sg++)
    stage([&](int lane, int) {
      if (lane < M.lanes) fd_backward_stage<R, ST>(M, rb, ws + L.D.oS, 1, lane, sg, nullptr, io.wi, io.wiB, io.gI, io.wiB);
    });
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      ws[L.oG + d] = rb[(size_t)(BL.oQb + d) * ST];
      ws[L.oG + n + d] = rb[(size_t)(BL.oVb + d) * ST];
      ws[L.oU + d] = rb[(size_t)(BL.oLam + d) * ST];
    }
  });
  // the point-Jacobian VJPs: J with lam u^T - mu qdd^T, then Jdot with -mu qdot^T and the points' own adjoints
  R* K = ws + L.oK;
  R* gb = ws + L.oGb;
  for (int deriv = 0; deriv < 2; deriv++) {
    if (deriv) stage([&](int lane, int nl) { jpdb_init<R>(M, K, lane, nl); });
    else stage([&](int lane, int nl) { jpb_init<R>(M, K, lane, nl); });
    for (int i = 0; i < k; i++) {
      const int b = N.body[i];
      const R* o = io.off ? io.off + 3 * i : nullptr;
      R* go = ws + L.oGo + 12 * deriv + 3 * i;
      stage([&](int lane, int nl) {
        for (int idx = lane; idx < 6 * n; idx += nl) {
          const int row = idx / n, d = idx - row * n, j = row - r0c;
          R g = R(0);
          if (j >= 0) {
            const int r = i * rpc + j;
            g = deriv ? -ws[L.oMu + r] * qd[d] : ws[L.oC + r] * ws[L.oU + d] - ws[L.oMu + r] * ws[F.oAct + d];
          }
          gb[idx] = g;
        }
      });
      if (deriv) {
        stage([&](int lane, int) { jpdb_walk<R>(M, s, qd, b, N.T[i], o, K, lane); });
        stage([&](int lane, int nl) { jpdb_terms<R>(M, b, gb, K, lane, nl); });
        stage([&](int lane, int) {
          if (lane == 0) for (int c = 0; c < 3; c++) K[jpdb_layout(M.nb, n).oPP + 3 + c] += ws[L.oPb + 3 * i + c];
        });
        stage([&](int lane, int) { jpdb_reduce<R>(M, s, qd, b, K, go, lane); });
      } else {
        stage([&](int lane, int) { jpb_walk<R>(M, s, b, N.T[i], o, K, lane); });
        stage([&](int lane, int nl) { jpb_terms<R>(M, b, gb, K, lane, nl); });
        stage([&](int lane, int) { jpb_reduce<R>(M, s, b, K, go, lane); });
      }
    }
    stage([&](int lane, int nl) {
      for (int d = lane; d < n; d += nl) {
        if (deriv) {
          R v = K[jpdb_layout(M.nb, n).oGq + n + d];
          for (int r = 0; r < m; r++) v -= ws[L.oJd + r * n + d] * ws[L.oMu + r];
          ws[L.oG + d] += K[jpdb_layout(M.nb, n).oGq + d];
          ws[L.oG + n + d] += v;
        } else {
          ws[L.oG + d] += K[jpb_layout(M.nb, n).oGq + d];
        }
      }
    });
  }
  stage([&](int lane, int nl) {
    const bool bad = ws[L.oFlag] != R(0);
    for (int d = lane; d < 2 * n; d += nl) io.gstate[d] = bad ? cfd_nan<R>() : ws[L.oG + d];
    for (int d = lane; d < n; d += nl) io.gtau[d] = bad ? cfd_nan<R>() : ws[L.oU + d];
    if (io.goff)
      for (int idx = lane; idx < 3 * k; idx += nl) io.goff[idx] = bad ? cfd_nan<R>() : ws[L.oGo + idx] + ws[L.oGo + 12 + idx];
    if (io.gI && bad)
      for (int idx = lane; idx < 10 * M.nb; idx += nl) io.gI[(size_t)idx * io.wiB] = (double)cfd_nan<R>();
  });
}

// ---- dense Jacobians (DESIGN.md §6p).  Row i of each block is the VJP above with the seed e_i on one output: n seeds on qdd, then m on
// the wrenches.  The forward is cfd_world's own, run once; the seed-free words it leaves (J, Jdot, Y, the factor, lam, qdd, the saved
// stream) serve every row.  Rounds of ST seeds: seed t's backward words sit in the extension below, its FD backward runs in row slot t,
// swept by thread t over every lane of the schedule (as k_dj's rows), and the point-Jacobian VJPs take the seeds one after the other on
// the warp.  The world's blocks: dqdd/dq, dqdd/dqdot, dqdd/dtau [n][n] and dwrench/dq, dwrench/dqdot, dwrench/dtau [m][n], row-major.
template <class R> struct CfdJacRows { R* Jq; R* Jqd; R* Jt; R* Wq; R* Wqd; R* Wt; };
// the working set: cfd_layout's, then per seed slot t mu [m], lambar [m], pbar [12], qddbar [n], [dL/dq ; dL/dqdot] [2n], u [n]
struct CfdjLayout { CfdLayout C; int oMu, oLb, oPb, oQb, oG, oU, total; };
NB2_HD CfdjLayout cfdj_layout(int nb, int n, int nslots, int nfree, int m, int st) {
  CfdjLayout L;
  L.C = cfd_layout(nb, n, nslots, nfree, m, st);
  L.oMu = L.C.total; L.oLb = L.oMu + st * m; L.oPb = L.oLb + st * m; L.oQb = L.oPb + 12 * st; L.oG = L.oQb + st * n; L.oU = L.oG + 2 * n * st;
  L.total = L.oU + n * st;
  return L;
}

template <class R, int ST, class Stage>
NB2_HD void cfdj_world(const Nb2ModelDev<R>& M, const CfdNodes<R>& N, const CfdRows<R>& io, const CfdJacRows<R>& out, R* ws, Stage&& stage) {
  const int n = M.ndof, k = N.k, rpc = N.point ? 3 : 6, m = k * rpc, rows = n + m;
  const CfdjLayout X = cfdj_layout(M.nb, M.ndof, M.nslots, M.nfree, m, ST);
  const CfdLayout& L = X.C;
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const R* s = io.state;
  cfd_world<R, ST, false>(M, N, io, ws, stage);  // qdd and the wrenches written
  for (int s0 = 0; s0 < rows; s0 += ST) {
    const int ns = (rows - s0 < ST) ? rows - s0 : ST;
    // the seeds: e_row on qdd (row < n) or on the wrench entry row - n; then in point form, in place
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * rows; idx += nl) {
        const int t = idx / rows, e = idx - t * rows;
        if (e < n) ws[X.oQb + t * n + e] = (s0 + t == e) ? R(1) : R(0);
        else ws[X.oLb + t * m + e - n] = (s0 + t == e) ? R(1) : R(0);
      }
    });
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * k; idx += nl) {
        const int t = idx / k, i = idx - t * k;
        R* lb = ws + X.oLb + t * m + i * rpc;
        cfd_point_form<R>(N, L, ws, i, lb, lb, ws + X.oPb + 12 * t + 3 * i);
      }
    });
    // mu = (J M^-1 J^T + rho I)^-1 (lambar + Y qddbar), slot t on lane t
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * m; idx += nl) {
        const int t = idx / m, r = idx - t * m;
        R v = ws[X.oLb + t * m + r];
        for (int d = 0; d < n; d++) v += ws[L.oY + r * n + d] * ws[X.oQb + t * n + d];
        ws[X.oMu + t * m + r] = v;
      }
    });
    stage([&](int lane, int) { if (lane < ns && ws[L.oFlag] == R(0)) cfd_solve<R>(ws + L.oA, m, ws + X.oMu + lane * m); });
    // g = qddbar - J^T mu, the FD backward seeded with g (slot t on thread t), then its rows
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * n; idx += nl) {
        const int t = idx / n, d = idx - t * n;
        R* rb = ws + L.D.oB + t;
        R g = ws[X.oQb + t * n + d];
        for (int r = 0; r < m; r++) g -= ws[L.oJ + r * n + d] * ws[X.oMu + t * m + r];
        rb[(size_t)(BL.oGV + d) * ST] = g;
        rb[(size_t)(BL.oSt + d) * ST] = s[d];
        rb[(size_t)(BL.oSt + n + d) * ST] = s[n + d];
      }
    });
    stage([&](int lane, int) {
      if (lane >= ns) return;
      R* rb = ws + L.D.oB + lane;
      for (int sg = 1; sg < NB2_BWD_STAGES - 1; sg++)
        for (int l = 0; l < M.lanes; l++) fd_backward_stage<R, ST>(M, rb, ws + L.D.oS, 1, l, sg, nullptr, io.wi, io.wiB, nullptr, 0);
    });
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * n; idx += nl) {
        const int t = idx / n, d = idx - t * n;
        const R* rb = ws + L.D.oB + t;
        ws[X.oG + 2 * n * t + d] = rb[(size_t)(BL.oQb + d) * ST];
        ws[X.oG + 2 * n * t + n + d] = rb[(size_t)(BL.oVb + d) * ST];
        ws[X.oU + n * t + d] = rb[(size_t)(BL.oLam + d) * ST];
      }
    });
    for (int t = 0; t < ns; t++)
      cfd_point_vjps<R>(M, N, io, L, ws, ws + X.oMu + t * m, ws + X.oU + t * n, ws + X.oPb + 12 * t, ws + X.oG + 2 * n * t, stage);
    // the round's rows, in address order within each block
    stage([&](int lane, int nl) {
      const bool bad = ws[L.oFlag] != R(0);
      for (int idx = lane; idx < ns * n; idx += nl) {
        const int t = idx / n, j = idx - t * n, row = s0 + t;
        const bool acc = row < n;
        const size_t e = (size_t)(acc ? row : row - n) * n + j;
        const R gq = ws[X.oG + 2 * n * t + j], gv = ws[X.oG + 2 * n * t + n + j], gt = ws[X.oU + n * t + j];
        (acc ? out.Jq : out.Wq)[e] = bad ? cfd_nan<R>() : gq;
        (acc ? out.Jqd : out.Wqd)[e] = bad ? cfd_nan<R>() : gv;
        (acc ? out.Jt : out.Wt)[e] = bad ? cfd_nan<R>() : gt;
      }
    });
  }
}

}  // namespace nb2
