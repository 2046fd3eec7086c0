// Impulse dynamics with bilateral contacts, batched (DESIGN.md §6q): the impact map at a touchdown.  k contacts (1 <= k <=
// NB2_MAX_CONTACT_BODIES) hold the rows of their points' world Jacobians J [m, n], as in constrained forward dynamics (nb2_cfd.cuh), and an
// instantaneous impulse Lam makes the post-impact velocity satisfy them with restitution e and damping rho:
//   M (qdot+ - qdot-) = J^T Lam ,   J qdot+ = -e J qdot- - rho Lam
//   =>  Lam = -(J M^-1 J^T + rho I)^-1 (1 + e) J qdot- ,   qdot+ = qdot- + M^-1 J^T Lam .
// Gravity, joint springs and damping, tau and limits play no part.  M^-1 f is one FD pass at [q ; 0] on the passive-free model (imp_model):
// at qdot = 0 the Coriolis term and its qdot-gradient vanish, so FD, its q-gradient and its inertia gradient are those of M(q)^-1 f.
//
// ONE WARP PER WORLD, one world per block, the stages and working set of cfd_world (cfd_layout; its Jdot block stays unused).  The row
// [q ; 0] sits in the seed block of the point-Jacobian VJPs, which the program needs only after its last FD pass.
//
// Backward (L(qdot+, w)), with the seeds vbar on qdot+ and lambar, pbar (cfd_point_form) from the impulses:
//   mu = (J M^-1 J^T + rho I)^-1 (lambar + Y vbar),   g = vbar - J^T mu,   u = M^-1 g ,
//   dL/dqdot- = vbar - (1 + e) J^T mu ,
//   dL/dq = <g, d(M^-1 J^T Lam)/dq>|_J (the FD backward seeded with g on the saved stream of FD([q ; 0], J^T Lam), which also gives u and
//           the inertia gradient) + the point-Jacobian VJP with the rank-one seed Lam u^T - mu (qdot+ + e qdot-)^T and the points' own
//           adjoints pbar (jpb_reduce<R, true>); dL/do_i from the same VJP.
#pragma once
#include "nb2_cfd.cuh"

namespace nb2 {

// the passive-free copy of an FD model: no gravity, springs or joint damping (the model's inertias, joints and schedule unchanged)
template <class R> NB2_HD Nb2ModelDev<R> imp_model(const Nb2ModelDev<R>& M) {
  Nb2ModelDev<R> P = M;
  for (int c = 0; c < 3; c++) P.gravity[c] = R(0);
  for (int d = 0; d < NB2_MAX_DOFS; d++) P.spring[d] = P.damping[d] = R(0);
  return P;
}

// one world's rows.  Forward: state [2n] (q, qdot-), offsets ([k][3], or NULL), vel [n] = qdot+, imp [k][6 or 3].  Backward adds the
// seeds gvel [n] and gimp [k][6 or 3] and writes gstate [2n], goff [k][3] (or NULL) and gI (word-major [10 nb][wiB], or NULL).
template <class R> struct ImpRows {
  const R* state; const R* off; R* vel; R* imp;
  const R* gvel; const R* gimp; R* gstate; R* goff; double* gI;
  const double* wi; size_t wiB;
  R rho, e;
};

// The program of one world; M is the passive-free model (imp_model).  BWD: the backward recomputes the forward and continues.
template <class R, int ST, bool BWD, class Stage>
NB2_HD void imp_world(const Nb2ModelDev<R>& M, const CfdNodes<R>& N, const ImpRows<R>& io, R* ws, Stage&& stage) {
  const int n = M.ndof, k = N.k, rpc = N.point ? 3 : 6, r0c = N.point ? 3 : 0, m = k * rpc;
  const CfdLayout L = cfd_layout(M, m, ST);
  const R* s = io.state;
  const R* qd = s + n;
  const R ep1 = R(1) + io.e;
  R* row = ws + L.oGb;  // [q ; 0]
  R* K = ws + L.oK;
  // ---- the saved stream of FD at [q ; 0] (tau = 0: the row's zero half), which the column sweeps read
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) { row[d] = s[d]; row[n + d] = R(0); }
  });
  stage([&](int lane, int nl) { dj_load<R>(M, ws, row, row + n, lane, nl); });
  cfd_fd_forward<R>(M, ws, io.wi, io.wiB, stage);
  // J and the points
  for (int i = 0; i < k; i++) {
    const int b = N.body[i];
    const R* o = io.off ? io.off + 3 * i : nullptr;
    stage([&](int lane, int nl) { jp_zero<R>(M, K, lane, nl); });
    stage([&](int lane, int) { jp_walk<R>(M, s, b, N.T[i], o, K, lane); });
    stage([&](int lane, int nl) { jp_columns<R>(M, b, K, lane, nl); });
    stage([&](int lane, int nl) {
      R* dst = ws + L.oJ + i * rpc * n;
      for (int idx = lane; idx < rpc * n; idx += nl) dst[idx] = K[r0c * n + idx];
      if (lane == 0) for (int c = 0; c < 3; c++) ws[L.oP + 3 * i + c] = K[jp_layout(n).oP + c];
    });
  }
  // c = (1 + e) J qdot-; the columns of M^-1 J^T in rounds of ST row slots
  stage([&](int lane, int nl) {
    for (int r = lane; r < m; r += nl) {
      R c = R(0);
      for (int d = 0; d < n; d++) c += ws[L.oJ + r * n + d] * qd[d];
      ws[L.oC + r] = ep1 * c;
    }
  });
  for (int q0 = 0; q0 < m; q0 += ST) {
    const int nrows = (m - q0 < ST) ? m - q0 : ST;
    stage([&](int lane, int) { if (lane < nrows) cfd_column<R, ST>(M, L, ws, row, q0 + lane, lane, io.wi, io.wiB); });
    stage([&](int lane, int nl) {
      const int lam = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree).oLam;
      for (int idx = lane; idx < nrows * n; idx += nl) {
        const int d = idx / nrows, t = idx - d * nrows;
        ws[L.oY + (q0 + t) * n + d] = ws[L.D.oB + t + (size_t)(lam + d) * ST];
      }
    });
  }
  // A = J M^-1 J^T + rho I (lower triangle), its factor, Lam = -A^-1 c
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
  if (!BWD) {
    // qdot+ = qdot- + sum_r Lam_r Y_r; the impulses (about the world origin for a 6-D contact)
    stage([&](int lane, int nl) {
      const bool bad = ws[L.oFlag] != R(0);
      for (int d = lane; d < n; d += nl) {
        R v = qd[d];
        for (int r = 0; r < m; r++) v += ws[L.oY + r * n + d] * ws[L.oC + r];
        io.vel[d] = bad ? cfd_nan<R>() : v;
      }
      for (int idx = lane; idx < m; idx += nl) {
        const int i = idx / rpc, j = idx - i * rpc;
        const R* lam = ws + L.oC + i * rpc;
        R v = lam[j];
        if (!N.point && j < 3) {
          const V3<R> t = cross(mk3<R>(ws[L.oP + 3 * i], ws[L.oP + 3 * i + 1], ws[L.oP + 3 * i + 2]), mk3<R>(lam[3], lam[4], lam[5]));
          v += j == 0 ? t.x : j == 1 ? t.y : t.z;
        }
        io.imp[idx] = bad ? cfd_nan<R>() : v;
      }
    });
    return;
  }
  // ---- backward: the seeds in point form, mu
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) ws[L.oQb + d] = io.gvel[d];
    for (int i = lane; i < k; i += nl) cfd_point_form<R>(N, L, ws, i, io.gimp + i * rpc, ws + L.oLb + i * rpc, ws + L.oPb + 3 * i);
  });
  stage([&](int lane, int nl) {
    for (int r = lane; r < m; r += nl) {
      R v = ws[L.oLb + r];
      for (int d = 0; d < n; d++) v += ws[L.oY + r * n + d] * ws[L.oQb + d];
      ws[L.oMu + r] = v;
    }
  });
  stage([&](int lane, int) { if (lane == 0 && ws[L.oFlag] == R(0)) cfd_solve<R>(ws + L.oA, m, ws + L.oMu); });
  // the saved stream of FD([q ; 0], J^T Lam)
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R t = R(0);
      for (int r = 0; r < m; r++) t += ws[L.oJ + r * n + d] * ws[L.oC + r];
      ws[L.oTau + d] = t;
    }
  });
  stage([&](int lane, int nl) { dj_load<R>(M, ws, row, ws + L.oTau, lane, nl); });
  cfd_fd_forward<R>(M, ws, io.wi, io.wiB, stage);
  // g = vbar - J^T mu into row slot 0, then the FD backward seeded with g on the lanes of the schedule
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  R* rb = ws + L.D.oB;
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R jm = R(0);
      for (int r = 0; r < m; r++) jm += ws[L.oJ + r * n + d] * ws[L.oMu + r];
      rb[(size_t)(BL.oGV + d) * ST] = ws[L.oQb + d] - jm;
      rb[(size_t)(BL.oSt + d) * ST] = row[d];
      rb[(size_t)(BL.oSt + n + d) * ST] = row[n + d];
      ws[L.oG + n + d] = ws[L.oQb + d] - ep1 * jm;  // dL/dqdot-
    }
  });
  for (int sg = 1; sg < NB2_BWD_STAGES - 1; sg++)
    stage([&](int lane, int) {
      if (lane < M.lanes) fd_backward_stage<R, ST>(M, rb, ws + L.D.oS, 1, lane, sg, nullptr, io.wi, io.wiB, io.gI, io.wiB);
    });
  // its dL/dq share and u; qdot+ + e qdot- (in the tau words, free again)
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      ws[L.oG + d] = rb[(size_t)(BL.oQb + d) * ST];
      ws[L.oU + d] = rb[(size_t)(BL.oLam + d) * ST];
      R v = qd[d];
      for (int r = 0; r < m; r++) v += ws[L.oY + r * n + d] * ws[L.oC + r];
      ws[L.oTau + d] = v + io.e * qd[d];
    }
  });
  // the point-Jacobian VJP, contact by contact: J with Lam u^T - mu (qdot+ + e qdot-)^T, the points with pbar (the seed block overwrites
  // the row [q ; 0], which is no longer read)
  R* gb = ws + L.oGb;
  stage([&](int lane, int nl) { jpb_init<R>(M, K, lane, nl); });
  for (int i = 0; i < k; i++) {
    const int b = N.body[i];
    const R* o = io.off ? io.off + 3 * i : nullptr;
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < 6 * n; idx += nl) {
        const int rw = idx / n, d = idx - rw * n, j = rw - r0c;
        R g = R(0);
        if (j >= 0) {
          const int r = i * rpc + j;
          g = ws[L.oC + r] * ws[L.oU + d] - ws[L.oMu + r] * ws[L.oTau + d];
        }
        gb[idx] = g;
      }
    });
    stage([&](int lane, int) { jpb_walk<R>(M, s, b, N.T[i], o, K, lane); });
    stage([&](int lane, int nl) { jpb_terms<R>(M, b, gb, K, lane, nl); });
    stage([&](int lane, int) { jpb_reduce<R, true>(M, s, b, K, ws + L.oGo + 3 * i, lane, ws + L.oPb + 3 * i); });
  }
  stage([&](int lane, int nl) {
    const bool bad = ws[L.oFlag] != R(0);
    for (int d = lane; d < n; d += nl) io.gstate[d] = bad ? cfd_nan<R>() : ws[L.oG + d] + K[jpb_layout(M.nb, n).oGq + d];
    for (int d = lane; d < n; d += nl) io.gstate[n + d] = bad ? cfd_nan<R>() : ws[L.oG + n + d];
    if (io.goff)
      for (int idx = lane; idx < 3 * k; idx += nl) io.goff[idx] = bad ? cfd_nan<R>() : ws[L.oGo + idx];
    if (io.gI && bad)
      for (int idx = lane; idx < 10 * M.nb; idx += nl) io.gI[(size_t)idx * io.wiB] = (double)cfd_nan<R>();
  });
}

// ---- dense Jacobians (DESIGN.md §6r).  Row i of each block is the backward above with the seed e_i on one output: n seeds on qdot+, then
// m on the impulses.  The forward is imp_world's own, run once; the seed-free words it leaves (J, the points, Y, the factor, Lam in the c
// words) serve every row, and so do the saved stream of FD([q ; 0], J^T Lam) and qdot+ + e qdot-, built once after it.  Rounds of ST seeds
// in cfdj_layout's per-slot words: mu, lambar, pbar, the seed vbar (its qddbar words), [dL/dq ; dL/dqdot-] and u.  Seed t's FD backward
// runs in row slot t, swept by thread t over every lane of the schedule; the dL/dqdot- row needs no sweep; the point-Jacobian VJPs take
// the seeds one after the other on the warp.  The world's blocks: dqdot+/dq, dqdot+/dqdot- [n][n] and dimp/dq, dimp/dqdot- [m][n],
// row-major.
template <class R> struct ImpJacRows { R* Vq; R* Vqd; R* Iq; R* Iqd; };

template <class R, int ST, class Stage>
NB2_HD void impj_world(const Nb2ModelDev<R>& M, const CfdNodes<R>& N, const ImpRows<R>& io, const ImpJacRows<R>& out, R* ws, Stage&& stage) {
  const int n = M.ndof, k = N.k, rpc = N.point ? 3 : 6, r0c = N.point ? 3 : 0, m = k * rpc, rows = n + m;
  const CfdjLayout X = cfdj_layout(M.nb, M.ndof, M.nslots, M.nfree, m, ST);
  const CfdLayout& L = X.C;
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const R* s = io.state;
  const R* qd = s + n;
  const R ep1 = R(1) + io.e;
  R* K = ws + L.oK;
  R* gb = ws + L.oGb;  // the row [q ; 0] until the first seed's point-Jacobian VJP
  imp_world<R, ST, false>(M, N, io, ws, stage);  // qdot+ and the impulses written
  // ---- seed-free: the saved stream of FD([q ; 0], J^T Lam) (read before the seed block overwrites the row), then qdot+ + e qdot- in the
  // tau words
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R t = R(0);
      for (int r = 0; r < m; r++) t += ws[L.oJ + r * n + d] * ws[L.oC + r];
      ws[L.oTau + d] = t;
    }
  });
  stage([&](int lane, int nl) { dj_load<R>(M, ws, gb, ws + L.oTau, lane, nl); });
  cfd_fd_forward<R>(M, ws, io.wi, io.wiB, stage);
  stage([&](int lane, int nl) {
    for (int d = lane; d < n; d += nl) {
      R v = qd[d];
      for (int r = 0; r < m; r++) v += ws[L.oY + r * n + d] * ws[L.oC + r];
      ws[L.oTau + d] = v + io.e * qd[d];
    }
  });
  for (int s0 = 0; s0 < rows; s0 += ST) {
    const int ns = (rows - s0 < ST) ? rows - s0 : ST;
    // the seeds: e_row on qdot+ (row < n) or on the impulse entry row - n; then in point form, in place
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
    // mu = (J M^-1 J^T + rho I)^-1 (lambar + Y vbar), slot t on lane t
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * m; idx += nl) {
        const int t = idx / m, r = idx - t * m;
        R v = ws[X.oLb + t * m + r];
        for (int d = 0; d < n; d++) v += ws[L.oY + r * n + d] * ws[X.oQb + t * n + d];
        ws[X.oMu + t * m + r] = v;
      }
    });
    stage([&](int lane, int) { if (lane < ns && ws[L.oFlag] == R(0)) cfd_solve<R>(ws + L.oA, m, ws + X.oMu + lane * m); });
    // g = vbar - J^T mu into row slot t at [q ; 0] (the state words from s and 0: the row may be overwritten), and the dL/dqdot- row
    stage([&](int lane, int nl) {
      for (int idx = lane; idx < ns * n; idx += nl) {
        const int t = idx / n, d = idx - t * n;
        R* rb = ws + L.D.oB + t;
        R jm = R(0);
        for (int r = 0; r < m; r++) jm += ws[L.oJ + r * n + d] * ws[X.oMu + t * m + r];
        const R vb = ws[X.oQb + t * n + d];
        rb[(size_t)(BL.oGV + d) * ST] = vb - jm;
        rb[(size_t)(BL.oSt + d) * ST] = s[d];
        rb[(size_t)(BL.oSt + n + d) * ST] = R(0);
        ws[X.oG + 2 * n * t + n + d] = vb - ep1 * jm;
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
        ws[X.oU + n * t + d] = rb[(size_t)(BL.oLam + d) * ST];
      }
    });
    // seed by seed, the point-Jacobian VJP: J with Lam u^T - mu (qdot+ + e qdot-)^T, the points with pbar
    for (int t = 0; t < ns; t++) {
      const R* mu = ws + X.oMu + t * m;
      const R* u = ws + X.oU + n * t;
      stage([&](int lane, int nl) { jpb_init<R>(M, K, lane, nl); });
      for (int i = 0; i < k; i++) {
        const int b = N.body[i];
        const R* o = io.off ? io.off + 3 * i : nullptr;
        stage([&](int lane, int nl) {
          for (int idx = lane; idx < 6 * n; idx += nl) {
            const int rw = idx / n, d = idx - rw * n, j = rw - r0c;
            R g = R(0);
            if (j >= 0) {
              const int r = i * rpc + j;
              g = ws[L.oC + r] * u[d] - mu[r] * ws[L.oTau + d];
            }
            gb[idx] = g;
          }
        });
        stage([&](int lane, int) { jpb_walk<R>(M, s, b, N.T[i], o, K, lane); });
        stage([&](int lane, int nl) { jpb_terms<R>(M, b, gb, K, lane, nl); });
        stage([&](int lane, int) { jpb_reduce<R, true>(M, s, b, K, ws + L.oGo + 3 * i, lane, ws + X.oPb + 12 * t + 3 * i); });
      }
      stage([&](int lane, int nl) {
        R* G = ws + X.oG + 2 * n * t;
        for (int d = lane; d < n; d += nl) G[d] = G[d] + K[jpb_layout(M.nb, n).oGq + d];
      });
    }
    // the round's rows, in address order within each block
    stage([&](int lane, int nl) {
      const bool bad = ws[L.oFlag] != R(0);
      for (int idx = lane; idx < ns * n; idx += nl) {
        const int t = idx / n, j = idx - t * n, row = s0 + t;
        const bool vel = row < n;
        const size_t e = (size_t)(vel ? row : row - n) * n + j;
        const R gq = ws[X.oG + 2 * n * t + j], gv = ws[X.oG + 2 * n * t + n + j];
        (vel ? out.Vq : out.Iq)[e] = bad ? cfd_nan<R>() : gq;
        (vel ? out.Vqd : out.Iqd)[e] = bad ? cfd_nan<R>() : gv;
      }
    });
  }
}

}  // namespace nb2
