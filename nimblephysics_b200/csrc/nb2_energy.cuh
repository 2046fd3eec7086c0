// Kinetic and potential energy and centroidal momentum of a skeleton, batched (DESIGN.md §6m), at the state [q ; qdot] in the step's
// velocity coordinates (free joints: body twist).  For the tree rooted at r, with V_i = [w_i ; v_i] the world spatial velocity of body i
// (about the world origin), G_i its spatial inertia {m, h, Ibar} and x_i = m_i p_i + R_i h_i its world first moment:
//   T = 1/2 sum_i V_i . G_i V_i                                     (= 1/2 qdot^T M qdot)
//   U = -g . sum_i x_i + 1/2 sum_d k_d (q_d - q0_d)^2               (gravity at each body's COM; the springs of the tree's dofs)
//   h = [A - c x P ; P]                                             (c = sum x_i / m_tot; [A ; P] = sum_i P_i, P_i = G_i V_i in world axes
//                                                                    about the origin: angular momentum about the COM, linear momentum)
// The stages reuse the COM-Jacobian ones of nb2_jac.cuh unchanged: jcdb_init (joint transforms), jc_moments (world poses, subtree first
// moments and masses), jcd_vel (world velocities, subtree linear momentum).  As there, every function is one stage of a kernel, run on
// lane `lane` of `nl` with the lanes exchanging data only between stages, so a host build can run a stage's lanes in any order.
//
// Backward (L = Tbar T + Ubar U + <hbar, h>).  With Pbar = [hbar_a ; hbar_l + c x hbar_a] (the adjoint of sum P_i, a twist) and
// xbar = (hbar_a x P) / m_tot - Ubar g (the adjoint of every x_i), body i contributes <G_i V_i, Tbar/2 V_i + Pbar> + <xbar, x_i>, so
//   dL/dV_i = Y_i = G_i (Tbar V_i + Pbar),   dL/dqdot_k = <s_k, sum of Y over the subtree of k's body>.
// A joint j moved by the world twist xi moves everything at or below it rigidly: dG = -(ad_xi^T G + G ad_xi), ds = ad_xi s,
// dx = w x x + m v.  So dL/dxi is the world wrench
//   Gam_j = sum_{i at/below j} ( -jd_wrench(V_i, Y_i) - jd_wrench(Pbar, P_i) + [x_i x xbar ; m_i xbar] + sum_{k of i} jd_wrench(s_k, qdot_k Ys_i) )
// (Ys_i: Y summed over the subtree of i), carried to the joint's coordinates as in the Jacobian backwards (jd_joint_grad).  The springs add
// Ubar k_d (q_d - q0_d).  The inertia gradient of body i, with u = Tbar/2 V_b + Pbar_b and V_b in its own frame (L is u . G V_b there):
//   dL/dm = u_l . v_l + p_i . xbar - (hbar_a x P) . c / m_tot,   dL/dh = v_l x u_a + u_l x w + R_i^T xbar,   dL/dIbar = sym(u_a w^T).
#pragma once
#include "nb2_jac.cuh"

namespace nb2 {

// Working set: the COM-derivative backward's W, HM, the total mass, V, Hd and gq [2n] (jcd_layout(nb, n, true)), then P [nb][6] (forward:
// P_i; backward: Y_i, then its subtree sums), X [nb][6] (forward: [nb] kinetic energies; backward: the body's wrench, then the subtree's
// Gam), S [8] (forward: the sums of P, T and the spring energy).
struct EmLayout { int oW, oHM, oMt, oV, oHd, oGq, oP, oX, oS, total; };
NB2_HD EmLayout em_layout(int nb, int n, bool bwd) {
  const JcdLayout C = jcd_layout(nb, n, true);
  EmLayout L;
  L.oW = C.oW; L.oHM = C.oHM; L.oMt = C.oMt; L.oV = C.oV; L.oHd = C.oHd; L.oGq = C.oGq;
  L.oP = L.oGq + 2 * n; L.oX = L.oP + 6 * nb; L.oS = L.oX + (bwd ? 6 * nb : nb);
  L.total = (L.oS + 8 + 3) & ~3;
  return L;
}

// forward stage 3 (after jcdb_init, jc_moments, jcd_vel), lanes over the tree's bodies: P_i and the body's kinetic energy
template <class R> NB2_HD void em_bodies(const Nb2ModelDev<R>& M, int root, const double* wi, size_t wiB, R* ws, int lane, int nl) {
  const EmLayout L = em_layout(M.nb, M.ndof, false);
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    const V6<R> Vb = AdInvT(W, ldv6(ws + L.oV + 6 * i)), Pb = mulG(m, h, Ib, Vb);
    put6(ws + L.oP + 6 * i, dAdInvT(W, Pb));
    ws[L.oX + i] = R(0.5) * dot(Vb, Pb);
  }
}
// forward stage 4, lanes over the sums (root -> leaf, in body order): c < 6 the component c of sum P_i, 6 the kinetic energy, 7 the springs
template <class R> NB2_HD void em_sums(const Nb2ModelDev<R>& M, const R* q, int root, R* ws, int lane, int nl) {
  const EmLayout L = em_layout(M.nb, M.ndof, false);
  for (int c = lane; c < 8; c += nl) {
    R s = R(0);
    for (int i = root; i < M.nb; i++) {
      if (jac_root(M, i) != root) continue;
      if (c < 6) s += ws[L.oP + 6 * i + c];
      else if (c == 6) s += ws[L.oX + i];
      else {
        const int o = M.dof_off[i];
        for (int k = 0; k < mm_nd(M.jtype[i]); k++) { const R e = q[o + k] - M.rest[o + k]; s += R(0.5) * M.spring[o + k] * e * e; }
      }
    }
    ws[L.oS + c] = s;
  }
}
// forward stage 5, lane 0: the world's kinetic and potential energy and momentum [6]
template <class R> NB2_HD void em_store(const Nb2ModelDev<R>& M, int root, const R* ws, R* kin, R* pot, R* mom, int lane) {
  if (lane != 0) return;
  const EmLayout L = em_layout(M.nb, M.ndof, false);
  const R* S = ws + L.oS;
  const R* hm = ws + L.oHM + 4 * root;
  const V3<R> x = mk3<R>(hm[0], hm[1], hm[2]), P = mk3<R>(S[3], S[4], S[5]);
  const V3<R> a = mk3<R>(S[0], S[1], S[2]) - cross(x, P) * (R(1) / ws[L.oMt]);
  *kin = S[6];
  *pot = S[7] - dot(mk3<R>(M.gravity[0], M.gravity[1], M.gravity[2]), x);
  mom[0] = a.x; mom[1] = a.y; mom[2] = a.z; mom[3] = P.x; mom[4] = P.y; mom[5] = P.z;
}

// the adjoints every body shares: Pbar, xbar and the total mass's (gh: hbar [6]); needs HM, the total mass and Hd (jcd_vel)
template <class R> struct EmSeed { V6<R> Pb; V3<R> xb; R mb; };
template <class R> NB2_HD EmSeed<R> em_seed(const Nb2ModelDev<R>& M, int root, const R* ws, R gU, const R* gh) {
  const EmLayout L = em_layout(M.nb, M.ndof, true);
  const R inv = R(1) / ws[L.oMt];
  const R* hm = ws + L.oHM + 4 * root;
  const R* hd = ws + L.oHd + 4 * root;
  const V3<R> c = mk3<R>(hm[0], hm[1], hm[2]) * inv, P = mk3<R>(hd[0], hd[1], hd[2]), ga = mk3<R>(gh[0], gh[1], gh[2]);
  const V3<R> cb = cross(ga, P);  // the adjoint of c
  EmSeed<R> e;
  e.Pb.a = ga; e.Pb.l = mk3<R>(gh[3], gh[4], gh[5]) + cross(c, ga);
  e.xb = cb * inv - mk3<R>(M.gravity[0], M.gravity[1], M.gravity[2]) * gU;
  e.mb = -dot(cb, c) * inv;
  return e;
}
// backward stage 3 (after jcdb_init, jc_moments, jcd_vel), lanes over bodies: Y_i, the body's wrench, the springs' position gradient, the
// inertia gradient (gI: fp64 [10 * nb][gIB] or nullptr, zero off the tree)
template <class R>
NB2_HD void emb_bodies(const Nb2ModelDev<R>& M, const R* q, int root, const double* wi, size_t wiB, R gT, R gU, const R* gh, R* ws, double* gI,
                       size_t gIB, int lane, int nl) {
  const EmLayout L = em_layout(M.nb, M.ndof, true);
  const EmSeed<R> e = em_seed(M, root, ws, gU, gh);
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) {
      if (gI) for (int k = 0; k < 10; k++) gI[(size_t)(10 * i + k) * gIB] = 0.0;
      continue;
    }
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    const V6<R> V = ldv6(ws + L.oV + 6 * i), Vb = AdInvT(W, V), Pbb = AdInvT(W, e.Pb);
    const V6<R> Y = dAdInvT(W, mulG(m, h, Ib, Vb * gT + Pbb)), P = dAdInvT(W, mulG(m, h, Ib, Vb));
    const V3<R> x = W.p * m + mul(W.R_, h);
    V6<R> X = zero6<R>() - jd_wrench(V, Y) - jd_wrench(e.Pb, P);
    X.a = X.a + cross(x, e.xb); X.l = X.l + e.xb * m;
    put6(ws + L.oP + 6 * i, Y);
    put6(ws + L.oX + 6 * i, X);
    const int o = M.dof_off[i];
    for (int k = 0; k < mm_nd(M.jtype[i]); k++) ws[L.oGq + o + k] += gU * M.spring[o + k] * (q[o + k] - M.rest[o + k]);
    if (gI) {
      const V6<R> u = Vb * (R(0.5) * gT) + Pbb;
      const V3<R> gh_ = cross(Vb.l, u.a) + cross(u.l, Vb.a) + mulT(W.R_, e.xb);
      const R gm = dot(u.l, Vb.l) + dot(W.p, e.xb) + e.mb;
      double* t = gI + (size_t)(10 * i) * gIB;
      t[0] = (double)gm; t[gIB] = (double)gh_.x; t[2 * gIB] = (double)gh_.y; t[3 * gIB] = (double)gh_.z;
      t[4 * gIB] = (double)(u.a.x * Vb.a.x); t[5 * gIB] = (double)(u.a.y * Vb.a.y); t[6 * gIB] = (double)(u.a.z * Vb.a.z);
      t[7 * gIB] = (double)(u.a.x * Vb.a.y + u.a.y * Vb.a.x);
      t[8 * gIB] = (double)(u.a.x * Vb.a.z + u.a.z * Vb.a.x);
      t[9 * gIB] = (double)(u.a.y * Vb.a.z + u.a.z * Vb.a.y);
    }
  }
}
// backward stage 4, lane 0: leaf -> root, Y and Gam summed over each subtree, dL/dqdot and the joints' position gradients
template <class R> NB2_HD void emb_reduce(const Nb2ModelDev<R>& M, const R* q, const R* qd, int root, R* ws, int lane) {
  if (lane != 0) return;
  const EmLayout L = em_layout(M.nb, M.ndof, true);
  const int n = M.ndof;
  R* gq = ws + L.oGq;
  for (int i = M.nb - 1; i >= root; i--) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const V6<R> Ys = ldv6(ws + L.oP + 6 * i);
    V6<R> G = ldv6(ws + L.oX + 6 * i);
    const int p = M.parent[i], jt = M.jtype[i], o = M.dof_off[i];
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k));
      gq[n + o + k] += dot(s, Ys);
      G = G + jd_wrench(s, Ys * qd[o + k]);
    }
    jd_joint_grad(M, q, i, dAdT(W, G), gq);
    if (p >= 0) { put6(ws + L.oP + 6 * p, ldv6(ws + L.oP + 6 * p) + Ys); put6(ws + L.oX + 6 * p, ldv6(ws + L.oX + 6 * p) + G); }
  }
}

}  // namespace nb2
