// Inverse-dynamics and energy regressors, batched (DESIGN.md §6n): the joint forces and energies of the contact-free step as linear maps
// of every canonical body's inertial parameters pi_j = (m, h, Ibar) (the layout of modelspec.mass_to_inertia).
//   ID:      tau(q, qdot, v'; pi) = sum_j Y[., j] . pi_j + tau_passive,   tau_passive = K (q - q0 + qdot dt) + D qdot
//            Y[d, j] = t(W, A_j) - t(ad(V_j, W), V_j)   with W = S_d carried to body j's frame (0 unless d's joint is at or above j)
//   energy:  T = sum_j YT[j] . pi_j,  YT[j] = 1/2 t(V_j, V_j);   U = sum_j YU[j] . pi_j + 1/2 sum_d k_d (q_d - q0_d)^2,
//            YU[j] = (-g . p_j, -R_j^T g, 0, ..., 0)
// t(Y, X) = d(Y^T G X)/d(m, h, Ibar) is inertia_param_form, V_j / A_j the body's velocity and acceleration (gravity as a base
// acceleration) in its own frame, and (R_j, p_j) its world pose.  Row d of Y is the ID backward's inertia gradient seeded with e_d
// (id_bwd_mass, where W is the field id_bwd_field sums over every dof).
//
// ONE WARP PER WORLD.  The working set (arithmetic type R, stride 1) sits in shared memory:
//   F    the ID forward scratch (fwd_layout): q, qdot, v', every body's V, sin/cos and A after the kinematics stages
//   X    [nb][12] world poses
//   S    [n][6] every dof's motion axis in world axes about the world origin
//   Y    the output buffer: one row of Y [nb][10], or YT and YU [2][nb][10]
// Every function is one stage: lanes exchange data only between stages (the kernels put a __syncwarp there), so a host build can run a
// stage's lanes in any order.  The stages reuse dj_load and the ID forward's passes (id_forward_stage) unchanged.
#pragma once
#include "nb2_djac.cuh"
#include "nb2_jac.cuh"

namespace nb2 {

struct RegLayout { int oF, oX, oS, oY, total; };
NB2_HD RegLayout reg_layout(int nb, int n, int nslots, int nfree, bool energy) {
  RegLayout L;
  L.oF = 0;
  L.oX = fwd_layout(nb, n, nslots, nfree).total;
  L.oS = L.oX + 12 * nb;
  L.oY = L.oS + 6 * n;
  L.total = (L.oY + (energy ? 20 : 10) * nb + 3) & ~3;
  return L;
}
template <class R> NB2_HD RegLayout reg_layout(const Nb2ModelDev<R>& M, bool energy) { return reg_layout(M.nb, M.ndof, M.nslots, M.nfree, energy); }

// stages 1 (trunk, lane 0) and 2 (limbs) on lane `lane` of the model's schedule (lanes >= M.lanes idle): V and A of every body
template <class R> NB2_HD void reg_kinematics(const Nb2ModelDev<R>& M, R* ws, int lane, int stage) {
  if (lane >= M.lanes) return;
  id_forward_stage<R, 1>(M, ws, nullptr, 1, false, lane, stage, nullptr, nullptr, 0);
}
// stage 3, lane 0: world poses root -> leaf
template <class R> NB2_HD void reg_poses(const Nb2ModelDev<R>& M, R* ws, int lane) {
  if (lane != 0) return;
  const RegLayout L = reg_layout(M, false);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  for (int i = 0; i < M.nb; i++) {
    const int p = M.parent[i];
    const Xf<R> T = body_xf_fwd<R, 1>(M, i, ws, F);
    stXf<R, 1>(ws + L.oX + 12 * i, p >= 0 ? jac_mul(ldXf<R, 1>(ws + L.oX + 12 * p), T) : T);
  }
}
// stage 4, lanes over bodies: the world axes of the body's dofs and (tp != nullptr) their passive forces K (q - q0 + qdot dt) + D qdot
template <class R> NB2_HD void reg_axes(const Nb2ModelDev<R>& M, R* ws, R* tp, int lane, int nl) {
  const RegLayout L = reg_layout(M, false);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  for (int i = lane; i < M.nb; i += nl) {
    const int jt = M.jtype[i], o = M.dof_off[i];
    const Xf<R> X = ldXf<R, 1>(ws + L.oX + 12 * i);
    for (int k = 0; k < mm_nd(jt); k++) {
      const int d = o + k;
      put6(ws + L.oS + 6 * d, AdT(X, mm_S<R>(jt, k)));
      if (tp) {
        const R qd = ws[F.oQ + d], vd = ws[F.oV + d];
        tp[d] = M.spring[d] * (qd - M.rest[d] + vd * M.dt) + M.damping[d] * vd;
      }
    }
  }
}
// stage 5 of ID row d, lanes over bodies: Y[d, j] of every body into the buffer.  In pre-order the bodies at or below dof d's body b are
// b .. e - 1, e the first later body whose parent precedes b.  (Dof offsets need not grow with the body index, hence the scan for b.)
template <class R> NB2_HD void reg_id_row(const Nb2ModelDev<R>& M, R* ws, int d, int lane, int nl) {
  const RegLayout L = reg_layout(M, false);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  int b = 0;
  while (d < M.dof_off[b] || d >= M.dof_off[b] + mm_nd(M.jtype[b])) b++;
  int e = b + 1;
  while (e < M.nb && M.parent[e] >= b) e++;
  const V6<R> Sw = ldv6(ws + L.oS + 6 * d);
  for (int j = lane; j < M.nb; j += nl) {
    R* y = ws + L.oY + 10 * j;
    if (j < b || j >= e) {
      for (int k = 0; k < 10; k++) y[k] = R(0);
      continue;
    }
    const R* bs = ws + F.oBody + NB2_FWD_BODY_WORDS * j;
    const V6<R> W = AdInvT(ldXf<R, 1>(ws + L.oX + 12 * j), Sw), V = ld6<R, 1>(bs), A = ld6<R, 1>(bs + 8);
    V6<R> Y2;
    Y2.a = cross_rn(V.a, W.a);
    Y2.l = cross_rn(V.a, W.l) + cross_rn(V.l, W.a);
    R t[10], t2[10];
    inertia_param_form(W, A, t);
    inertia_param_form(Y2, V, t2);
    for (int k = 0; k < 10; k++) y[k] = t[k] - t2[k];
  }
}
// energy stage 5, lanes over bodies: YT[j] and YU[j] into the buffer
template <class R> NB2_HD void reg_energy_cols(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) {
  const RegLayout L = reg_layout(M, true);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const V3<R> g = mk3<R>(M.gravity[0], M.gravity[1], M.gravity[2]);
  for (int j = lane; j < M.nb; j += nl) {
    const V6<R> V = ld6<R, 1>(ws + F.oBody + NB2_FWD_BODY_WORDS * j);
    const Xf<R> X = ldXf<R, 1>(ws + L.oX + 12 * j);
    R t[10];
    inertia_param_form(V, V, t);
    R* yt = ws + L.oY + 10 * j;
    R* yu = yt + 10 * M.nb;
    for (int k = 0; k < 10; k++) { yt[k] = R(0.5) * t[k]; yu[k] = R(0); }
    const V3<R> rg = mulT(X.R_, g);
    yu[0] = -dot(g, X.p); yu[1] = -rg.x; yu[2] = -rg.y; yu[3] = -rg.z;
  }
}
// lane 0: 1/2 sum_d k_d (q_d - q0_d)^2 in dof order
template <class R> NB2_HD void reg_spring_energy(const Nb2ModelDev<R>& M, const R* ws, R* out, int lane) {
  if (lane != 0) return;
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  R s = R(0);
  for (int d = 0; d < M.ndof; d++) { const R e = ws[F.oQ + d] - M.rest[d]; s += R(0.5) * M.spring[d] * e * e; }
  *out = s;
}

// lanes over words: `count` contiguous words of the buffer to global memory, consecutive lanes on consecutive addresses.  On the device a
// streaming store: the output is written once and not read back by the kernel.
template <class R> NB2_HD void reg_store(const R* buf, R* dst, int count, int lane, int nl) {
  for (int k = lane; k < count; k += nl) {
#ifdef __CUDA_ARCH__
    __stcs(dst + k, buf[k]);
#else
    dst[k] = buf[k];
#endif
  }
}

}  // namespace nb2
