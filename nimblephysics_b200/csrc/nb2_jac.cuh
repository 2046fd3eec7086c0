// World Jacobians of body points and of a skeleton's centre of mass, batched (DESIGN.md §6i).  Columns are in the step's velocity
// coordinates (free joints: body twist, S = I6), in the world's dof order, as M of nb2_mm.cuh.
//   body point e (canonical body b, point x_b in b's frame): J_e [6, n] with J_e qdot = [omega_b ; d/dt p_e], world axes.  The column of
//     a dof k on the chain root -> b is [a_k ; b_k + a_k x p_e], s_k = [a_k ; b_k] its world screw about the world origin; other columns are 0.
//   centre of mass of the tree rooted at r: J_com [3, n], column k = (M_k b_k + a_k x H_k) / m_tot, M_k / H_k the mass and the world
//     first moment (sum m_i p_i + R_i h_i) of the bodies at or below the body of dof k.
//
// Every function below is one stage of a kernel, run on lane `lane` of `nl` with the lanes exchanging data only between stages (the
// kernels put a __syncwarp there), so a host build can run a stage's lanes in any order — the pattern of nb2_mm.cuh.
//
// Backward (L = <G, J>).  A joint j moved by the world twist xi = [w; v] moves everything at or below it rigidly: the columns of the dofs
// at or below j rotate (dc = [w x a ; w x c_lin], the point moving with them), and the point moves under the columns above j
// (dc_lin = a_k x dp, dp = w x p_e + v).  So dL/dxi is the world wrench
//   point:  Gam_j = [ sum_{k at/below j} (a_k x ga_k + c_k,lin x gl_k) + p_e x P_j ; P_j ],   P_j = sum_{k above j} gl_k x a_k
//   COM:    Gam_j = [ sum_{k in subtree(j)} c_k x g_k + H_j x U_p(j) ; M_j U_p(j) ] / m_tot,  U_i = sum_{k on chain(i)} g_k x a_k
// carried to the joint's child frame (c_j = X*^T Gam_j): S^T c_j for a revolute / prismatic dof, the free joint's [phi; p] through
// Jr(phi) (cid_free_q_grad).  The offset gradient is R_e^T sum_k gl_k x a_k; the COM's mass gradient is
//   dL/dm_i = (beta_i + p_i . U_i) / m_tot - L / m_tot,   dL/dh_i = R_i^T U_i / m_tot,   beta_i = sum_{k on chain(i)} g_k . b_k.
#pragma once
#include "nb2_mm.cuh"

#define NB2_MAX_JACOBIAN_NODES 32  // node records travel in a __grid_constant__ parameter (see JacNodes below)

namespace nb2 {

// the nodes of one call: canonical body (-1: static, an all-zero block) and the body's frame <- node frame (R row-major 9, p 3)
template <class R> struct JacNodes {
  int k;
  int body[NB2_MAX_JACOBIAN_NODES];
  R T[NB2_MAX_JACOBIAN_NODES][12];
};

template <class R> NB2_HD Xf<R> jac_mul(const Xf<R>& A, const Xf<R>& B) { Xf<R> C; C.R_ = mul(A.R_, B.R_); C.p = mul(A.R_, B.p) + A.p; return C; }
template <class R> NB2_HD Xf<R> jac_eye() { Xf<R> T; T.R_ = eye3<R>(); T.p = zero3<R>(); return T; }
template <class R> NB2_HD int jac_root(const Nb2ModelDev<R>& M, int i) { while (M.parent[i] >= 0) i = M.parent[i]; return i; }
// the node's point in the frame of its body: T (R o + p), o = nullptr: the node's origin
template <class R> NB2_HD V3<R> jac_node_point(const R* T, const R* o) {
  const Xf<R> X = ldXf<R, 1>(T);
  return o ? mul(X.R_, mk3<R>(o[0], o[1], o[2])) + X.p : X.p;
}

// ---- body point, forward: one warp per (world, node).  Working set: col [6][n] (the output block, row-major), W_b [12], p_e [3].
struct JpLayout { int oCol, oW, oP, total; };
NB2_HD JpLayout jp_layout(int n) { JpLayout L; L.oCol = 0; L.oW = 6 * n; L.oP = L.oW + 12; L.total = (L.oP + 3 + 3) & ~3; return L; }

// stage 0, lanes over words: zeroed block
template <class R> NB2_HD void jp_zero(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) { mm_zero(ws, 6 * M.ndof, lane, nl); }
// stage 1, lane 0: leaf -> root, each chain dof's screw in the frame of b (T = pose of b in the joint's frame), then W_b and p_e
template <class R> NB2_HD void jp_walk(const Nb2ModelDev<R>& M, const R* q, int b, const R* Tn, const R* o, R* ws, int lane) {
  if (lane != 0 || b < 0) return;
  const JpLayout L = jp_layout(M.ndof);
  const int n = M.ndof;
  Xf<R> T = jac_eye<R>();
  for (int j = b; j >= 0; j = M.parent[j]) {
    const int jt = M.jtype[j], o0 = M.dof_off[j];
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdInvT(T, mm_S<R>(jt, k));
      for (int r = 0; r < 6; r++) ws[L.oCol + r * n + o0 + k] = comp6(s, r);
    }
    T = jac_mul(cid_xf(M, j, q), T);
  }
  stXf<R, 1>(ws + L.oW, T);
  const V3<R> p = mul(T.R_, jac_node_point(Tn, o)) + T.p;
  ws[L.oP] = p.x; ws[L.oP + 1] = p.y; ws[L.oP + 2] = p.z;
}
// stage 2, lanes over columns: world screw and the point's velocity (columns off the chain stay 0)
template <class R> NB2_HD void jp_columns(const Nb2ModelDev<R>& M, int b, R* ws, int lane, int nl) {
  if (b < 0) return;
  const JpLayout L = jp_layout(M.ndof);
  const int n = M.ndof;
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  for (int d = lane; d < n; d += nl) {
    R* c = ws + L.oCol + d;
    V6<R> s; s.a = mk3<R>(c[0], c[n], c[2 * n]); s.l = mk3<R>(c[3 * n], c[4 * n], c[5 * n]);
    if (s.a.x == R(0) && s.a.y == R(0) && s.a.z == R(0) && s.l.x == R(0) && s.l.y == R(0) && s.l.z == R(0)) continue;
    s = AdT(W, s);
    s.l = s.l + cross(s.a, p);
    for (int r = 0; r < 6; r++) c[r * n] = comp6(s, r);
  }
}

// ---- body point, backward: one warp per world, its nodes one after the other (the warp owns the world's gradient row).  Working set:
// gq [n], T_{j<-b} [nb][12] of the chain bodies, chain screws in frame b [n][6], r_t / u_t [n][6], W_b [12], p_e [3], R_e [12] and the
// chain (dof, body) int16 pairs leaf -> root [n].
struct JpbLayout { int oGq, oT, oS, oRU, oW, oP, oRe, oCh, total; };
NB2_HD JpbLayout jpb_layout(int nb, int n) {
  JpbLayout L;
  L.oGq = 0; L.oT = n; L.oS = L.oT + 12 * nb; L.oRU = L.oS + 6 * n; L.oW = L.oRU + 6 * n; L.oP = L.oW + 12; L.oRe = L.oP + 3; L.oCh = L.oRe + 12;
  L.total = L.oCh + n;  // the chain: 2n int16 in n words of R >= 4 bytes
  return L;
}
template <class R> NB2_HD void jpb_init(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) {
  for (int d = lane; d < M.ndof; d += nl) ws[jpb_layout(M.nb, M.ndof).oGq + d] = R(0);
}
// node stage a, lane 0: the chain leaf -> root, T_{j<-b}, each chain dof's screw in frame b, W_b, p_e and R_e.  Returns nothing; the
// chain length is re-derived by jpb_chain_len.
template <class R> NB2_HD void jpb_walk(const Nb2ModelDev<R>& M, const R* q, int b, const R* Tn, const R* o, R* ws, int lane) {
  if (lane != 0 || b < 0) return;
  const JpbLayout L = jpb_layout(M.nb, M.ndof);
  int16_t* ch = reinterpret_cast<int16_t*>(ws + L.oCh);
  Xf<R> T = jac_eye<R>();
  int t = 0;
  for (int j = b; j >= 0; j = M.parent[j]) {
    stXf<R, 1>(ws + L.oT + 12 * j, T);
    const int jt = M.jtype[j];
    for (int k = 0; k < mm_nd(jt); k++, t++) {
      put6(ws + L.oS + 6 * t, AdInvT(T, mm_S<R>(jt, k)));
      ch[2 * t] = (int16_t)(M.dof_off[j] + k); ch[2 * t + 1] = (int16_t)j;
    }
    T = jac_mul(cid_xf(M, j, q), T);
  }
  stXf<R, 1>(ws + L.oW, T);
  const Xf<R> Te = ldXf<R, 1>(Tn);
  const V3<R> p = mul(T.R_, jac_node_point(Tn, o)) + T.p;
  const M3<R> Re = mul(T.R_, Te.R_);
  ws[L.oP] = p.x; ws[L.oP + 1] = p.y; ws[L.oP + 2] = p.z;
  stXf<R, 1>(ws + L.oRe, Xf<R>{Re, zero3<R>()});
}
template <class R> NB2_HD int jpb_chain_len(const Nb2ModelDev<R>& M, int b) {
  int D = 0;
  for (int j = b; j >= 0; j = M.parent[j]) D += mm_nd(M.jtype[j]);
  return D;
}
// node stage b, lanes over the chain's dofs: world screw, incoming column gradient g (row-major [6][n]), r_t and u_t
template <class R> NB2_HD void jpb_terms(const Nb2ModelDev<R>& M, int b, const R* g, R* ws, int lane, int nl) {
  const JpbLayout L = jpb_layout(M.nb, M.ndof);
  const int n = M.ndof, D = jpb_chain_len(M, b);
  const int16_t* ch = reinterpret_cast<const int16_t*>(ws + L.oCh);
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  for (int t = lane; t < D; t += nl) {
    const int d = ch[2 * t];
    const V6<R> s = AdT(W, ldv6(ws + L.oS + 6 * t));
    const V3<R> ga = mk3<R>(g[d], g[n + d], g[2 * n + d]), gl = mk3<R>(g[3 * n + d], g[4 * n + d], g[5 * n + d]);
    const V3<R> cl = s.l + cross(s.a, p);
    V6<R> ru; ru.a = cross(s.a, ga) + cross(cl, gl); ru.l = cross(gl, s.a);
    put6(ws + L.oRU + 6 * t, ru);
  }
}
// node stage c, lane 0: leaf -> root over the chain's joints, the joints' position gradients; the offset gradient (go: [3] or nullptr).
// PE: the loss also depends on the point itself, with adjoint pe [3]; the point moves with every joint of the chain, so pe joins the
// column term P of every joint and the offset gradient.
template <class R, bool PE = false>
NB2_HD void jpb_reduce(const Nb2ModelDev<R>& M, const R* q, int b, R* ws, R* go, int lane, const R* pe = nullptr) {
  if (lane != 0) return;
  const JpbLayout L = jpb_layout(M.nb, M.ndof);
  const int D = jpb_chain_len(M, b);
  const int16_t* ch = reinterpret_cast<const int16_t*>(ws + L.oCh);
  R* gq = ws + L.oGq;
  V3<R> Ptot = zero3<R>();
  for (int t = 0; t < D; t++) Ptot = Ptot + ldv6(ws + L.oRU + 6 * t).l;
  if (PE) Ptot = Ptot + mk3<R>(pe[0], pe[1], pe[2]);
  if (go) {
    const V3<R> v = b >= 0 ? mulT(ldXf<R, 1>(ws + L.oRe).R_, Ptot) : zero3<R>();
    go[0] = v.x; go[1] = v.y; go[2] = v.z;
  }
  if (b < 0) return;
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  V3<R> Rs = zero3<R>(), Us = zero3<R>();
  for (int t = 0; t < D;) {
    const int j = ch[2 * t + 1];
    int t1 = t;
    for (; t1 < D && ch[2 * t1 + 1] == j; t1++) { const V6<R> ru = ldv6(ws + L.oRU + 6 * t1); Rs = Rs + ru.a; Us = Us + ru.l; }
    const V3<R> P = Ptot - Us;
    V6<R> G; G.a = Rs + cross(p, P); G.l = P;
    const V6<R> c = dAdInvT(ldXf<R, 1>(ws + L.oT + 12 * j), dAdT(W, G));
    const int jt = M.jtype[j], o = M.dof_off[j];
    if (jt == NB2_JT_FREE) cid_free_q_grad(q, o, c, gq);
    else gq[o] += S_dot(jt, c);
    t = t1;
  }
}
template <class R> NB2_HD void jpb_store_row(const Nb2ModelDev<R>& M, const R* ws, R* gpos, int lane, int nl) {
  for (int d = lane; d < M.ndof; d += nl) gpos[d] = ws[jpb_layout(M.nb, M.ndof).oGq + d];
}

// ---- centre of mass: one warp per world.  Working set: W [nb][12] (joint transforms, then world poses), HM [nb][4] (subtree first
// moment and mass), then forward: col [3][n]; backward: UB [nb][4] (U_i, beta_i), C [nb][4] (subtree sum of c_k x g_k, and g_k . c_k
// of the body's own dofs), gq [n].  The tree's total mass sits in word oMt.
struct JcLayout { int oW, oHM, oMt, oCol, oUB, oC, oGq, total; };
NB2_HD JcLayout jc_layout(int nb, int n, bool bwd) {
  JcLayout L;
  L.oW = 0; L.oHM = 12 * nb; L.oMt = L.oHM + 4 * nb; L.oCol = L.oMt + 4;
  L.oUB = L.oCol; L.oC = L.oUB + 4 * nb; L.oGq = L.oC + 4 * nb;
  L.total = bwd ? ((L.oGq + n + 3) & ~3) : ((L.oCol + 3 * n + 3) & ~3);
  return L;
}
// stage 0, lanes over bodies / words: the joint transforms of the tree's bodies; forward: zeroed block, backward: gq = 0
template <class R> NB2_HD void jc_init(const Nb2ModelDev<R>& M, const R* q, int root, bool bwd, R* ws, int lane, int nl) {
  const JcLayout L = jc_layout(M.nb, M.ndof, bwd);
  for (int i = lane; i < M.nb; i += nl) if (jac_root(M, i) == root) stXf<R, 1>(ws + L.oW + 12 * i, cid_xf(M, i, q));
  if (bwd) for (int d = lane; d < M.ndof; d += nl) ws[L.oGq + d] = R(0);
  else mm_zero(ws + L.oCol, 3 * M.ndof, lane, nl);
}
// stage 1, lane 0: world poses root -> leaf, each body's first moment and mass, summed leaf -> root; the total mass
template <class R> NB2_HD void jc_moments(const Nb2ModelDev<R>& M, int root, const double* wi, size_t wiB, R* ws, int lane, int nl) {
  if (lane != 0) return;
  const JcLayout L = jc_layout(M.nb, M.ndof, false);
  for (int i = root; i < M.nb; i++) {
    if (jac_root(M, i) != root) continue;
    const int p = M.parent[i];
    const Xf<R> W = p >= 0 ? jac_mul(ldXf<R, 1>(ws + L.oW + 12 * p), ldXf<R, 1>(ws + L.oW + 12 * i)) : ldXf<R, 1>(ws + L.oW + 12 * i);
    stXf<R, 1>(ws + L.oW + 12 * i, W);
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    const V3<R> x = W.p * m + mul(W.R_, h);
    R* hm = ws + L.oHM + 4 * i;
    hm[0] = x.x; hm[1] = x.y; hm[2] = x.z; hm[3] = m;
  }
  for (int i = M.nb - 1; i > root; i--) {
    const int p = M.parent[i];
    if (p < 0 || jac_root(M, i) != root) continue;
    for (int k = 0; k < 4; k++) ws[L.oHM + 4 * p + k] += ws[L.oHM + 4 * i + k];
  }
  ws[L.oMt] = ws[L.oHM + 4 * root + 3];
}
// forward stage 2, lanes over the tree's bodies: the columns of each body's dofs
template <class R> NB2_HD void jc_columns(const Nb2ModelDev<R>& M, int root, R* ws, int lane, int nl) {
  const JcLayout L = jc_layout(M.nb, M.ndof, false);
  const int n = M.ndof;
  const R inv = R(1) / ws[L.oMt];
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const R* hm = ws + L.oHM + 4 * i;
    const V3<R> H = mk3<R>(hm[0], hm[1], hm[2]);
    const int jt = M.jtype[i], o = M.dof_off[i];
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k));
      const V3<R> c = (s.l * hm[3] + cross(s.a, H)) * inv;
      ws[L.oCol + o + k] = c.x; ws[L.oCol + n + o + k] = c.y; ws[L.oCol + 2 * n + o + k] = c.z;
    }
  }
}
// backward stage 2, lanes over the tree's bodies: per body, u_i = sum g_k x a_k, beta_i = sum g_k . b_k, sum c_k x g_k and sum g_k . c_k
// over its own dofs (c_k unnormalised); g row-major [3][n]
template <class R> NB2_HD void jcb_terms(const Nb2ModelDev<R>& M, int root, const R* g, R* ws, int lane, int nl) {
  const JcLayout L = jc_layout(M.nb, M.ndof, true);
  const int n = M.ndof;
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const R* hm = ws + L.oHM + 4 * i;
    const V3<R> H = mk3<R>(hm[0], hm[1], hm[2]);
    const int jt = M.jtype[i], o = M.dof_off[i];
    V3<R> u = zero3<R>(), C = zero3<R>();
    R beta = R(0), sd = R(0);
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k));
      const V3<R> gk = mk3<R>(g[o + k], g[n + o + k], g[2 * n + o + k]);
      const V3<R> c = s.l * hm[3] + cross(s.a, H);
      u = u + cross(gk, s.a); beta += dot(gk, s.l); C = C + cross(c, gk); sd += dot(gk, c);
    }
    R* ub = ws + L.oUB + 4 * i; ub[0] = u.x; ub[1] = u.y; ub[2] = u.z; ub[3] = beta;
    R* cc = ws + L.oC + 4 * i; cc[0] = C.x; cc[1] = C.y; cc[2] = C.z; cc[3] = sd;
  }
}
// backward stage 3, lane 0: U and beta root -> leaf (prefix over the chain), the subtree sums of C leaf -> root, L * m_tot into word oMt + 1
template <class R> NB2_HD void jcb_sums(const Nb2ModelDev<R>& M, int root, R* ws, int lane) {
  if (lane != 0) return;
  const JcLayout L = jc_layout(M.nb, M.ndof, true);
  R S = R(0);
  for (int i = root; i < M.nb; i++) {
    if (jac_root(M, i) != root) continue;
    S += ws[L.oC + 4 * i + 3];
    const int p = M.parent[i];
    if (p >= 0) for (int k = 0; k < 4; k++) ws[L.oUB + 4 * i + k] += ws[L.oUB + 4 * p + k];
  }
  for (int i = M.nb - 1; i > root; i--) {
    const int p = M.parent[i];
    if (p < 0 || jac_root(M, i) != root) continue;
    for (int k = 0; k < 3; k++) ws[L.oC + 4 * p + k] += ws[L.oC + 4 * i + k];
  }
  ws[L.oMt + 1] = S;
}
// backward stage 4, lanes over bodies: the position gradient of each body's dofs, its inertia gradient (gI: fp64 [10 * nb][gIB] or nullptr,
// zero off the tree)
template <class R> NB2_HD void jcb_grads(const Nb2ModelDev<R>& M, const R* q, int root, R* ws, double* gI, size_t gIB, int lane, int nl) {
  const JcLayout L = jc_layout(M.nb, M.ndof, true);
  const R mt = ws[L.oMt], inv = R(1) / mt, S = ws[L.oMt + 1];
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) {
      if (gI) for (int k = 0; k < 10; k++) gI[(size_t)(10 * i + k) * gIB] = 0.0;
      continue;
    }
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const int p = M.parent[i], jt = M.jtype[i], o = M.dof_off[i];
    const R* hm = ws + L.oHM + 4 * i;
    const V3<R> Up = p >= 0 ? mk3<R>(ws[L.oUB + 4 * p], ws[L.oUB + 4 * p + 1], ws[L.oUB + 4 * p + 2]) : zero3<R>();
    V6<R> G;
    G.a = (mk3<R>(ws[L.oC + 4 * i], ws[L.oC + 4 * i + 1], ws[L.oC + 4 * i + 2]) + cross(mk3<R>(hm[0], hm[1], hm[2]), Up)) * inv;
    G.l = Up * (hm[3] * inv);
    const V6<R> c = dAdT(W, G);
    if (jt == NB2_JT_FREE) cid_free_q_grad(q, o, c, ws + L.oGq);
    else ws[L.oGq + o] += S_dot(jt, c);
    if (gI) {
      const R* ub = ws + L.oUB + 4 * i;
      const V3<R> U = mk3<R>(ub[0], ub[1], ub[2]), gh = mulT(W.R_, U) * inv;
      const R gm = (ub[3] + dot(W.p, U)) * inv - S * inv * inv;
      double* t = gI + (size_t)(10 * i) * gIB;
      t[0] = (double)gm; t[gIB] = (double)gh.x; t[2 * gIB] = (double)gh.y; t[3 * gIB] = (double)gh.z;
      for (int k = 4; k < 10; k++) t[k * gIB] = 0.0;
    }
  }
}
template <class R> NB2_HD void jcb_store_row(const Nb2ModelDev<R>& M, const R* ws, R* gpos, int lane, int nl) {
  for (int d = lane; d < M.ndof; d += nl) gpos[d] = ws[jc_layout(M.nb, M.ndof, true).oGq + d];
}

// ==== time derivatives of the Jacobians above (DESIGN.md §6j), at the state [q ; qdot]: Jdot = d/dt J(q(t)) along a motion through q
// with velocity qdot (free joints: Rdot = R [omega]x, pdot = R v, the tangent of the step's position update), so that
// xddot_e = J_e qddot + Jdot_e qdot.  With V_c(k) the world spatial velocity of the body dof k moves (the chain's s_j qdot_j summed from the
// root down to that body, its own joint included) and V_b = [w_b ; v_b] the velocity of the node's body:
//   sdot_k = V_c(k) xm s_k ([w ; v] xm [a ; b] = [w x a ; w x b + v x a], `ad`),   pdot_e = v_b + w_b x p_e
//   body point: column k = [adot_k ; bdot_k + adot_k x p_e + a_k x pdot_e]
//   COM:        column k = (M_k bdot_k + adot_k x H_k + a_k x Hdot_k) / m_tot,   Hdot = sum m_i v_i + w_i x x_i (x_i = m_i p_i + R_i h_i)
//
// Backward (L = <G, Jdot>).  Everything is a function of the world screws s_k, the point p_e (COM: the bodies' first moments x_i) and
// qdot.  Reverse mode through the formulas above gives the adjoints sbar_k = the direct terms + qdot_k * (the sum of Vbar over the
// velocities s_k enters), and dL/dqdot_k = <s_k, that same sum>.  A joint j moved by the world twist xi moves every screw and point at or
// below it rigidly (ds = xi xm s, dp = w x p + v, dx = w x x + m v), so dL/dxi is the world wrench
//   Gam_j = sum_{k at/below j} [a_k x abar_k + b_k x bbar_k ; a_k x bbar_k] + sum_{points at/below j} [p x pbar ; pbar]   (COM: [x x xbar ; m xbar])
// carried to the joint's frame and its coordinates as in the backwards above.  jd_wrench is the screw term.
template <class R> NB2_HD V6<R> jd_wrench(const V6<R>& s, const V6<R>& sb) {
  V6<R> r; r.a = cross(s.a, sb.a) + cross(s.l, sb.l); r.l = cross(s.a, sb.l); return r;
}
// the joint's coordinate gradient from its frame's wrench c (accumulated into gq)
template <class R> NB2_HD void jd_joint_grad(const Nb2ModelDev<R>& M, const R* q, int j, const V6<R>& c, R* gq) {
  const int jt = M.jtype[j], o = M.dof_off[j];
  if (jt == NB2_JT_FREE) cid_free_q_grad(q, o, c, gq);
  else gq[o] += S_dot(jt, c);
}

// ---- body point, forward: one warp per (world, node).  Working set: col [6][n] (the output block, row-major; the chain's screws in frame
// b first), Vlo [n][6] (frame b: the velocity of the chain below each dof's body), W_b [12], p_e [3], V_b [6] (frame b).
struct JpdLayout { int oCol, oV, oW, oP, oVb, total; };
NB2_HD JpdLayout jpd_layout(int n) {
  JpdLayout L; L.oCol = 0; L.oV = 6 * n; L.oW = 12 * n; L.oP = L.oW + 12; L.oVb = L.oP + 3; L.total = (L.oVb + 6 + 3) & ~3; return L;
}
// stage 1, lane 0 (after jp_zero): leaf -> root as jp_walk, each chain dof's screw and the velocity of the chain below its body (frame b)
template <class R> NB2_HD void jpd_walk(const Nb2ModelDev<R>& M, const R* q, const R* qd, int b, const R* Tn, const R* o, R* ws, int lane) {
  if (lane != 0 || b < 0) return;
  const JpdLayout L = jpd_layout(M.ndof);
  const int n = M.ndof;
  Xf<R> T = jac_eye<R>();
  V6<R> lo = zero6<R>();
  for (int j = b; j >= 0; j = M.parent[j]) {
    const int jt = M.jtype[j], o0 = M.dof_off[j];
    V6<R> own = zero6<R>();
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdInvT(T, mm_S<R>(jt, k));
      for (int r = 0; r < 6; r++) ws[L.oCol + r * n + o0 + k] = comp6(s, r);
      put6(ws + L.oV + 6 * (o0 + k), lo);
      own = own + s * qd[o0 + k];
    }
    lo = lo + own;
    T = jac_mul(cid_xf(M, j, q), T);
  }
  stXf<R, 1>(ws + L.oW, T);
  const V3<R> p = mul(T.R_, jac_node_point(Tn, o)) + T.p;
  ws[L.oP] = p.x; ws[L.oP + 1] = p.y; ws[L.oP + 2] = p.z;
  put6(ws + L.oVb, lo);
}
// stage 2, lanes over columns: the columns of Jdot (columns off the chain stay 0)
template <class R> NB2_HD void jpd_columns(const Nb2ModelDev<R>& M, int b, R* ws, int lane, int nl) {
  if (b < 0) return;
  const JpdLayout L = jpd_layout(M.ndof);
  const int n = M.ndof;
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  const V6<R> Vbb = ldv6(ws + L.oVb), Vb = AdT(W, Vbb);
  const V3<R> pd = Vb.l + cross(Vb.a, p);
  for (int d = lane; d < n; d += nl) {
    R* c = ws + L.oCol + d;
    V6<R> s; s.a = mk3<R>(c[0], c[n], c[2 * n]); s.l = mk3<R>(c[3 * n], c[4 * n], c[5 * n]);
    if (s.a.x == R(0) && s.a.y == R(0) && s.a.z == R(0) && s.l.x == R(0) && s.l.y == R(0) && s.l.z == R(0)) continue;
    s = AdT(W, s);
    const V6<R> sd = ad(AdT(W, Vbb - ldv6(ws + L.oV + 6 * d)), s);
    V6<R> col; col.a = sd.a; col.l = sd.l + cross(sd.a, p) + cross(s.a, pd);
    for (int r = 0; r < 6; r++) c[r * n] = comp6(col, r);
  }
}

// ---- body point, backward: one warp per world, its nodes one after the other.  Working set: gq [2n] (dL/dq, dL/dqdot), T_{j<-b} [nb][12],
// per chain dof t (leaf -> root): S [n][6] (screw, frame b, then world), V [n][6] (velocity below, frame b, then Vbar_c), Sb [n][6] (the
// direct screw adjoint), PP [n][6] (gl x a and gl x adot); W_b [12], p_e [3], V_b [6] (frame b), R_e [12], the chain (dof, body) int16
// pairs [n].
struct JpdbLayout { int oGq, oT, oS, oV, oSb, oPP, oW, oP, oVb, oRe, oCh, total; };
NB2_HD JpdbLayout jpdb_layout(int nb, int n) {
  JpdbLayout L;
  L.oGq = 0; L.oT = 2 * n; L.oS = L.oT + 12 * nb; L.oV = L.oS + 6 * n; L.oSb = L.oV + 6 * n; L.oPP = L.oSb + 6 * n; L.oW = L.oPP + 6 * n;
  L.oP = L.oW + 12; L.oVb = L.oP + 3; L.oRe = L.oVb + 6; L.oCh = L.oRe + 12;
  L.total = (L.oCh + n + 3) & ~3;  // the chain: 2n int16 in n words of R >= 4 bytes
  return L;
}
template <class R> NB2_HD void jpdb_init(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) { mm_zero(ws + jpdb_layout(M.nb, M.ndof).oGq, 2 * M.ndof, lane, nl); }
// node stage a, lane 0: the chain leaf -> root (as jpb_walk), each chain dof's screw and the velocity below its body, W_b, p_e, V_b, R_e
template <class R> NB2_HD void jpdb_walk(const Nb2ModelDev<R>& M, const R* q, const R* qd, int b, const R* Tn, const R* o, R* ws, int lane) {
  if (lane != 0 || b < 0) return;
  const JpdbLayout L = jpdb_layout(M.nb, M.ndof);
  int16_t* ch = reinterpret_cast<int16_t*>(ws + L.oCh);
  Xf<R> T = jac_eye<R>();
  V6<R> lo = zero6<R>();
  int t = 0;
  for (int j = b; j >= 0; j = M.parent[j]) {
    stXf<R, 1>(ws + L.oT + 12 * j, T);
    const int jt = M.jtype[j];
    V6<R> own = zero6<R>();
    for (int k = 0; k < mm_nd(jt); k++, t++) {
      const V6<R> s = AdInvT(T, mm_S<R>(jt, k));
      put6(ws + L.oS + 6 * t, s);
      put6(ws + L.oV + 6 * t, lo);
      own = own + s * qd[M.dof_off[j] + k];
      ch[2 * t] = (int16_t)(M.dof_off[j] + k); ch[2 * t + 1] = (int16_t)j;
    }
    lo = lo + own;
    T = jac_mul(cid_xf(M, j, q), T);
  }
  stXf<R, 1>(ws + L.oW, T);
  const Xf<R> Te = ldXf<R, 1>(Tn);
  const V3<R> p = mul(T.R_, jac_node_point(Tn, o)) + T.p;
  ws[L.oP] = p.x; ws[L.oP + 1] = p.y; ws[L.oP + 2] = p.z;
  put6(ws + L.oVb, lo);
  stXf<R, 1>(ws + L.oRe, Xf<R>{mul(T.R_, Te.R_), zero3<R>()});
}
// node stage b, lanes over the chain's dofs: world screw, Vbar_c = ad*(sdot adjoint), the direct screw adjoint, gl x a and gl x adot
// (g: the node's incoming block, row-major [6][n])
template <class R> NB2_HD void jpdb_terms(const Nb2ModelDev<R>& M, int b, const R* g, R* ws, int lane, int nl) {
  if (b < 0) return;
  const JpdbLayout L = jpdb_layout(M.nb, M.ndof);
  const int n = M.ndof, D = jpb_chain_len(M, b);
  const int16_t* ch = reinterpret_cast<const int16_t*>(ws + L.oCh);
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  const V6<R> Vbb = ldv6(ws + L.oVb), Vb = AdT(W, Vbb);
  const V3<R> pd = Vb.l + cross(Vb.a, p);
  for (int t = lane; t < D; t += nl) {
    const int d = ch[2 * t];
    const V6<R> s = AdT(W, ldv6(ws + L.oS + 6 * t)), V = AdT(W, Vbb - ldv6(ws + L.oV + 6 * t));
    const V6<R> sd = ad(V, s);
    const V3<R> ga = mk3<R>(g[d], g[n + d], g[2 * n + d]), gl = mk3<R>(g[3 * n + d], g[4 * n + d], g[5 * n + d]);
    V6<R> e; e.a = ga + cross(p, gl); e.l = gl;  // the adjoint of sdot
    V6<R> sb; sb.a = cross(e.a, V.a) + cross(e.l, V.l) + cross(pd, gl); sb.l = cross(e.l, V.a);
    V6<R> pp; pp.a = cross(gl, s.a); pp.l = cross(gl, sd.a);
    put6(ws + L.oS + 6 * t, s);
    put6(ws + L.oV + 6 * t, jd_wrench(s, e));
    put6(ws + L.oSb + 6 * t, sb);
    put6(ws + L.oPP + 6 * t, pp);
  }
}
// node stage c, lane 0: leaf -> root over the chain's joints, dL/dqdot and the joints' position gradients; the offset gradient (go: [3]
// or nullptr)
template <class R> NB2_HD void jpdb_reduce(const Nb2ModelDev<R>& M, const R* q, const R* qd, int b, R* ws, R* go, int lane) {
  if (lane != 0) return;
  const JpdbLayout L = jpdb_layout(M.nb, M.ndof);
  if (b < 0) {
    if (go) go[0] = go[1] = go[2] = R(0);
    return;
  }
  const int n = M.ndof, D = jpb_chain_len(M, b);
  const int16_t* ch = reinterpret_cast<const int16_t*>(ws + L.oCh);
  R* gq = ws + L.oGq;
  const Xf<R> W = ldXf<R, 1>(ws + L.oW);
  const V3<R> p = mk3<R>(ws[L.oP], ws[L.oP + 1], ws[L.oP + 2]);
  const V6<R> Vb = AdT(W, ldv6(ws + L.oVb));
  V3<R> P = zero3<R>(), pb = zero3<R>();
  for (int t = 0; t < D; t++) { const V6<R> pp = ldv6(ws + L.oPP + 6 * t); P = P + pp.a; pb = pb + pp.l; }
  pb = pb + cross(P, Vb.a);  // pdot = v_b + w_b x p
  if (go) {
    const V3<R> v = mulT(ldXf<R, 1>(ws + L.oRe).R_, pb);
    go[0] = v.x; go[1] = v.y; go[2] = v.z;
  }
  V6<R> Vs; Vs.a = cross(p, P); Vs.l = P;      // Vbar_b; below, the sum of Vbar over the velocities a dof enters
  V6<R> G; G.a = cross(p, pb); G.l = pb;       // the point moves with every joint of the chain
  for (int t = 0; t < D;) {
    const int j = ch[2 * t + 1];
    int t1 = t;
    for (; t1 < D && ch[2 * t1 + 1] == j; t1++) Vs = Vs + ldv6(ws + L.oV + 6 * t1);
    for (int u = t; u < t1; u++) {
      const int d = ch[2 * u];
      const V6<R> s = ldv6(ws + L.oS + 6 * u);
      gq[n + d] += dot(s, Vs);
      G = G + jd_wrench(s, ldv6(ws + L.oSb + 6 * u) + Vs * qd[d]);
    }
    jd_joint_grad(M, q, j, dAdInvT(ldXf<R, 1>(ws + L.oT + 12 * j), dAdT(W, G)), gq);
    t = t1;
  }
}
// the world's gradient row [2n]
template <class R> NB2_HD void jd_store_row(int n, const R* gq, R* gs, int lane, int nl) { for (int d = lane; d < 2 * n; d += nl) gs[d] = gq[d]; }

// ---- centre of mass: one warp per world.  Working set: jc_layout's W, HM and the total mass (jc_init / jc_moments fill them), then
// forward: col [3][n]; both: V [nb][6] (world velocities), Hd [nb][4] (subtree Hdot); backward: gq [2n], Sb [n][6] (direct screw
// adjoints), A [nb][8] (Hbar, Hdbar, Mbar, then their sums over the ancestors; the body's share of L * m_tot), Vbar [nb][6], X [nb][6]
// (the first moment's wrench, then the subtree's Gam).  Word oMt + 1 holds L * m_tot.
struct JcdLayout { int oW, oHM, oMt, oCol, oV, oHd, oGq, oSb, oA, oVb, oX, total; };
NB2_HD JcdLayout jcd_layout(int nb, int n, bool bwd) {
  const JcLayout C = jc_layout(nb, n, false);
  JcdLayout L;
  L.oW = C.oW; L.oHM = C.oHM; L.oMt = C.oMt; L.oCol = C.oCol;
  L.oV = L.oCol + (bwd ? 0 : 3 * n); L.oHd = L.oV + 6 * nb;
  L.oGq = L.oHd + 4 * nb; L.oSb = L.oGq + 2 * n; L.oA = L.oSb + 6 * n; L.oVb = L.oA + 8 * nb; L.oX = L.oVb + 6 * nb;
  L.total = ((bwd ? L.oX + 6 * nb : L.oGq) + 3) & ~3;
  return L;
}
// backward stage 0, lanes over bodies / words: the joint transforms of the tree's bodies (as jc_init), gq = 0
template <class R> NB2_HD void jcdb_init(const Nb2ModelDev<R>& M, const R* q, int root, R* ws, int lane, int nl) {
  const JcdLayout L = jcd_layout(M.nb, M.ndof, true);
  for (int i = lane; i < M.nb; i += nl) if (jac_root(M, i) == root) stXf<R, 1>(ws + L.oW + 12 * i, cid_xf(M, i, q));
  mm_zero(ws + L.oGq, 2 * M.ndof, lane, nl);
}
// stage 2 (after jc_moments), lane 0: world velocities root -> leaf, each body's Hdot share summed leaf -> root
template <class R> NB2_HD void jcd_vel(const Nb2ModelDev<R>& M, const R* qd, int root, const double* wi, size_t wiB, bool bwd, R* ws, int lane) {
  if (lane != 0) return;
  const JcdLayout L = jcd_layout(M.nb, M.ndof, bwd);
  for (int i = root; i < M.nb; i++) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const int p = M.parent[i], jt = M.jtype[i], o = M.dof_off[i];
    V6<R> V = p >= 0 ? ldv6(ws + L.oV + 6 * p) : zero6<R>();
    for (int k = 0; k < mm_nd(jt); k++) V = V + AdT(W, mm_S<R>(jt, k)) * qd[o + k];
    put6(ws + L.oV + 6 * i, V);
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    const V3<R> xd = V.l * m + cross(V.a, W.p * m + mul(W.R_, h));
    R* hd = ws + L.oHd + 4 * i;
    hd[0] = xd.x; hd[1] = xd.y; hd[2] = xd.z; hd[3] = R(0);
  }
  for (int i = M.nb - 1; i > root; i--) {
    const int p = M.parent[i];
    if (p < 0 || jac_root(M, i) != root) continue;
    for (int k = 0; k < 3; k++) ws[L.oHd + 4 * p + k] += ws[L.oHd + 4 * i + k];
  }
}
// forward stage 3, lanes over the tree's bodies: the columns of each body's dofs
template <class R> NB2_HD void jcd_columns(const Nb2ModelDev<R>& M, int root, R* ws, int lane, int nl) {
  const JcdLayout L = jcd_layout(M.nb, M.ndof, false);
  const int n = M.ndof;
  const R inv = R(1) / ws[L.oMt];
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const R* hm = ws + L.oHM + 4 * i;
    const V3<R> H = mk3<R>(hm[0], hm[1], hm[2]), Hd = mk3<R>(ws[L.oHd + 4 * i], ws[L.oHd + 4 * i + 1], ws[L.oHd + 4 * i + 2]);
    const V6<R> V = ldv6(ws + L.oV + 6 * i);
    const int jt = M.jtype[i], o = M.dof_off[i];
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k)), sd = ad(V, s);
      const V3<R> c = (sd.l * hm[3] + cross(sd.a, H) + cross(s.a, Hd)) * inv;
      ws[L.oCol + o + k] = c.x; ws[L.oCol + n + o + k] = c.y; ws[L.oCol + 2 * n + o + k] = c.z;
    }
  }
}
// backward stage 3, lanes over the tree's bodies: per body, the direct adjoints of its dofs' screws, Vbar from its sdot terms, and
// Hbar = sum g x adot, Hdbar = sum g x a, Mbar = sum g . bdot, the body's share of L * m_tot; g row-major [3][n]
template <class R> NB2_HD void jcdb_terms(const Nb2ModelDev<R>& M, int root, const R* g, R* ws, int lane, int nl) {
  const JcdLayout L = jcd_layout(M.nb, M.ndof, true);
  const int n = M.ndof;
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const R* hm = ws + L.oHM + 4 * i;
    const V3<R> H = mk3<R>(hm[0], hm[1], hm[2]), Hd = mk3<R>(ws[L.oHd + 4 * i], ws[L.oHd + 4 * i + 1], ws[L.oHd + 4 * i + 2]);
    const V6<R> V = ldv6(ws + L.oV + 6 * i);
    const int jt = M.jtype[i], o = M.dof_off[i];
    V3<R> Hb = zero3<R>(), Hdb = zero3<R>();
    V6<R> Vb = zero6<R>();
    R Mb = R(0), Lp = R(0);
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k)), sd = ad(V, s);
      const V3<R> gk = mk3<R>(g[o + k], g[n + o + k], g[2 * n + o + k]);
      Lp += dot(gk, sd.l * hm[3] + cross(sd.a, H) + cross(s.a, Hd));
      V6<R> e; e.a = cross(H, gk); e.l = gk * hm[3];  // the adjoint of sdot
      V6<R> sb; sb.a = cross(e.a, V.a) + cross(e.l, V.l) + cross(Hd, gk); sb.l = cross(e.l, V.a);
      put6(ws + L.oSb + 6 * (o + k), sb);
      Vb = Vb + jd_wrench(s, e);
      Hb = Hb + cross(gk, sd.a); Hdb = Hdb + cross(gk, s.a); Mb += dot(gk, sd.l);
    }
    R* a = ws + L.oA + 8 * i;
    a[0] = Hb.x; a[1] = Hb.y; a[2] = Hb.z; a[3] = Hdb.x; a[4] = Hdb.y; a[5] = Hdb.z; a[6] = Mb; a[7] = Lp;
    put6(ws + L.oVb + 6 * i, Vb);
  }
}
// backward stage 4, lane 0: Hbar, Hdbar and Mbar summed over each body's ancestors (root -> leaf), L * m_tot into word oMt + 1
template <class R> NB2_HD void jcdb_prefix(const Nb2ModelDev<R>& M, int root, R* ws, int lane) {
  if (lane != 0) return;
  const JcdLayout L = jcd_layout(M.nb, M.ndof, true);
  R S = R(0);
  for (int i = root; i < M.nb; i++) {
    if (jac_root(M, i) != root) continue;
    S += ws[L.oA + 8 * i + 7];
    const int p = M.parent[i];
    if (p >= 0) for (int k = 0; k < 7; k++) ws[L.oA + 8 * i + k] += ws[L.oA + 8 * p + k];
  }
  ws[L.oMt + 1] = S;
}
// backward stage 5, lanes over bodies: the first moment's adjoint (x enters H and Hdot), its wrench, Vbar from Hdot, and the inertia
// gradient (gI: fp64 [10 * nb][gIB] or nullptr, zero off the tree)
template <class R> NB2_HD void jcdb_bodies(const Nb2ModelDev<R>& M, int root, const double* wi, size_t wiB, R* ws, double* gI, size_t gIB, int lane,
                                           int nl) {
  const JcdLayout L = jcd_layout(M.nb, M.ndof, true);
  const R inv = R(1) / ws[L.oMt], S = ws[L.oMt + 1];
  for (int i = lane; i < M.nb; i += nl) {
    if (jac_root(M, i) != root) {
      if (gI) for (int k = 0; k < 10; k++) gI[(size_t)(10 * i + k) * gIB] = 0.0;
      continue;
    }
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    const V3<R> x = W.p * m + mul(W.R_, h);
    const R* a = ws + L.oA + 8 * i;
    const V3<R> Y = mk3<R>(a[3], a[4], a[5]);
    const V6<R> V = ldv6(ws + L.oV + 6 * i);
    V6<R> Vb = ldv6(ws + L.oVb + 6 * i);
    Vb.a = Vb.a + cross(x, Y); Vb.l = Vb.l + Y * m;
    put6(ws + L.oVb + 6 * i, Vb);
    const V3<R> xb = mk3<R>(a[0], a[1], a[2]) + cross(Y, V.a);
    V6<R> X; X.a = cross(x, xb); X.l = xb * m;
    put6(ws + L.oX + 6 * i, X);
    if (gI) {
      const V3<R> gh = mulT(W.R_, xb) * inv;
      const R gm = (a[6] + dot(Y, V.l) + dot(W.p, xb)) * inv - S * inv * inv;
      double* t = gI + (size_t)(10 * i) * gIB;
      t[0] = (double)gm; t[gIB] = (double)gh.x; t[2 * gIB] = (double)gh.y; t[3 * gIB] = (double)gh.z;
      for (int k = 4; k < 10; k++) t[k * gIB] = 0.0;
    }
  }
}
// backward stage 6, lane 0: leaf -> root, Vbar and Gam summed over each subtree, dL/dqdot and the joints' position gradients
template <class R> NB2_HD void jcdb_reduce(const Nb2ModelDev<R>& M, const R* q, const R* qd, int root, R* ws, int lane) {
  if (lane != 0) return;
  const JcdLayout L = jcd_layout(M.nb, M.ndof, true);
  const int n = M.ndof;
  const R inv = R(1) / ws[L.oMt];
  R* gq = ws + L.oGq;
  for (int i = M.nb - 1; i >= root; i--) {
    if (jac_root(M, i) != root) continue;
    const Xf<R> W = ldXf<R, 1>(ws + L.oW + 12 * i);
    const V6<R> Vs = ldv6(ws + L.oVb + 6 * i);
    V6<R> G = ldv6(ws + L.oX + 6 * i);
    const int p = M.parent[i], jt = M.jtype[i], o = M.dof_off[i];
    for (int k = 0; k < mm_nd(jt); k++) {
      const V6<R> s = AdT(W, mm_S<R>(jt, k));
      gq[n + o + k] += dot(s, Vs) * inv;
      G = G + jd_wrench(s, ldv6(ws + L.oSb + 6 * (o + k)) + Vs * qd[o + k]);
    }
    jd_joint_grad(M, q, i, dAdT(W, G * inv), gq);
    if (p >= 0) { put6(ws + L.oVb + 6 * p, ldv6(ws + L.oVb + 6 * p) + Vs); put6(ws + L.oX + 6 * p, ldv6(ws + L.oX + 6 * p) + G); }
  }
}

}  // namespace nb2
