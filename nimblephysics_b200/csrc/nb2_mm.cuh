// Joint-space mass matrix M(q) and its inverse, batched (DESIGN.md §6h).  M is the matrix the step inverts, in the step's velocity
// coordinates (free joints: body twist, S = I6), block-diagonal over trees; contacts, limits, springs and damping are not part of it.
//
// ONE WARP PER WORLD.  The world's working set sits in that warp's slice of shared memory (stride 1, arithmetic type R), the n x n
// result is staged there and written as one contiguous block.  Every function below is one stage of a kernel: it runs on lane `lane`
// of `nl`, and lanes exchange data only between stages (the kernels put a __syncwarp there), so a host build can run a stage's lanes
// in any order.  All outputs are exactly symmetric: one triangle is computed and mirrored.
#pragma once
#include "nb2_dyn.cuh"

namespace nb2 {

// dofs of body i and the column k of its S
NB2_HD int mm_nd(int jt) { return jt == NB2_JT_FREE ? 6 : 1; }
template <class R> NB2_HD V6<R> mm_S(int jt, int k) {
  V6<R> s = zero6<R>();
  if (jt == NB2_JT_FREE) { if (k < 3) (&s.a.x)[k] = R(1); else (&s.l.x)[k - 3] = R(1); }
  else if (jt == NB2_JT_REV) s.a.z = R(1);
  else s.l.z = R(1);
  return s;
}
template <class R> NB2_HD V6<R> ldv6(const R* p) { return row6(p); }

// zero n*n words of the staging from lane `lane` of `nl`
template <class R> NB2_HD void mm_zero(R* mat, int nn, int lane, int nl) { for (int k = lane; k < nn; k += nl) mat[k] = R(0); }

// ---- M forward: the composite-rigid-body algorithm.  Working set: X [nb][12] (parent <- child at q), Ic [nb][21], mat [n][n].
struct MmLayout { int oX, oI, oMat, total; };
NB2_HD MmLayout mm_layout(int nb, int n) { MmLayout L; L.oX = 0; L.oI = 12 * nb; L.oMat = (L.oI + 21 * nb + 3) & ~3; L.total = L.oMat + n * n; return L; }

// stage 0, lanes over bodies: joint transforms, each body's own inertia, zeroed staging
template <class R> NB2_HD void crba_init(const Nb2ModelDev<R>& M, const R* q, const double* wi, size_t wiB, R* ws, int lane, int nl) {
  const MmLayout L = mm_layout(M.nb, M.ndof);
  for (int i = lane; i < M.nb; i += nl) {
    if (M.parent[i] >= 0) stXf<R, 1>(ws + L.oX + 12 * i, cid_xf(M, i, q));
    R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, i, &m, &h, &Ib);
    stSI<R, 1, false>(ws + L.oI + 21 * i, rigidSI(m, h, Ib));
  }
  mm_zero(ws + L.oMat, M.ndof * M.ndof, lane, nl);
}
// stage 1, lane 0: composite inertias leaf -> root
template <class R> NB2_HD void crba_composite(const Nb2ModelDev<R>& M, R* ws, int lane) {
  if (lane != 0) return;
  const MmLayout L = mm_layout(M.nb, M.ndof);
  for (int i = M.nb - 1; i >= 0; i--) {
    const int p = M.parent[i];
    if (p < 0) continue;
    stSI<R, 1, true>(ws + L.oI + 21 * p, xform_inertia(ldXf<R, 1>(ws + L.oX + 12 * i), ldSI<R, 1>(ws + L.oI + 21 * i)));
  }
}
// stage 2, lanes over bodies: F = Ic_i S_a carried to the root; M[dof_j][dof_a] = S_j^T F for every dof j at or above dof a
template <class R> NB2_HD void crba_columns(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) {
  const MmLayout L = mm_layout(M.nb, M.ndof);
  const int n = M.ndof;
  R* mat = ws + L.oMat;
  for (int i = lane; i < M.nb; i += nl) {
    const int jti = M.jtype[i], nd = mm_nd(jti);
    const SI<R> Ic = ldSI<R, 1>(ws + L.oI + 21 * i);
    for (int a = 0; a < nd; a++) {
      const int da = M.dof_off[i] + a;
      V6<R> F = mul(Ic, mm_S<R>(jti, a));
      for (int b = 0; b <= a; b++) {
        const R v = (jti == NB2_JT_FREE) ? comp6(F, b) : S_dot(jti, F);
        mat[(size_t)da * n + M.dof_off[i] + b] = v; mat[(size_t)(M.dof_off[i] + b) * n + da] = v;
      }
      for (int j = i; M.parent[j] >= 0;) {
        F = dAdInvT(ldXf<R, 1>(ws + L.oX + 12 * j), F);
        j = M.parent[j];
        const int jt = M.jtype[j], o = M.dof_off[j];
        for (int b = 0; b < mm_nd(jt); b++) {
          const R v = (jt == NB2_JT_FREE) ? comp6(F, b) : S_dot(jt, F);
          mat[(size_t)da * n + o + b] = v; mat[(size_t)(o + b) * n + da] = v;
        }
      }
    }
  }
}

// ---- M^-1 forward: the step's articulated inertias (fwd_pass1 / fwd_pass2 at zero velocity and force) and one bias-free unit-force
// sweep pair per column (leaf -> root along the column's chain, then root -> leaf over its tree).  Working set: the forward scratch
// (fwd_layout), the free bodies' (I^A)^-1 [nfree][21], per lane u [n] and A [nb][6], mat [n][n].
struct MinvLayout { int oScr, oIinv, oLane, laneW, oMat, total; };
NB2_HD MinvLayout minv_layout(int nb, int n, int nslots, int nfree, int nl) {
  MinvLayout L;
  L.oScr = 0; L.oIinv = fwd_layout(nb, n, nslots, nfree).total; L.oLane = L.oIinv + 21 * nfree; L.laneW = n + 6 * nb;
  L.oMat = (L.oLane + nl * L.laneW + 3) & ~3; L.total = L.oMat + n * n;
  return L;
}
// stage 0, lanes over words: q in, zero velocity and force, zeroed staging
template <class R> NB2_HD void minv_init(const Nb2ModelDev<R>& M, const R* q, R* ws, int lane, int nl) {
  const MinvLayout L = minv_layout(M.nb, M.ndof, M.nslots, M.nfree, nl);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  for (int d = lane; d < M.ndof; d += nl) { ws[L.oScr + F.oQ + d] = q[d]; ws[L.oScr + F.oV + d] = R(0); }
  for (int a = lane; a < M.na; a += nl) ws[L.oScr + F.oAct + a] = R(0);
  mm_zero(ws + L.oMat, M.ndof * M.ndof, lane, nl);
}
// stage 1, lane 0: the step's kinematics and articulated-inertia passes over the whole tree
template <class R> NB2_HD void minv_articulated(const Nb2ModelDev<R>& M, R* ws, const double* wi, size_t wiB, int lane, int nl) {
  if (lane != 0) return;
  const MinvLayout L = minv_layout(M.nb, M.ndof, M.nslots, M.nfree, nl);
  fwd_pass1<R, 1>(M, ws + L.oScr, 0, M.nb);
  fwd_pass2<R, 1>(M, ws + L.oScr, nullptr, 0, false, 0, M.nb, ws + L.oIinv, wi, wiB);
}
// stage 2, lanes over columns: column d of M^-1 (rows >= d written, mirrored)
template <class R> NB2_HD void minv_columns(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) {
  const MinvLayout L = minv_layout(M.nb, M.ndof, M.nslots, M.nfree, nl);
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof;
  R* scr = ws + L.oScr;
  R* u = ws + L.oLane + lane * L.laneW;
  R* A = u + n;
  R* mat = ws + L.oMat;
  for (int d = lane; d < n; d += nl) {
    int b = 0;  // the body owning dof d: dofs keep the model's order, which need not follow the bodies' DFS order (SDF Atlas)
    while (b + 1 < M.nb && !(M.dof_off[b] <= d && d < M.dof_off[b] + mm_nd(M.jtype[b]))) b++;
    for (int k = 0; k < n; k++) u[k] = R(0);
    // leaf -> root: the unit force at dof d, then the bias force each joint passes to its parent
    u[d] = R(1);
    V6<R> beta;
    {
      const int jt = M.jtype[b], o = M.dof_off[b];
      if (jt == NB2_JT_FREE) beta = mm_S<R>(jt, d - o);  // a 6-dof joint passes its own joint force on
      else { const R* bs = scr + F.oBody + NB2_FWD_BODY_WORDS * b; beta = ldv6(bs + 8) * bs[14]; }
    }
    int r = b;
    for (int i = b; M.parent[i] >= 0;) {
      const V6<R> pA = dAdInvT(body_xf_fwd<R, 1>(M, i, scr, F), beta);
      i = M.parent[i]; r = i;
      const int jt = M.jtype[i], o = M.dof_off[i];
      if (jt == NB2_JT_FREE) {
        for (int k = 0; k < 6; k++) u[o + k] = -comp6(pA, k);
        break;  // transmits pA + u = 0
      }
      const R* bs = scr + F.oBody + NB2_FWD_BODY_WORDS * i;
      const V6<R> U = ldv6(bs + 8);
      u[o] = -S_dot(jt, pA);
      beta = pA + U * (bs[14] * u[o]);
    }
    while (M.parent[r] >= 0) r = M.parent[r];
    // root -> leaf over the tree: qdd and the accelerations
    for (int i = r; i < M.nb && (i == r || M.parent[i] >= 0); i++) {
      const int jt = M.jtype[i], o = M.dof_off[i], p = M.parent[i];
      const V6<R> Ap = (p >= 0) ? AdInvT(body_xf_fwd<R, 1>(M, i, scr, F), ldv6(A + 6 * p)) : zero6<R>();
      V6<R> Ai;
      if (jt == NB2_JT_FREE) {
        const V6<R> y = mul(ldSI<R, 1>(ws + L.oIinv + 21 * M.free_idx[i]), ldv6(u + o));
        const V6<R> qdd = y - Ap;
        for (int k = 0; k < 6; k++) if (o + k >= d) { const R v = comp6(qdd, k); mat[(size_t)(o + k) * n + d] = v; mat[(size_t)d * n + o + k] = v; }
        Ai = y;
      } else {
        const R* bs = scr + F.oBody + NB2_FWD_BODY_WORDS * i;
        const R qdd = bs[14] * (u[o] - dot(ldv6(bs + 8), Ap));
        if (o >= d) { mat[(size_t)o * n + d] = qdd; mat[(size_t)d * n + o] = qdd; }
        Ai = Ap + S_times<R>(jt, qdd);
      }
      put6(A + 6 * i, Ai);
    }
  }
}

// ---- backward.  L = <G, M> with Gs = (G + G^T)/2 and M = sum_b J_b^T G_b J_b, J_b body b's body-frame Jacobian (columns c_k = X_{b<-j(k)} S_k
// over the dofs k at or above b).  With w_k = sum_l Gs_kl c_l and f_k = G_b w_k:
//   dL/d(inertia of b) = sum_k form(c_k, w_k)                             (inertia_param_form)
//   dL/dxi_m = -2 c_m^T sum_{k strictly above m} c_k x* f_k  for every joint m at or above b  (d c_k / d q_m = c_k x S_m in frame m)
// The columns are formed from the tree-root frame (Xr: each body's pose relative to its tree's root body), so nothing depends on a free
// root's pose and the root's own dofs get no term.  Working set: X [nb][12], Xr [nb][12], s [n][6] (S_k in the root frame), Gs [n][n],
// c [n][6], r [n][6] (c_k x* f_k), per-lane partial inertia gradients [nl][10], gq [n], the chain's dofs [n] and bodies [n] (ints).
struct MmbLayout { int oX, oXr, oS, oG, oC, oRr, oT, oGq, oChain, total; };
NB2_HD MmbLayout mmb_layout(int nb, int n, int nl) {
  MmbLayout L;
  L.oX = 0; L.oXr = 12 * nb; L.oS = L.oXr + 12 * nb; L.oG = L.oS + 6 * n; L.oC = L.oG + n * n; L.oRr = L.oC + 6 * n; L.oT = L.oRr + 6 * n;
  L.oGq = L.oT + 10 * nl; L.oChain = L.oGq + n; L.total = L.oChain + n;  // the chain: 2n int16 in n words of R >= 4 bytes
  return L;
}
// stage 0, lanes over bodies / entries: transforms, Gs from the row-major gradient g (nullptr: Gs already staged), gq = 0
template <class R> NB2_HD void mmb_init(const Nb2ModelDev<R>& M, const R* q, const R* g, R* ws, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int n = M.ndof;
  for (int i = lane; i < M.nb; i += nl) if (M.parent[i] >= 0) stXf<R, 1>(ws + L.oX + 12 * i, cid_xf(M, i, q));
  if (g) for (int e = lane; e < n * n; e += nl) { const int i = e / n, j = e - i * n; ws[L.oG + e] = R(0.5) * (g[e] + g[(size_t)j * n + i]); }
  for (int d = lane; d < n; d += nl) ws[L.oGq + d] = R(0);
}
// stage 1, lane 0: poses relative to the tree root, root -> leaf, and every dof's S in its root frame
template <class R> NB2_HD void mmb_root_frames(const Nb2ModelDev<R>& M, R* ws, int lane, int nl) {
  if (lane != 0) return;
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  for (int i = 0; i < M.nb; i++) {
    const int p = M.parent[i];
    Xf<R> T;
    if (p < 0) { T.R_ = eye3<R>(); T.p = zero3<R>(); }
    else {
      const Xf<R> A = ldXf<R, 1>(ws + L.oXr + 12 * p), X = ldXf<R, 1>(ws + L.oX + 12 * i);
      T.R_ = mul(A.R_, X.R_); T.p = mul(A.R_, X.p) + A.p;
    }
    stXf<R, 1>(ws + L.oXr + 12 * i, T);
    const int jt = M.jtype[i];
    for (int k = 0; k < mm_nd(jt); k++) put6(ws + L.oS + 6 * (M.dof_off[i] + k), AdT(T, mm_S<R>(jt, k)));
  }
}
// body b, stage a, lane 0: the chain of b, its dofs leaf -> root (int16 pairs: dof, body)
template <class R> NB2_HD int mmb_chain(const Nb2ModelDev<R>& M, const R* ws, int b, int nl, const int16_t** ch) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  *ch = reinterpret_cast<const int16_t*>(ws + L.oChain);
  int D = 0;
  for (int j = b; j >= 0; j = M.parent[j]) D += mm_nd(M.jtype[j]);
  return D;
}
template <class R> NB2_HD void mmb_body_chain(const Nb2ModelDev<R>& M, R* ws, int b, int lane, int nl) {
  if (lane != 0) return;
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  int16_t* ch = reinterpret_cast<int16_t*>(ws + L.oChain);
  int t = 0;
  for (int j = b; j >= 0; j = M.parent[j])
    for (int k = mm_nd(M.jtype[j]) - 1; k >= 0; k--) { ch[2 * t] = (int16_t)(M.dof_off[j] + k); ch[2 * t + 1] = (int16_t)j; t++; }
}
// body b, stage b, lanes over the chain's dofs: c_k in frame b
template <class R> NB2_HD void mmb_body_columns(const Nb2ModelDev<R>& M, R* ws, int b, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int16_t* ch; const int D = mmb_chain(M, ws, b, nl, &ch);
  const Xf<R> Tb = ldXf<R, 1>(ws + L.oXr + 12 * b);
  for (int t = lane; t < D; t += nl) put6(ws + L.oC + 6 * t, AdInvT(Tb, ldv6(ws + L.oS + 6 * ch[2 * t])));
}
// body b, stage c, lanes over the chain's dofs: w_k, f_k, r_k and the lane's share of the inertia gradient
template <class R> NB2_HD void mmb_body_forces(const Nb2ModelDev<R>& M, R* ws, int b, const double* wi, size_t wiB, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int n = M.ndof;
  const int16_t* ch; const int D = mmb_chain(M, ws, b, nl, &ch);
  R m; V3<R> h; S3<R> Ib; inertia_of(M, wi, wiB, b, &m, &h, &Ib);
  R acc[10];
  for (int k = 0; k < 10; k++) acc[k] = R(0);
  for (int t = lane; t < D; t += nl) {
    const R* grow = ws + L.oG + (size_t)ch[2 * t] * n;
    V6<R> w = zero6<R>();
    for (int e = 0; e < D; e++) w = w + ldv6(ws + L.oC + 6 * e) * grow[ch[2 * e]];
    const V6<R> c = ldv6(ws + L.oC + 6 * t);
    put6(ws + L.oRr + 6 * t, crf(c, mulG(m, h, Ib, w)));
    R tk[10]; inertia_param_form(c, w, tk);
    for (int k = 0; k < 10; k++) acc[k] += tk[k];
  }
  for (int k = 0; k < 10; k++) ws[L.oT + 10 * lane + k] = acc[k];
}
// body b, stage d, lane 0: the inertia gradient of b, and the joints' terms root -> b (prefix of r over the dofs strictly above each joint)
template <class R> NB2_HD void mmb_body_reduce(const Nb2ModelDev<R>& M, R* ws, int b, double* gI, size_t gIB, int lane, int nl) {
  if (lane != 0) return;
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int16_t* ch; const int D = mmb_chain(M, ws, b, nl, &ch);
  if (gI) for (int k = 0; k < 10; k++) {
    R s = R(0);
    for (int l = 0; l < nl; l++) s += ws[L.oT + 10 * l + k];
    gI[(size_t)(10 * b + k) * gIB] = (double)s;
  }
  V6<R> P = zero6<R>();
  bool above = false;  // the tree root's dofs have nothing above them: they get no term at all
  for (int t = D - 1; t >= 0;) {
    const int j = ch[2 * t + 1];
    int t0 = t;
    while (t0 > 0 && ch[2 * (t0 - 1) + 1] == j) t0--;
    if (above) for (int s = t0; s <= t; s++) ws[L.oGq + ch[2 * s]] -= R(2) * dot(ldv6(ws + L.oC + 6 * s), P);
    for (int s = t0; s <= t; s++) P = P + ldv6(ws + L.oRr + 6 * s);
    above = true;
    t = t0 - 1;
  }
}
// stage after the last body, lanes over bodies: a non-root free joint's twist dual -> dL/d[phi; p] (cid_free_q_grad)
template <class R> NB2_HD void mmb_free_q(const Nb2ModelDev<R>& M, const R* q, R* ws, int lane, int nl) {
  R* gq = ws + mmb_layout(M.nb, M.ndof, nl).oGq;
  for (int i = lane; i < M.nb; i += nl) {
    if (M.jtype[i] != NB2_JT_FREE || M.parent[i] < 0) continue;
    const int o = M.dof_off[i];
    const V6<R> c = ldv6(gq + o);
    for (int k = 0; k < 6; k++) gq[o + k] = R(0);
    cid_free_q_grad(q, o, c, gq);
  }
}
template <class R> NB2_HD void mmb_store_row(const Nb2ModelDev<R>& M, const R* ws, R* gpos, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  for (int d = lane; d < M.ndof; d += nl) gpos[d] = ws[L.oGq + d];
}

// ---- M^-1 backward: G_M = -M^-1 Gs M^-1, then the M backward.  Stage 1: T = Gs Minv into the caller's workspace row (lanes over rows);
// stage 2: Gs <- -(Minv T), symmetrised pairwise (lanes over pairs i <= j).  Minv staged in the mat words after the M-backward working set.
NB2_HD int mminvb_words(int nb, int n, int nl) { return mmb_layout(nb, n, nl).total + n * n; }
template <class R> NB2_HD void mminvb_load(const Nb2ModelDev<R>& M, const R* minv, const R* g, R* ws, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int n = M.ndof;
  R* mi = ws + L.total;
  for (int e = lane; e < n * n; e += nl) {
    const int i = e / n, j = e - i * n;
    mi[e] = minv[e];
    ws[L.oG + e] = R(0.5) * (g[e] + g[(size_t)j * n + i]);
  }
}
template <class R> NB2_HD void mminvb_left(const Nb2ModelDev<R>& M, const R* ws, R* T, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int n = M.ndof;
  const R* mi = ws + L.total;
  for (int e = lane; e < n * n; e += nl) {
    const int i = e / n, j = e - i * n;
    R s = R(0);
    for (int k = 0; k < n; k++) s += ws[L.oG + i * n + k] * mi[k * n + j];
    T[e] = s;
  }
}
template <class R> NB2_HD void mminvb_right(const Nb2ModelDev<R>& M, R* ws, const R* T, int lane, int nl) {
  const MmbLayout L = mmb_layout(M.nb, M.ndof, nl);
  const int n = M.ndof;
  const R* mi = ws + L.total;
  for (int e = lane; e < n * n; e += nl) {
    const int i = e / n, j = e - i * n;
    if (i > j) continue;
    R a = R(0), c = R(0);
    for (int k = 0; k < n; k++) { a += mi[i * n + k] * T[k * n + j]; c += mi[j * n + k] * T[k * n + i]; }
    const R v = R(-0.5) * (a + c);
    ws[L.oG + i * n + j] = v; ws[L.oG + j * n + i] = v;
  }
}

}  // namespace nb2
