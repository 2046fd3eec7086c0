// Per-world forward (ABA + semi-implicit Euler) and backward (adjoint) of one contact-free timestep.
//
// What it computes is the reference's World::step (dart/simulation/World.cpp:221-254, 307-333) and
// BackpropSnapshot::backpropState (dart/neural/BackpropSnapshot.cpp:121-194, 382-479) for a world without
// active constraints.  HOW is new:
//   * canonical model (nb2_model.h): joint axes along +z, so S^T I S is one matrix entry and I S one column;
//   * gravity enters as a fictitious base acceleration (same q-ddot as the reference's per-body gravity force);
//   * the backward never materialises the five n x n Jacobians of the reference (BackpropSnapshot.cpp:159-178):
//     with lambda = M^-1 g_v'  (one ABA-style solve reusing the forward's articulated inertias) it evaluates the
//     vector-Jacobian products of inverse dynamics, (d ID/dq)^T lambda and (d ID/dv)^T lambda, by one reverse sweep
//     of RNEA — O(nb) instead of O(nb * n) — which is exactly  posVel^T g, velVel^T g, forceVel^T g.
//
// One world is processed by ONE thread; per-world working storage `scr` is strided by ST (32 on the device:
// [word][lane] interleaving in shared memory => bank-conflict free; 1 in the host build used by tests).
// All control flow depends on the model only, i.e. is warp-uniform.
#pragma once
#include <stddef.h>

#include "nb2_math.cuh"
#include "nb2_model.h"

namespace nb2 {

// per-body record of the forward scratch: V(6) [overwritten by A in pass 3: nothing reads a body's V after its own
// pass-3 step, and its children only need its A], sin/cos(2), U(6), psi, u
#define NB2_FWD_BODY_WORDS 16
struct FwdLayout {
  int oQ, oV, oAct, oBody, oSlot, oFree, total;  // oAct: the raw action row (na <= n words)
};
NB2_HD FwdLayout fwd_layout(int nb, int n, int nslots, int nfree) {
  FwdLayout L;
  L.oQ = 0; L.oV = n; L.oAct = 2 * n; L.oBody = 3 * n;
  L.oSlot = L.oBody + NB2_FWD_BODY_WORDS * nb;
  L.oFree = L.oSlot + 27 * nslots;
  L.total = L.oFree + 18 * nfree;
  return L;
}
struct BwdLayout {
  int oGQ, oGV, oLam, oQb, oVb, oSt, oAct, oBody, oSlot, oFree, total;
};
NB2_HD BwdLayout bwd_layout(int nb, int n, int nslots, int nfree, int slotw = 18) {
  BwdLayout L;
  L.oGQ = 0; L.oGV = n; L.oLam = 2 * n; L.oQb = 3 * n; L.oVb = 4 * n; L.oSt = 5 * n; L.oAct = 7 * n; L.oBody = 8 * n;  // oSt: the step's input state [q; v]; oAct: action row in, dL/daction out
  L.oSlot = L.oBody + 7 * nb;
  L.oFree = L.oSlot + slotw * nslots;
  L.total = L.oFree + 6 * nfree;
  return L;
}

template <class R, int ST> NB2_HD V6<R> ld6(const R* p) {
  V6<R> v; v.a.x = p[0]; v.a.y = p[ST]; v.a.z = p[2 * ST]; v.l.x = p[3 * ST]; v.l.y = p[4 * ST]; v.l.z = p[5 * ST]; return v;
}
template <class R, int ST> NB2_HD void st6(R* p, const V6<R>& v) {
  p[0] = v.a.x; p[ST] = v.a.y; p[2 * ST] = v.a.z; p[3 * ST] = v.l.x; p[4 * ST] = v.l.y; p[5 * ST] = v.l.z;
}
template <class R, int ST> NB2_HD void add6(R* p, const V6<R>& v) {
  p[0] += v.a.x; p[ST] += v.a.y; p[2 * ST] += v.a.z; p[3 * ST] += v.l.x; p[4 * ST] += v.l.y; p[5 * ST] += v.l.z;
}
template <class R, int ST> NB2_HD SI<R> ldSI(const R* p) {
  SI<R> I;
  I.A.xx = p[0]; I.A.yy = p[ST]; I.A.zz = p[2 * ST]; I.A.xy = p[3 * ST]; I.A.xz = p[4 * ST]; I.A.yz = p[5 * ST];
  I.B.m00 = p[6 * ST]; I.B.m01 = p[7 * ST]; I.B.m02 = p[8 * ST]; I.B.m10 = p[9 * ST]; I.B.m11 = p[10 * ST]; I.B.m12 = p[11 * ST];
  I.B.m20 = p[12 * ST]; I.B.m21 = p[13 * ST]; I.B.m22 = p[14 * ST];
  I.C.xx = p[15 * ST]; I.C.yy = p[16 * ST]; I.C.zz = p[17 * ST]; I.C.xy = p[18 * ST]; I.C.xz = p[19 * ST]; I.C.yz = p[20 * ST];
  return I;
}
template <class R, int ST, bool ADD> NB2_HD void stSI(R* p, const SI<R>& I) {
#define NB2_W(k, val) if (ADD) p[(k) * ST] += (val); else p[(k) * ST] = (val);
  NB2_W(0, I.A.xx) NB2_W(1, I.A.yy) NB2_W(2, I.A.zz) NB2_W(3, I.A.xy) NB2_W(4, I.A.xz) NB2_W(5, I.A.yz)
  NB2_W(6, I.B.m00) NB2_W(7, I.B.m01) NB2_W(8, I.B.m02) NB2_W(9, I.B.m10) NB2_W(10, I.B.m11) NB2_W(11, I.B.m12)
  NB2_W(12, I.B.m20) NB2_W(13, I.B.m21) NB2_W(14, I.B.m22)
  NB2_W(15, I.C.xx) NB2_W(16, I.C.yy) NB2_W(17, I.C.zz) NB2_W(18, I.C.xy) NB2_W(19, I.C.xz) NB2_W(20, I.C.yz)
#undef NB2_W
}
// saved-for-backward stream (element type = the arithmetic type R): word k of world w lives at sv[k * B]
// (sv already offset by w) -> coalesced
template <class R> NB2_HD void sv_st6(R* sv, size_t B, int k, const V6<R>& v) {
  sv[(size_t)k * B] = v.a.x; sv[(size_t)(k + 1) * B] = v.a.y; sv[(size_t)(k + 2) * B] = v.a.z;
  sv[(size_t)(k + 3) * B] = v.l.x; sv[(size_t)(k + 4) * B] = v.l.y; sv[(size_t)(k + 5) * B] = v.l.z;
}
template <class R> NB2_HD V6<R> tof(const V6<R>& v) { return v; }
template <class R> NB2_HD V6<R> sv_ld6(const R* sv, size_t B, int k) {
  V6<R> v;
  v.a.x = (R)sv[(size_t)k * B]; v.a.y = (R)sv[(size_t)(k + 1) * B]; v.a.z = (R)sv[(size_t)(k + 2) * B];
  v.l.x = (R)sv[(size_t)(k + 3) * B]; v.l.y = (R)sv[(size_t)(k + 4) * B]; v.l.z = (R)sv[(size_t)(k + 5) * B];
  return v;
}

// Per-body constants (Xtree 12 + inertia 10 words).  `bt` is an optional copy of these tables in shared memory
// ([body][NB2_BT_WORDS]): with several lanes per world the lanes of a warp sit on DIFFERENT bodies, and a constant-bank
// load with a lane-varying index is replayed once per distinct address, while shared memory serves them in one pass.
// bt == nullptr reads the kernel-parameter copy (one thread per world: the index is warp-uniform, constant bank is ideal).
#define NB2_BT_WORDS 22
template <class R> NB2_HD Xf<R> xtree(const Nb2ModelDev<R>& M, const R* bt, int i) {
  Xf<R> T;
  if (bt) {
    const R* t = bt + NB2_BT_WORDS * i;
    T.R_.m00 = t[0]; T.R_.m01 = t[1]; T.R_.m02 = t[2]; T.R_.m10 = t[3]; T.R_.m11 = t[4]; T.R_.m12 = t[5];
    T.R_.m20 = t[6]; T.R_.m21 = t[7]; T.R_.m22 = t[8];
    T.p = mk3<R>(t[9], t[10], t[11]);
    return T;
  }
  T.R_.m00 = M.Xtree[i][0]; T.R_.m01 = M.Xtree[i][1]; T.R_.m02 = M.Xtree[i][2];
  T.R_.m10 = M.Xtree[i][3]; T.R_.m11 = M.Xtree[i][4]; T.R_.m12 = M.Xtree[i][5];
  T.R_.m20 = M.Xtree[i][6]; T.R_.m21 = M.Xtree[i][7]; T.R_.m22 = M.Xtree[i][8];
  T.p = mk3<R>(M.Xtree[i][9], M.Xtree[i][10], M.Xtree[i][11]);
  return T;
}
template <class R> NB2_HD Xf<R> xtree(const Nb2ModelDev<R>& M, int i) { return xtree<R>(M, (const R*)nullptr, i); }
// parent <- child transform of a revolute-z joint: Xtree * Rz(theta)
template <class R> NB2_HD Xf<R> xf_rev(const Nb2ModelDev<R>& M, const R* bt, int i, R s, R c) {
  Xf<R> X = xtree(M, bt, i), T;
  T.R_.m00 = c * X.R_.m00 + s * X.R_.m01; T.R_.m01 = c * X.R_.m01 - s * X.R_.m00; T.R_.m02 = X.R_.m02;
  T.R_.m10 = c * X.R_.m10 + s * X.R_.m11; T.R_.m11 = c * X.R_.m11 - s * X.R_.m10; T.R_.m12 = X.R_.m12;
  T.R_.m20 = c * X.R_.m20 + s * X.R_.m21; T.R_.m21 = c * X.R_.m21 - s * X.R_.m20; T.R_.m22 = X.R_.m22;
  T.p = X.p;
  return T;
}
template <class R> NB2_HD Xf<R> xf_rev(const Nb2ModelDev<R>& M, int i, R s, R c) { return xf_rev<R>(M, (const R*)nullptr, i, s, c); }
template <class R> NB2_HD Xf<R> xf_pris(const Nb2ModelDev<R>& M, const R* bt, int i, R d) {
  Xf<R> T = xtree(M, bt, i);
  T.p.x += T.R_.m02 * d; T.p.y += T.R_.m12 * d; T.p.z += T.R_.m22 * d;
  return T;
}
template <class R> NB2_HD Xf<R> xf_pris(const Nb2ModelDev<R>& M, int i, R d) { return xf_pris<R>(M, (const R*)nullptr, i, d); }
// wi: optional PER-WORLD inertia table (fp64, word-major [10*nb][wiB] like grad_inertia, already offset to the world) that replaces
// the model's: the worlds of a warp are adjacent, so its loads coalesce.  nullptr = the model's table (kernel parameter or `bt`).
template <class R> NB2_HD void inertia_of(const Nb2ModelDev<R>& M, const R* bt, const double* wi, size_t wiB, int i, R* m, V3<R>* h, S3<R>* Ib) {
  if (wi) {
    const double* t = wi + (size_t)(10 * i) * wiB;
    *m = (R)t[0]; *h = mk3<R>((R)t[wiB], (R)t[2 * wiB], (R)t[3 * wiB]);
    Ib->xx = (R)t[4 * wiB]; Ib->yy = (R)t[5 * wiB]; Ib->zz = (R)t[6 * wiB];
    Ib->xy = (R)t[7 * wiB]; Ib->xz = (R)t[8 * wiB]; Ib->yz = (R)t[9 * wiB];
    return;
  }
  if (bt) {
    const R* t = bt + NB2_BT_WORDS * i + 12;
    *m = t[0]; *h = mk3<R>(t[1], t[2], t[3]);
    Ib->xx = t[4]; Ib->yy = t[5]; Ib->zz = t[6]; Ib->xy = t[7]; Ib->xz = t[8]; Ib->yz = t[9];
    return;
  }
  *m = M.inertia[i][0];
  *h = mk3<R>(M.inertia[i][1], M.inertia[i][2], M.inertia[i][3]);
  Ib->xx = M.inertia[i][4]; Ib->yy = M.inertia[i][5]; Ib->zz = M.inertia[i][6];
  Ib->xy = M.inertia[i][7]; Ib->xz = M.inertia[i][8]; Ib->yz = M.inertia[i][9];
}
template <class R, int ST> NB2_HD Xf<R> ldXf(const R* p) {
  Xf<R> T;
  T.R_.m00 = p[0]; T.R_.m01 = p[ST]; T.R_.m02 = p[2 * ST]; T.R_.m10 = p[3 * ST]; T.R_.m11 = p[4 * ST]; T.R_.m12 = p[5 * ST];
  T.R_.m20 = p[6 * ST]; T.R_.m21 = p[7 * ST]; T.R_.m22 = p[8 * ST];
  T.p = mk3<R>(p[9 * ST], p[10 * ST], p[11 * ST]);
  return T;
}
template <class R, int ST> NB2_HD void stXf(R* p, const Xf<R>& T) {
  p[0] = T.R_.m00; p[ST] = T.R_.m01; p[2 * ST] = T.R_.m02; p[3 * ST] = T.R_.m10; p[4 * ST] = T.R_.m11; p[5 * ST] = T.R_.m12;
  p[6 * ST] = T.R_.m20; p[7 * ST] = T.R_.m21; p[8 * ST] = T.R_.m22; p[9 * ST] = T.p.x; p[10 * ST] = T.p.y; p[11 * ST] = T.p.z;
}
// transform of body i during the sweeps that follow the kinematics pass (forward scratch layout)
template <class R, int ST> NB2_HD Xf<R> body_xf_fwd(const Nb2ModelDev<R>& M, const R* bt, int i, const R* scr, const FwdLayout& L) {
  const int jt = M.jtype[i];
  if (jt == NB2_JT_REV) { const R* b = scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * i + 6) * ST; return xf_rev(M, bt, i, b[0], b[ST]); }
  if (jt == NB2_JT_PRIS) return xf_pris(M, bt, i, scr[(size_t)(L.oQ + M.dof_off[i]) * ST]);
  return ldXf<R, ST>(scr + (size_t)(L.oFree + 18 * M.free_idx[i]) * ST);
}
// S * x for 1-dof joints / eta = ad(V, S v)
template <class R> NB2_HD V6<R> S_times(int jt, R x) {
  V6<R> s = zero6<R>();
  if (jt == NB2_JT_REV) s.a.z = x; else s.l.z = x;
  return s;
}
template <class R> NB2_HD R S_dot(int jt, const V6<R>& f) { return (jt == NB2_JT_REV) ? f.a.z : f.l.z; }

// generalized force on dof d: World.cpp:2061-2086 scatters the action through the action map, unmapped dofs get 0
template <class R, int ST> NB2_HD R tau_of(const Nb2ModelDev<R>& M, const R* scr, int oAct, int d) {
  const int a = M.act_of_dof[d];
  return (a >= 0) ? scr[(size_t)(oAct + a) * ST] : R(0);
}

// =====================================================================================================
// forward: state=[q;v] (fp32 row), action (fp32 row) -> next state row; optionally streams intermediates to `sv`
// =====================================================================================================
template <class R, int ST>
NB2_HD void fwd_pass1(const Nb2ModelDev<R>& M, R* scr, int lo, int hi, const R* bt = nullptr) {
  const int nb = M.nb, n = M.ndof;
  const FwdLayout L = fwd_layout(nb, n, M.nslots, M.nfree);
  const R dt = M.dt;
  (void)nb; (void)n; (void)dt;
  // ---------------- pass 1, root -> leaf: joint transforms and spatial velocities (Frame.cpp:144-160)
  for (int i = lo; i < hi; i++) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i];
    R* bs = scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * i) * ST;
    V6<R> Vp = (p >= 0) ? ld6<R, ST>(scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * p) * ST) : zero6<R>();
    V6<R> V;
    if (jt == NB2_JT_REV) {
      R s, c; nb2_sincos(scr[(size_t)(L.oQ + o) * ST], &s, &c);
      bs[6 * ST] = s; bs[7 * ST] = c;
      V = AdInvT(xf_rev(M, bt, i, s, c), Vp);
      V.a.z += scr[(size_t)(L.oV + o) * ST];
    } else if (jt == NB2_JT_PRIS) {
      V = AdInvT(xf_pris(M, bt, i, scr[(size_t)(L.oQ + o) * ST]), Vp);
      V.l.z += scr[(size_t)(L.oV + o) * ST];
    } else {  // FREE (FreeJoint.cpp:74-81, 1027-1061)
      const R* q = scr + (size_t)(L.oQ + o) * ST;
      const R* v = scr + (size_t)(L.oV + o) * ST;
      Xf<R> X = xtree(M, bt, i), T;
      M3<R> Rq = expmap(mk3<R>(q[0], q[ST], q[2 * ST]));
      T.R_ = mul(X.R_, Rq);
      T.p = mul(X.R_, mk3<R>(q[3 * ST], q[4 * ST], q[5 * ST])) + X.p;
      stXf<R, ST>(scr + (size_t)(L.oFree + 18 * M.free_idx[i]) * ST, T);
      V = AdInvT(T, Vp) + ld6<R, ST>(v);
    }
    st6<R, ST>(bs, V);
  }

}

template <class R, int ST>
NB2_HD void fwd_pass2(const Nb2ModelDev<R>& M, R* scr, R* sv, size_t B, bool save, int lo, int hi, const R* bt = nullptr, R* iinv_out = nullptr,
                      const double* wi = nullptr, size_t wiB = 0) {
  const int nb = M.nb, n = M.ndof;
  const FwdLayout L = fwd_layout(nb, n, M.nslots, M.nfree);
  const R dt = M.dt;
  (void)nb; (void)n; (void)dt;
  // ---------------- pass 2, leaf -> root: articulated inertia, bias force, total joint force
  // (BodyNode.cpp:2046-2114, GenericJoint.hpp:2168-2185, 2276-2301, 2395-2421, 2554-2571)
  SI<R> hI = zeroSI<R>();
  V6<R> hp = zero6<R>();
  bool hvalid = false;
  for (int i = hi - 1; i >= lo; i--) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i], fl = M.flags[i];
    R* bs = scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * i) * ST;
    R m; V3<R> h; S3<R> Ib; inertia_of(M, bt, wi, wiB, i, &m, &h, &Ib);
    const V6<R> V = ld6<R, ST>(bs);
    SI<R> IA = rigidSI(m, h, Ib);
    V6<R> pA = crf(V, mulG(m, h, Ib, V));
    if (hvalid) { IA = IA + hI; pA = pA + hp; }
    if (fl & NB2_F_HAS_SLOT) {
      for (int k = 0; k < M.slot_count[i]; k++) {  // contributions of the children that could not hand off in registers
        const R* sl = scr + (size_t)(L.oSlot + 27 * (M.slot_self[i] + k)) * ST;
        IA = IA + ldSI<R, ST>(sl);
        pA = pA + ld6<R, ST>(sl + 21 * ST);
      }
    }
    SI<R> Pi; V6<R> beta;
    if (jt != NB2_JT_FREE) {
      const R vq = scr[(size_t)(L.oV + o) * ST];
      V6<R> U, eta;
      R D;
      if (jt == NB2_JT_REV) {
        U.a = mk3<R>(IA.A.xz, IA.A.yz, IA.A.zz); U.l = mk3<R>(IA.B.m20, IA.B.m21, IA.B.m22); D = IA.A.zz;
        eta.a = mk3<R>(V.a.y * vq, -V.a.x * vq, R(0)); eta.l = mk3<R>(V.l.y * vq, -V.l.x * vq, R(0));
      } else {
        U.a = mk3<R>(IA.B.m02, IA.B.m12, IA.B.m22); U.l = mk3<R>(IA.C.xz, IA.C.yz, IA.C.zz); D = IA.C.zz;
        eta.a = zero3<R>(); eta.l = mk3<R>(V.a.y * vq, -V.a.x * vq, R(0));
      }
      const R psi = nb2_rcp(D);
      const R qv = scr[(size_t)(L.oQ + o) * ST];
      const R u = tau_of<R, ST>(M, scr, L.oAct, o) - M.spring[o] * (qv - M.rest[o] + vq * dt) - M.damping[o] * vq
                  - (dot(U, eta) + S_dot(jt, pA));
      st6<R, ST>(bs + 8 * ST, U);
      bs[14 * ST] = psi; bs[15 * ST] = u;
      if (p >= 0) {
        const R k = -psi;
        Pi = IA;
        Pi.A.xx += k * U.a.x * U.a.x; Pi.A.yy += k * U.a.y * U.a.y; Pi.A.zz += k * U.a.z * U.a.z;
        Pi.A.xy += k * U.a.x * U.a.y; Pi.A.xz += k * U.a.x * U.a.z; Pi.A.yz += k * U.a.y * U.a.z;
        Pi.C.xx += k * U.l.x * U.l.x; Pi.C.yy += k * U.l.y * U.l.y; Pi.C.zz += k * U.l.z * U.l.z;
        Pi.C.xy += k * U.l.x * U.l.y; Pi.C.xz += k * U.l.x * U.l.z; Pi.C.yz += k * U.l.y * U.l.z;
        Pi.B.m00 += k * U.a.x * U.l.x; Pi.B.m01 += k * U.a.x * U.l.y; Pi.B.m02 += k * U.a.x * U.l.z;
        Pi.B.m10 += k * U.a.y * U.l.x; Pi.B.m11 += k * U.a.y * U.l.y; Pi.B.m12 += k * U.a.y * U.l.z;
        Pi.B.m20 += k * U.a.z * U.l.x; Pi.B.m21 += k * U.a.z * U.l.y; Pi.B.m22 += k * U.a.z * U.l.z;
        beta = pA + mul(IA, eta) + U * (psi * u);
      }
    } else {
      const R* q = scr + (size_t)(L.oQ + o) * ST;
      const R* v = scr + (size_t)(L.oV + o) * ST;
      R t[6];
#pragma unroll
      for (int k = 0; k < 6; k++) t[k] = tau_of<R, ST>(M, scr, L.oAct, o + k);
      const V6<R> Vj = ld6<R, ST>(v);
      const V6<R> eta = ad(V, Vj);
      const V6<R> bf = mul(IA, eta) + pA;
      V6<R> u;
      u.a.x = t[0] - M.spring[o] * (q[0] - M.rest[o] + Vj.a.x * dt) - M.damping[o] * Vj.a.x - bf.a.x;
      u.a.y = t[1] - M.spring[o + 1] * (q[ST] - M.rest[o + 1] + Vj.a.y * dt) - M.damping[o + 1] * Vj.a.y - bf.a.y;
      u.a.z = t[2] - M.spring[o + 2] * (q[2 * ST] - M.rest[o + 2] + Vj.a.z * dt) - M.damping[o + 2] * Vj.a.z - bf.a.z;
      u.l.x = t[3] - M.spring[o + 3] * (q[3 * ST] - M.rest[o + 3] + Vj.l.x * dt) - M.damping[o + 3] * Vj.l.x - bf.l.x;
      u.l.y = t[4] - M.spring[o + 4] * (q[4 * ST] - M.rest[o + 4] + Vj.l.y * dt) - M.damping[o + 4] * Vj.l.y - bf.l.y;
      u.l.z = t[5] - M.spring[o + 5] * (q[5 * ST] - M.rest[o + 5] + Vj.l.z * dt) - M.damping[o + 5] * Vj.l.z - bf.l.z;
      const SI<R> Iinv = spd6_inverse(IA);
      const V6<R> y = mul(Iinv, u);
      st6<R, ST>(scr + (size_t)(L.oFree + 18 * M.free_idx[i] + 12) * ST, y);
      if (iinv_out) stSI<R, 1, false>(iinv_out + 21 * M.free_idx[i], Iinv);  // fused contact kernel: the contact stage needs it (per-world array, stride 1)
      if (save) {
        const int k0 = nb * 21 + M.free_idx[i] * 33;
        R* s = sv + (size_t)k0 * B;
        s[0] = (R)Iinv.A.xx; s[B] = (R)Iinv.A.yy; s[2 * B] = (R)Iinv.A.zz; s[3 * B] = (R)Iinv.A.xy; s[4 * B] = (R)Iinv.A.xz; s[5 * B] = (R)Iinv.A.yz;
        s[6 * B] = (R)Iinv.B.m00; s[7 * B] = (R)Iinv.B.m01; s[8 * B] = (R)Iinv.B.m02; s[9 * B] = (R)Iinv.B.m10; s[10 * B] = (R)Iinv.B.m11; s[11 * B] = (R)Iinv.B.m12;
        s[12 * B] = (R)Iinv.B.m20; s[13 * B] = (R)Iinv.B.m21; s[14 * B] = (R)Iinv.B.m22;
        s[15 * B] = (R)Iinv.C.xx; s[16 * B] = (R)Iinv.C.yy; s[17 * B] = (R)Iinv.C.zz; s[18 * B] = (R)Iinv.C.xy; s[19 * B] = (R)Iinv.C.xz; s[20 * B] = (R)Iinv.C.yz;
      }
      if (p >= 0) { Pi = zeroSI<R>(); beta = bf + u; }  // a 6-dof joint transmits only its own joint force
    }
    hvalid = false;
    if (p >= 0) {
      const Xf<R> T = body_xf_fwd<R, ST>(M, bt, i, scr, L);
      const SI<R> Ic = xform_inertia(T, Pi);
      const V6<R> pc = dAdInvT(T, beta);
      if (fl & NB2_F_HANDOFF) { hI = Ic; hp = pc; hvalid = true; }
      else {
        R* sl = scr + (size_t)(L.oSlot + 27 * M.slot_parent[i]) * ST;  // this child's own slot: plain store
        stSI<R, ST, false>(sl, Ic); st6<R, ST>(sl + 21 * ST, pc);
      }
    }
  }

}

template <class R, int ST>
NB2_HD void fwd_pass3(const Nb2ModelDev<R>& M, R* scr, R* sv, size_t B, bool save, int lo, int hi, const R* bt = nullptr) {
  const int nb = M.nb, n = M.ndof;
  const FwdLayout L = fwd_layout(nb, n, M.nslots, M.nfree);
  const R dt = M.dt;
  (void)nb; (void)n; (void)dt;
  // ---------------- pass 3, root -> leaf: accelerations (BodyNode.cpp:2159-2185, GenericJoint.hpp:2656-2676),
  // then integrate: v+ = v + dt qdd ; q+ = q (+) dt v  with the PRE-step velocity (World.cpp:307-322)
  V6<R> A0; A0.a = zero3<R>(); A0.l = mk3<R>(-M.gravity[0], -M.gravity[1], -M.gravity[2]);
  for (int i = lo; i < hi; i++) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i];
    R* bs = scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * i) * ST;
    const Xf<R> T = body_xf_fwd<R, ST>(M, bt, i, scr, L);
    const V6<R> Ap = AdInvT(T, (p >= 0) ? ld6<R, ST>(scr + (size_t)(L.oBody + NB2_FWD_BODY_WORDS * p) * ST) : A0);  // the parent's V slot holds its A by now
    const V6<R> V = ld6<R, ST>(bs);
    V6<R> A;
    if (jt != NB2_JT_FREE) {
      const R vq = scr[(size_t)(L.oV + o) * ST], qv = scr[(size_t)(L.oQ + o) * ST];
      const V6<R> U = ld6<R, ST>(bs + 8 * ST);
      const R psi = bs[14 * ST], u = bs[15 * ST];
      const R qdd = psi * (u - dot(U, Ap));
      A = Ap;
      if (jt == NB2_JT_REV) { A.a.z += qdd; A.a.x += V.a.y * vq; A.a.y -= V.a.x * vq; A.l.x += V.l.y * vq; A.l.y -= V.l.x * vq; }
      else { A.l.z += qdd; A.l.x += V.a.y * vq; A.l.y -= V.a.x * vq; }
      scr[(size_t)(L.oQ + o) * ST] = qv + vq * dt;   // q+, v+ replace q, v in the scratch (nothing reads this body's q, v again);
      scr[(size_t)(L.oV + o) * ST] = vq + qdd * dt;  // fwd_store writes them out coalesced
      if (save) {
        R* s = sv + (size_t)(i * 21) * B;
        sv_st6(s, B, 0, tof(V)); sv_st6(s, B, 6, tof(A)); sv_st6(s, B, 12, tof(U));
        s[18 * B] = (R)psi;
        s[19 * B] = (jt == NB2_JT_REV) ? (R)bs[6 * ST] : R(0); s[20 * B] = (jt == NB2_JT_REV) ? (R)bs[7 * ST] : R(0);  // sin, cos (revolute only)
        sv[(size_t)(nb * 21 + M.nfree * 33 + o) * B] = qdd;
      }
    } else {
      const R* q = scr + (size_t)(L.oQ + o) * ST;
      const R* fr = scr + (size_t)(L.oFree + 18 * M.free_idx[i]) * ST;
      const V6<R> Vj = ld6<R, ST>(scr + (size_t)(L.oV + o) * ST);
      const V6<R> y = ld6<R, ST>(fr + 12 * ST);
      const V6<R> qdd = y - Ap;
      A = y + ad(V, Vj);
      // FreeJoint::integratePositionsExplicit, identity-Jacobian branch (FreeJoint.cpp:922-929)
      const V3<R> phi = mk3<R>(q[0], q[ST], q[2 * ST]);
      const M3<R> Rq = expmap(phi);
      const V3<R> phin = logmap(mul(Rq, expmap(Vj.a * dt)));
      const V3<R> pn = mk3<R>(q[3 * ST], q[4 * ST], q[5 * ST]) + mul(Rq, Vj.l * dt);
      R* qo = scr + (size_t)(L.oQ + o) * ST;
      R* vo = scr + (size_t)(L.oV + o) * ST;
      qo[0] = phin.x; qo[ST] = phin.y; qo[2 * ST] = phin.z; qo[3 * ST] = pn.x; qo[4 * ST] = pn.y; qo[5 * ST] = pn.z;
      vo[0] = Vj.a.x + qdd.a.x * dt; vo[ST] = Vj.a.y + qdd.a.y * dt; vo[2 * ST] = Vj.a.z + qdd.a.z * dt;
      vo[3 * ST] = Vj.l.x + qdd.l.x * dt; vo[4 * ST] = Vj.l.y + qdd.l.y * dt; vo[5 * ST] = Vj.l.z + qdd.l.z * dt;
      if (save) {
        R* s = sv + (size_t)(i * 21) * B;
        sv_st6(s, B, 0, tof(V)); sv_st6(s, B, 6, tof(A));
        for (int k = 12; k < 21; k++) s[(size_t)k * B] = R(0);
        R* sf = sv + (size_t)(nb * 21 + M.free_idx[i] * 33 + 21) * B;
        for (int k = 0; k < 12; k++) sf[(size_t)k * B] = fr[(size_t)k * ST];
        R* sq = sv + (size_t)(nb * 21 + M.nfree * 33 + o) * B;
        sq[0] = qdd.a.x; sq[B] = qdd.a.y; sq[2 * B] = qdd.a.z; sq[3 * B] = qdd.l.x; sq[4 * B] = qdd.l.y; sq[5 * B] = qdd.l.z;
      }
    }
    st6<R, ST>(bs, A);  // A replaces V (see NB2_FWD_BODY_WORDS)
  }
}

// ---- group I/O.  A GROUP is the set of worlds one warp works on (32/lanes of them on the device, one in the host
// emulation and in the single-thread paths); its worlds are consecutive, so their state / action / output rows form
// one contiguous block of global memory that the group's threads copy cooperatively (fully coalesced, every byte
// touched once — the entry points may hand in mapped host memory).  scr0 = scratch of the group's first world.
// Copy loops of the group I/O: 16-byte vector accesses when the block is aligned (it is whenever the batch pointers are,
// since a group starts at a multiple of 4 worlds), several independent loads in flight per thread (the source may be
// host memory behind PCIe), index -> (world slot, dof) by multiply-high with the precomputed reciprocal.
#define NB2_IO_UNROLL 4
struct alignas(16) F4 { float x, y, z, w; };
NB2_HD unsigned fast_div(unsigned idx, unsigned magic) {
#ifdef __CUDA_ARCH__
  return __umulhi(idx, magic);
#else
  return (unsigned)(((unsigned long long)idx * magic) >> 32);
#endif
}
template <class F> NB2_HD void group_read(const float* src, int tot, int tid, int nthr, const F& f) {
  if ((((size_t)src) & 15) == 0) {
    const F4* s4 = reinterpret_cast<const F4*>(src);
    const int tot4 = tot >> 2;
    for (int base = tid; base < tot4; base += nthr * NB2_IO_UNROLL) {
      F4 v[NB2_IO_UNROLL];
#pragma unroll
      for (int u = 0; u < NB2_IO_UNROLL; u++) { const int j = base + u * nthr; if (j < tot4) v[u] = s4[j]; }
#pragma unroll
      for (int u = 0; u < NB2_IO_UNROLL; u++) {
        const int j = base + u * nthr;
        if (j < tot4) { f(4 * j, v[u].x); f(4 * j + 1, v[u].y); f(4 * j + 2, v[u].z); f(4 * j + 3, v[u].w); }
      }
    }
    for (int idx = 4 * tot4 + tid; idx < tot; idx += nthr) f(idx, src[idx]);
  } else {
    for (int base = tid; base < tot; base += nthr * NB2_IO_UNROLL) {
      float v[NB2_IO_UNROLL];
#pragma unroll
      for (int u = 0; u < NB2_IO_UNROLL; u++) { const int idx = base + u * nthr; v[u] = (idx < tot) ? src[idx] : 0.f; }
#pragma unroll
      for (int u = 0; u < NB2_IO_UNROLL; u++) { const int idx = base + u * nthr; if (idx < tot) f(idx, v[u]); }
    }
  }
}
template <class F> NB2_HD void group_write(float* dst, int tot, int tid, int nthr, const F& f) {
  if ((((size_t)dst) & 15) == 0) {
    F4* d4 = reinterpret_cast<F4*>(dst);
    const int tot4 = tot >> 2;
    for (int j = tid; j < tot4; j += nthr) { F4 v; v.x = f(4 * j); v.y = f(4 * j + 1); v.z = f(4 * j + 2); v.w = f(4 * j + 3); d4[j] = v; }
    for (int idx = 4 * tot4 + tid; idx < tot; idx += nthr) dst[idx] = f(idx);
  } else {
    for (int idx = tid; idx < tot; idx += nthr) dst[idx] = f(idx);
  }
}

template <class R, int ST> struct WordScatter {  // element d of row `slot` of a [*, width] block -> scratch word (base + d) (+ device copy)
  R* scr0; int width, base; unsigned magic; float* copy;
  NB2_HD void operator()(int idx, float v) const {
    const int slot = (int)fast_div((unsigned)idx, magic), d = idx - slot * width;
    scr0[(size_t)(base + d) * ST + slot] = (R)v;
    if (copy) copy[idx] = v;
  }
};
template <class R, int ST> struct WordGather {
  const R* scr0; int width, base; unsigned magic;
  NB2_HD float operator()(int idx) const {
    const int slot = (int)fast_div((unsigned)idx, magic), d = idx - slot * width;
    return (float)scr0[(size_t)(base + d) * ST + slot];
  }
};

// ---- group I/O.  A GROUP is the set of worlds one warp works on (32/lanes of them on the device, a few in the host
// emulation, one in the single-thread paths); its worlds are consecutive, so their state / action / output rows form
// one contiguous block of global memory that the group's threads copy cooperatively (fully coalesced, every byte
// touched once — the entry points may hand in mapped host memory).  scr0 = scratch of the group's first world.
// The copies are pure word moves (q, v and the raw action row are adjacent in the scratch); the action map and the
// gradient clipping are applied per body inside the sweeps, where the model tables are indexed (almost) uniformly.
template <class R, int ST>
NB2_HD void fwd_load(const Nb2ModelDev<R>& M, R* scr0, const float* st0, const float* act0, int nworlds, int tid, int nthr,
                     float* st_copy0 = nullptr, float* act_copy0 = nullptr) {
  const int n2 = 2 * M.ndof, na = M.na;
  const FwdLayout L = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  WordScatter<R, ST> ss{scr0, n2, L.oQ, M.magic_n2, st_copy0};  // oV = oQ + n
  group_read(st0, nworlds * n2, tid, nthr, ss);
  WordScatter<R, ST> as{scr0, na, L.oAct, M.magic_na, act_copy0};
  group_read(act0, nworlds * na, tid, nthr, as);
}
template <class R, int ST>
NB2_HD void fwd_store(const Nb2ModelDev<R>& M, const R* scr0, float* out0, int nworlds, int tid, int nthr) {
  const int n2 = 2 * M.ndof;
  const FwdLayout L = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  WordGather<R, ST> sg{scr0, n2, L.oQ, M.magic_n2};
  group_write(out0, nworlds * n2, tid, nthr, sg);
}

// The sweeps are cut into STAGES so that M.lanes threads can cooperate on one world: lane 0 owns the TRUNK (an
// ancestor-closed set of bodies), every lane owns some LIMB subtrees (modelspec._partition_tree).  A warp barrier is
// needed only where data crosses threads (NB2_FWD_SYNC_MASK bit = "barrier after this stage"):
//   0 group load of q, v, tau (fwd_load)                     | barrier
//   1 kinematics of the trunk           (lane 0, root->leaf) | barrier
//   2 kinematics of the limbs           (every lane)
//   3 articulated inertias of the limbs (every lane, leaf->root) | barrier
//   4 articulated inertias of the trunk (lane 0)
//   5 accelerations + integration, trunk (lane 0)            | barrier
//   6 accelerations + integration, limbs (every lane)        | barrier
//   7 group store of q+, v+ (fwd_store)
// With lanes == 1 everything is trunk.  Each pass body is instantiated once (the stage index is a run-time value).
#define NB2_FWD_STAGES 8
#define NB2_FWD_SYNC_MASK 0x6Bu       /* after stages 0, 1, 3, 5, 6 */
#define NB2_FWD_SYNC_MASK_1LANE 0x41u /* lanes == 1: only the group load / store exchange data between threads */
template <class R, int ST>
NB2_HD void world_forward_stage(const Nb2ModelDev<R>& M, R* scr, R* sv, size_t B, bool save, int lane, int stage, const R* bt = nullptr, R* iinv_out = nullptr,
                                const double* wi = nullptr, size_t wiB = 0) {
  const int pass = (stage + 1) >> 1;                          // stages 1..6 -> passes 1, 2, 3
  const bool trunk = (stage == 1) | (stage == 4) | (stage == 5);
  if (trunk && lane != 0) return;
  const int nr = trunk ? M.trunk_n : M.limb_n[lane];
  for (int rr = 0; rr < nr; rr++) {
    const int r = (pass == 2) ? nr - 1 - rr : rr;
    const int lo = trunk ? M.trunk_lo[r] : M.limb_lo[lane][r], hi = trunk ? M.trunk_hi[r] : M.limb_hi[lane][r];
    if (pass == 1) fwd_pass1<R, ST>(M, scr, lo, hi, bt);
    else if (pass == 2) fwd_pass2<R, ST>(M, scr, sv, B, save, lo, hi, bt, iinv_out, wi, wiB);
    else fwd_pass3<R, ST>(M, scr, sv, B, save, lo, hi, bt);
  }
}

// what the contact-stage adjoint (nb2_cw.cuh, contact_backward) hands to the reverse sweep B3 / the assembly: per-world arrays
// (stride ST like the scratch; the fused contact kernels use ST = 1).  inj is COMPACT: one record per collision body
// (inj_of_body[i] = record index or -1), Uw_bar(6) Up_bar(6) G(6) H(6).
template <class T, int ST> struct SPd { T* p; NB2_HD T& operator[](int i) const { return p[(size_t)i * ST]; } NB2_HD SPd operator+(int k) const { SPd r; r.p = p + (size_t)k * ST; return r; } };
template <int ST>
struct BwdContactData {
  SPd<double, ST> Aacc, Uplus, aeff, vplus, inj, JcTmu;
  const int16_t* inj_of_body;
  int active; int error;
  // restitution (nb2_cw.cuh, contact_backward): bounce != 0 asks for a SECOND reverse sweep B3 (pass2 = 1) with the field of -nu_e, the
  // unconstrained accelerations of the saved stream and the v* injections; it ADDS to qbar / vbar and leaves JcTmu / the inertia gradient alone
  int bounce = 0, pass2 = 0;
};

// Products rounded on their own (never contracted into an FMA): which product of a*b + c*d the compiler fuses depends on the
// surrounding code, and the inertia gradient must have the same bits in the shared-table and the per-world-inertia
// instantiations of the reverse sweep.
NB2_HD float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
NB2_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
template <class R> NB2_HD V3<R> cross_rn(const V3<R>& a, const V3<R>& b) {
  return mk3<R>(mul_rn(a.y, b.z) - mul_rn(a.z, b.y), mul_rn(a.z, b.x) - mul_rn(a.x, b.z), mul_rn(a.x, b.y) - mul_rn(a.y, b.x));
}
// d(Y^T G X)/d(m, h(3), Ibar(xx,yy,zz,xy,xz,yz)) for G X = [Ibar w + h x v ; m v - h x w]
template <class R> NB2_HD void inertia_param_form(const V6<R>& Y, const V6<R>& X, R* t) {
  t[0] = mul_rn(Y.l.x, X.l.x) + mul_rn(Y.l.y, X.l.y) + mul_rn(Y.l.z, X.l.z);
  const V3<R> dh = cross_rn(X.l, Y.a) + cross_rn(Y.l, X.a);
  t[1] = dh.x; t[2] = dh.y; t[3] = dh.z;
  t[4] = mul_rn(Y.a.x, X.a.x); t[5] = mul_rn(Y.a.y, X.a.y); t[6] = mul_rn(Y.a.z, X.a.z);
  t[7] = mul_rn(Y.a.x, X.a.y) + mul_rn(Y.a.y, X.a.x); t[8] = mul_rn(Y.a.x, X.a.z) + mul_rn(Y.a.z, X.a.x);
  t[9] = mul_rn(Y.a.y, X.a.z) + mul_rn(Y.a.z, X.a.y);
}

// =====================================================================================================
// backward: g_next = dL/d[q+;v+]  ->  g_state = dL/d[q;v], g_action = dL/d action
// =====================================================================================================
template <class R, int ST, bool CONTACT>
NB2_HD void bwd_B1(const Nb2ModelDev<R>& M, R* scr, const float* st, const R* sv, size_t B, int lo, int hi, const R* bt = nullptr) {
  const int nb = M.nb, n = M.ndof;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(nb, n, M.nslots, M.nfree, SLOTW);
  const R dt = M.dt;
  const int kFree = nb * 21, kQdd = nb * 21 + M.nfree * 33;
  (void)n; (void)dt; (void)kFree; (void)kQdd;
  // ---------------- B1, leaf -> root: bias pass of lambda = M^-1 g_v'  (impulse-ABA form,
  // BodyNode.cpp:2117-2138, GenericJoint.hpp:2482-2498, 2607-2613) reusing the forward's U, psi
  V6<R> hp = zero6<R>();
  bool hvalid = false;
  for (int i = hi - 1; i >= lo; i--) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i], fl = M.flags[i];
    const R* s = sv + (size_t)(i * 21) * B;
    V6<R> pI = hvalid ? hp : zero6<R>();
    if (fl & NB2_F_HAS_SLOT)
      for (int k = 0; k < M.slot_count[i]; k++) pI = pI + ld6<R, ST>(scr + (size_t)(L.oSlot + SLOTW * (M.slot_self[i] + k)) * ST);
    V6<R> beta;
    if (jt != NB2_JT_FREE) {
      const R up = scr[(size_t)(L.oGV + o) * ST] - S_dot(jt, pI);
      scr[(size_t)(L.oBody + 7 * i) * ST] = up;
      if (p >= 0) beta = pI + sv_ld6<R>(s, B, 12) * ((R)s[18 * B] * up);
    } else {
      const V6<R> up = ld6<R, ST>(scr + (size_t)(L.oGV + o) * ST) - pI;
      st6<R, ST>(scr + (size_t)(L.oFree + 6 * M.free_idx[i]) * ST, up);
      if (p >= 0) beta = pI + up;
    }
    hvalid = false;
    if (p >= 0) {
      Xf<R> T;
      if (jt == NB2_JT_REV) T = xf_rev(M, bt, i, (R)s[19 * B], (R)s[20 * B]);
      else if (jt == NB2_JT_PRIS) T = xf_pris(M, bt, i, scr[(size_t)(L.oSt + o) * ST]);
      else { R t12[12]; for (int k = 0; k < 12; k++) t12[k] = (R)sv[(size_t)(kFree + M.free_idx[i] * 33 + 21 + k) * B]; T = ldXf<R, 1>(t12); }
      const V6<R> pc = dAdInvT(T, beta);
      if (fl & NB2_F_HANDOFF) { hp = pc; hvalid = true; }
      else {
        R* sl = scr + (size_t)(L.oSlot + SLOTW * M.slot_parent[i]) * ST;
        st6<R, ST>(sl, pc);
      }
    }
  }
}

template <class R, int ST, bool CONTACT>
NB2_HD void bwd_B2(const Nb2ModelDev<R>& M, R* scr, const float* st, const R* sv, size_t B, int lo, int hi, const R* bt = nullptr) {
  const int nb = M.nb, n = M.ndof;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(nb, n, M.nslots, M.nfree, SLOTW);
  const R dt = M.dt;
  const int kFree = nb * 21, kQdd = nb * 21 + M.nfree * 33;
  (void)n; (void)dt; (void)kFree; (void)kQdd;
  // ---------------- B2, root -> leaf: lambda and the spatial "velocities" W it induces
  // (BodyNode.cpp:2188-2215, GenericJoint.hpp:2713-2725)
  for (int i = lo; i < hi; i++) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i];
    const R* s = sv + (size_t)(i * 21) * B;
    R* bs = scr + (size_t)(L.oBody + 7 * i) * ST;
    V6<R> W;
    if (jt != NB2_JT_FREE) {
      Xf<R> T = (jt == NB2_JT_REV) ? xf_rev(M, bt, i, (R)s[19 * B], (R)s[20 * B]) : xf_pris(M, bt, i, scr[(size_t)(L.oSt + o) * ST]);
      W = (p >= 0) ? AdInvT(T, ld6<R, ST>(scr + (size_t)(L.oBody + 7 * p + 1) * ST)) : zero6<R>();
      const R lam = (R)s[18 * B] * (bs[0] - dot(sv_ld6<R>(s, B, 12), W));
      scr[(size_t)(L.oLam + o) * ST] = lam;
      if (jt == NB2_JT_REV) W.a.z += lam; else W.l.z += lam;
    } else {
      const R* sf = sv + (size_t)(kFree + M.free_idx[i] * 33) * B;
      R t12[12]; for (int k = 0; k < 12; k++) t12[k] = (R)sf[(size_t)(21 + k) * B];
      const Xf<R> T = ldXf<R, 1>(t12);
      const V6<R> Wp = (p >= 0) ? AdInvT(T, ld6<R, ST>(scr + (size_t)(L.oBody + 7 * p + 1) * ST)) : zero6<R>();
      R i21[21]; for (int k = 0; k < 21; k++) i21[k] = (R)sf[(size_t)k * B];
      const SI<R> Iinv = ldSI<R, 1>(i21);
      W = mul(Iinv, ld6<R, ST>(scr + (size_t)(L.oFree + 6 * M.free_idx[i]) * ST));
      st6<R, ST>(scr + (size_t)(L.oLam + o) * ST, W - Wp);
    }
    st6<R, ST>(bs + ST, W);
  }
}

template <class R, int ST, bool CONTACT>
NB2_HD void bwd_B3(const Nb2ModelDev<R>& M, R* scr, const float* st, const R* sv, size_t B, const BwdContactData<ST>& cd, int lo, int hi,
                   float* gI = nullptr, const R* bt = nullptr, size_t gIB = 0, const double* wi = nullptr, size_t wiB = 0, double* gIa = nullptr) {
  const int nb = M.nb, n = M.ndof;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(nb, n, M.nslots, M.nfree, SLOTW);
  const R dt = M.dt;
  const int kFree = nb * 21, kQdd = nb * 21 + M.nfree * 33;
  (void)n; (void)dt; (void)kFree; (void)kQdd;
  // ---------------- B3, leaf -> root: reverse sweep of RNEA, seeded with lambda on the joint forces.
  //   forward RNEA:  V_i = X^-1 V_p + S v ;  A_i = X^-1 A_p + S a + ad(V_i, S v) ;  F_i = G A_i + V_i x* G V_i ;
  //                  f_i = F_i + sum_c X*_c f_c ; tau_i = S^T f_i
  //   adjoints:      fbar_i = W_i (from B2) ;  Abar_i = G W_i + sum_c X*_c Abar_c ;
  //                  Vbar_i = -W x* (G V) + G ad(W, V) + (S v) x* Abar_i + sum_c X*_c Vbar_c
  //                  vbar_i = S^T (Vbar_i - V_i x* Abar_i)
  //                  c_i    = -( (X^-1 A_p) x* Abar_i + (X^-1 V_p) x* Vbar_i + (X^-1 W_p) x* f_i ) ; qbar_i = B_i(q)^T c_i
  V6<R> hA = zero6<R>(), hV = zero6<R>(), hf = zero6<R>();
  V6<R> hUw = zero6<R>(), hUp = zero6<R>(), hG = zero6<R>(), hH = zero6<R>();
  bool hvalid = false;
  for (int i = hi - 1; i >= lo; i--) {
    const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i], fl = M.flags[i];
    const R* s = sv + (size_t)(i * 21) * B;
    R m; V3<R> h; S3<R> Ib; inertia_of(M, bt, wi, wiB, i, &m, &h, &Ib);
    const V6<R> V = sv_ld6<R>(s, B, 0);
    V6<R> A = sv_ld6<R>(s, B, 6);
    if (CONTACT && cd.active && !cd.pass2) { const auto a6 = cd.Aacc + 6 * i; A.a = mk3<R>((R)a6[0], (R)a6[1], (R)a6[2]); A.l = mk3<R>((R)a6[3], (R)a6[4], (R)a6[5]); }
    const V6<R> W = ld6<R, ST>(scr + (size_t)(L.oBody + 7 * i + 1) * ST);
    const V6<R> GV = mulG(m, h, Ib, V);
    V6<R> f = mulG(m, h, Ib, A) + crf(V, GV);
    if (gI || gIa) {
      // dL/d(inertia parameters of body i) = -dt * W . d(G A + V x* G V) = -dt * [ t(W, A) - t(ad(V, W), V) ] with
      // t(Y, X) = d(Y^T G X)/d(m, h, Ibar)   (the mass-vel Jacobian of BackpropSnapshot.cpp:580-640 contracted with g_v').
      // With active contacts W is the field of w = lambda - nu and A the REALISED acceleration: same identity (the
      // constraint rows do not depend on the inertias).
      V6<R> Y2;  // ad(V, W), products rounded on their own (see mul_rn)
      Y2.a = cross_rn(V.a, W.a);
      Y2.l = cross_rn(V.a, W.l) + cross_rn(V.l, W.a);
      R t[10];
      inertia_param_form(W, A, t);
      R t2[10];
      inertia_param_form(Y2, V, t2);
#pragma unroll
      for (int k = 0; k < 10; k++) {
        const float gk = (float)(-dt * (t[k] - t2[k]));
        // gIa (rollouts): every pass ADDS its fp32 term to an fp64 sum over the horizon, the same sum the step-by-step loop forms in
        // autograd (one thread owns the world's row: no atomics)
        if (gIa) gIa[(size_t)(10 * i + k) * gIB] += (double)gk;
        else if (CONTACT && cd.pass2) gI[(size_t)(10 * i + k) * gIB] += gk; else gI[(size_t)(10 * i + k) * gIB] = gk;
      }
    }
    V6<R> Abar = mulG(m, h, Ib, W);
    V6<R> Vbar = mulG(m, h, Ib, ad(W, V)) - crf(W, GV);
    if (hvalid) { Abar = Abar + hA; Vbar = Vbar + hV; f = f + hf; }
    V6<R> Uw = zero6<R>(), Up = zero6<R>(), Gc = zero6<R>(), Hc = zero6<R>();  // contact adjoints (CONTACT only)
    if (CONTACT && cd.active) {
      const int ci = cd.inj_of_body[i];
      if (ci >= 0) {
        const auto b24 = cd.inj + 24 * ci;
        Uw.a = mk3<R>((R)b24[0], (R)b24[1], (R)b24[2]); Uw.l = mk3<R>((R)b24[3], (R)b24[4], (R)b24[5]);
        Up.a = mk3<R>((R)b24[6], (R)b24[7], (R)b24[8]); Up.l = mk3<R>((R)b24[9], (R)b24[10], (R)b24[11]);
        Gc.a = mk3<R>((R)b24[12], (R)b24[13], (R)b24[14]); Gc.l = mk3<R>((R)b24[15], (R)b24[16], (R)b24[17]);
        Hc.a = mk3<R>((R)b24[18], (R)b24[19], (R)b24[20]); Hc.l = mk3<R>((R)b24[21], (R)b24[22], (R)b24[23]);
      }
      if (hvalid) { Uw = Uw + hUw; Up = Up + hUp; Gc = Gc + hG; Hc = Hc + hH; }
    }
    if (fl & NB2_F_HAS_SLOT) {
      for (int k = 0; k < M.slot_count[i]; k++) {
        const R* sl = scr + (size_t)(L.oSlot + SLOTW * (M.slot_self[i] + k)) * ST;
        Abar = Abar + ld6<R, ST>(sl); Vbar = Vbar + ld6<R, ST>(sl + 6 * ST); f = f + ld6<R, ST>(sl + 12 * ST);
        if (CONTACT && cd.active) { Uw = Uw + ld6<R, ST>(sl + 18 * ST); Up = Up + ld6<R, ST>(sl + 24 * ST); Gc = Gc + ld6<R, ST>(sl + 30 * ST); Hc = Hc + ld6<R, ST>(sl + 36 * ST); }
      }
    }
    V6<R> Sv, Sa, Sl;
    Xf<R> T;
    if (jt != NB2_JT_FREE) {
      Sv = S_times<R>(jt, scr[(size_t)(L.oSt + n + o) * ST]);
      Sa = S_times<R>(jt, (CONTACT && cd.active && !cd.pass2) ? (R)cd.aeff[o] : (R)sv[(size_t)(kQdd + o) * B]);
      Sl = S_times<R>(jt, scr[(size_t)(L.oLam + o) * ST]);
      T = (jt == NB2_JT_REV) ? xf_rev(M, bt, i, (R)s[19 * B], (R)s[20 * B]) : xf_pris(M, bt, i, scr[(size_t)(L.oSt + o) * ST]);
    } else {
      Sv.a = mk3<R>(scr[(size_t)(L.oSt + n + o) * ST], scr[(size_t)(L.oSt + n + o + 1) * ST], scr[(size_t)(L.oSt + n + o + 2) * ST]); Sv.l = mk3<R>(scr[(size_t)(L.oSt + n + o + 3) * ST], scr[(size_t)(L.oSt + n + o + 4) * ST], scr[(size_t)(L.oSt + n + o + 5) * ST]);
      Sa = sv_ld6<R>(sv + (size_t)(kQdd + o) * B, B, 0);
      if (CONTACT && cd.active && !cd.pass2) { const auto a6 = cd.aeff + o; Sa.a = mk3<R>((R)a6[0], (R)a6[1], (R)a6[2]); Sa.l = mk3<R>((R)a6[3], (R)a6[4], (R)a6[5]); }
      Sl = ld6<R, ST>(scr + (size_t)(L.oLam + o) * ST);
      R t12[12]; for (int k = 0; k < 12; k++) t12[k] = (R)sv[(size_t)(kFree + M.free_idx[i] * 33 + 21 + k) * B];
      T = ldXf<R, 1>(t12);
    }
    Vbar = Vbar + crf(Sv, Abar);
    const V6<R> vb6 = Vbar - crf(V, Abar);
    const V6<R> Alam = A - Sa - ad(V, Sv), Vlam = V - Sv, Wlam = W - Sl;
    V6<R> c6 = zero6<R>() - (crf(Alam, Abar) + crf(Vlam, Vbar) + crf(Wlam, f));
    if (CONTACT && cd.active) {
      // kinematic-chain part of d/dq [J_r(q) w] and [J_r(q) v+], and the contact-frame part (wrench Gc), see nb2_cw.cuh
      V6<R> Upl; { const auto u6 = cd.Uplus + 6 * i; Upl.a = mk3<R>((R)u6[0], (R)u6[1], (R)u6[2]); Upl.l = mk3<R>((R)u6[3], (R)u6[4], (R)u6[5]); }
      V6<R> Svp;
      if (jt != NB2_JT_FREE) Svp = S_times<R>(jt, (R)cd.vplus[o]);
      else { const auto v6p = cd.vplus + o; Svp.a = mk3<R>((R)v6p[0], (R)v6p[1], (R)v6p[2]); Svp.l = mk3<R>((R)v6p[3], (R)v6p[4], (R)v6p[5]); }
      c6 = c6 - crf(Wlam, Uw) - crf(Upl - Svp, Up) + Gc;
      if (!cd.pass2) {
        if (jt != NB2_JT_FREE) cd.JcTmu[o] = (double)S_dot(jt, Hc);
        else { auto j6 = cd.JcTmu + o; j6[0] = (double)Hc.a.x; j6[1] = (double)Hc.a.y; j6[2] = (double)Hc.a.z; j6[3] = (double)Hc.l.x; j6[4] = (double)Hc.l.y; j6[5] = (double)Hc.l.z; }
      }
    }
    const bool add = CONTACT && cd.pass2;  // second sweep of a bouncing world: accumulate
    if (jt != NB2_JT_FREE) {
      const R vb = S_dot(jt, vb6), qb = S_dot(jt, c6);
      scr[(size_t)(L.oVb + o) * ST] = add ? scr[(size_t)(L.oVb + o) * ST] + vb : vb;
      scr[(size_t)(L.oQb + o) * ST] = add ? scr[(size_t)(L.oQb + o) * ST] + qb : qb;
    } else {
      const V3<R> phi = mk3<R>(scr[(size_t)(L.oSt + o) * ST], scr[(size_t)(L.oSt + o + 1) * ST], scr[(size_t)(L.oSt + o + 2) * ST]);
      V6<R> qb, vb = vb6;
      qb.a = mulT(so3_Jr(phi), c6.a);
      qb.l = mul(expmap(phi), c6.l);
      if (add) { vb = vb + ld6<R, ST>(scr + (size_t)(L.oVb + o) * ST); qb = qb + ld6<R, ST>(scr + (size_t)(L.oQb + o) * ST); }
      st6<R, ST>(scr + (size_t)(L.oVb + o) * ST, vb);
      st6<R, ST>(scr + (size_t)(L.oQb + o) * ST, qb);
    }
    hvalid = false;
    if (p >= 0) {
      const V6<R> cA = dAdInvT(T, Abar), cV = dAdInvT(T, Vbar), cf = dAdInvT(T, f);
      V6<R> cUw, cUp, cG, cH;
      if (CONTACT && cd.active) { cUw = dAdInvT(T, Uw); cUp = dAdInvT(T, Up); cG = dAdInvT(T, Gc); cH = dAdInvT(T, Hc); }
      if (fl & NB2_F_HANDOFF) { hA = cA; hV = cV; hf = cf; if (CONTACT && cd.active) { hUw = cUw; hUp = cUp; hG = cG; hH = cH; } hvalid = true; }
      else {
        R* sl = scr + (size_t)(L.oSlot + SLOTW * M.slot_parent[i]) * ST;
        st6<R, ST>(sl, cA); st6<R, ST>(sl + 6 * ST, cV); st6<R, ST>(sl + 12 * ST, cf);
        if (CONTACT && cd.active) { st6<R, ST>(sl + 18 * ST, cUw); st6<R, ST>(sl + 24 * ST, cUp); st6<R, ST>(sl + 30 * ST, cG); st6<R, ST>(sl + 36 * ST, cH); }
      }
    }
  }
}

// last step of the backward for one dof: clipLossGradientsToBounds (BackpropSnapshot.cpp:425-479; exact equality against
// the pre-step state / action) and the scatter of dL/dtau through the action map (:404-417).  Results replace qbar / vbar
// and the action value in the scratch; bwd_store copies them out.
template <class R, int ST>
NB2_HD void finish_dof(const Nb2ModelDev<R>& M, R* scr, const BwdLayout& L, int d, R gq_, R gv_, R lam) {
  const int n = M.ndof;
  float gq = (float)gq_, gv = (float)gv_;
  const float qd = (float)scr[(size_t)(L.oSt + d) * ST], vd = (float)scr[(size_t)(L.oSt + n + d) * ST];  // exact: fp32 inputs widened
  if (qd == M.pos_lo[d] && gq > 0.f) gq = 0.f;
  if (qd == M.pos_hi[d] && gq < 0.f) gq = 0.f;
  if (vd == M.vel_lo[d] && gv > 0.f) gv = 0.f;
  if (vd == M.vel_hi[d] && gv < 0.f) gv = 0.f;
  scr[(size_t)(L.oQb + d) * ST] = (R)gq;
  scr[(size_t)(L.oVb + d) * ST] = (R)gv;
  const int a = M.act_of_dof[d];
  if (a >= 0) {
    float gt = (float)(M.dt * lam);
    const float fd = (float)scr[(size_t)(L.oAct + a) * ST];
    if (fd == M.force_lo[d] && gt > 0.f) gt = 0.f;
    if (fd == M.force_hi[d] && gt < 0.f) gt = 0.f;
    scr[(size_t)(L.oAct + a) * ST] = (R)gt;
  }
}

template <class R, int ST, bool CONTACT>
NB2_HD void bwd_assemble(const Nb2ModelDev<R>& M, R* scr, const float* st, const BwdContactData<ST>& cd, int lo, int hi) {
  const int nb = M.nb, n = M.ndof;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(nb, n, M.nslots, M.nfree, SLOTW);
  const R dt = M.dt;
  const int kFree = nb * 21, kQdd = nb * 21 + M.nfree * 33;
  (void)n; (void)dt; (void)kFree; (void)kQdd;
  // ---------------- assemble:  g_tau = dt lambda ;  g_q = Pqq^T g_q' - dt (qbar + K lambda) ;
  //                             g_v = Pvq^T g_q' + g_v' - dt (vbar + (D + dt K) lambda)
  for (int i = lo; i < hi; i++) {
    const int jt = M.jtype[i], o = M.dof_off[i];
    if (jt != NB2_JT_FREE) {
      const R lam = scr[(size_t)(L.oLam + o) * ST];
      const R gq = scr[(size_t)(L.oGQ + o) * ST];
      R gv = scr[(size_t)(L.oGV + o) * ST];
      if (CONTACT && cd.active) gv -= (R)cd.JcTmu[o];  // dL/dv* = g - A_c mu
      finish_dof<R, ST>(M, scr, L, o, gq - dt * (scr[(size_t)(L.oQb + o) * ST] + M.spring[o] * lam),
                        dt * gq + gv - dt * (scr[(size_t)(L.oVb + o) * ST] + (M.damping[o] + dt * M.spring[o]) * lam), lam);
    } else {
      // free-joint position update q+ = [log(R(phi) exp(w dt)); p + R(phi) v dt] (the reference differentiates this by
      // finite differences, FreeJoint.cpp:950-1007; closed form here)
      const V3<R> phi = mk3<R>(scr[(size_t)(L.oSt + o) * ST], scr[(size_t)(L.oSt + o + 1) * ST], scr[(size_t)(L.oSt + o + 2) * ST]);
      const V3<R> w = mk3<R>(scr[(size_t)(L.oSt + n + o) * ST], scr[(size_t)(L.oSt + n + o + 1) * ST], scr[(size_t)(L.oSt + n + o + 2) * ST]);
      const V3<R> vl = mk3<R>(scr[(size_t)(L.oSt + n + o + 3) * ST], scr[(size_t)(L.oSt + n + o + 4) * ST], scr[(size_t)(L.oSt + n + o + 5) * ST]);
      const M3<R> Rq = expmap(phi), E = expmap(w * dt);
      const V3<R> phin = logmap(mul(Rq, E));
      const V6<R> g = ld6<R, ST>(scr + (size_t)(L.oGQ + o) * ST);
      const V3<R> t = mulT(so3_Jr_inv(phin), g.a);                 // Jr^-T(phi+) g_phi+
      V6<R> gq, gvp;
      gq.a = mulT(so3_Jr(phi), mul(E, t) + cross(vl * dt, mulT(Rq, g.l)));
      gq.l = g.l;
      gvp.a = mulT(so3_Jr(w * dt), t) * dt;
      gvp.l = mulT(Rq, g.l) * dt;
      const V6<R> lam = ld6<R, ST>(scr + (size_t)(L.oLam + o) * ST);
      const V6<R> qb = ld6<R, ST>(scr + (size_t)(L.oQb + o) * ST), vb = ld6<R, ST>(scr + (size_t)(L.oVb + o) * ST);
      V6<R> gv = ld6<R, ST>(scr + (size_t)(L.oGV + o) * ST);
      if (CONTACT && cd.active) { const auto j6 = cd.JcTmu + o; gv.a = gv.a - mk3<R>((R)j6[0], (R)j6[1], (R)j6[2]); gv.l = gv.l - mk3<R>((R)j6[3], (R)j6[4], (R)j6[5]); }
      R lamv[6] = {lam.a.x, lam.a.y, lam.a.z, lam.l.x, lam.l.y, lam.l.z};
      R qbv[6] = {qb.a.x, qb.a.y, qb.a.z, qb.l.x, qb.l.y, qb.l.z}, vbv[6] = {vb.a.x, vb.a.y, vb.a.z, vb.l.x, vb.l.y, vb.l.z};
      R gqv[6] = {gq.a.x, gq.a.y, gq.a.z, gq.l.x, gq.l.y, gq.l.z}, gvpv[6] = {gvp.a.x, gvp.a.y, gvp.a.z, gvp.l.x, gvp.l.y, gvp.l.z};
      R gvv[6] = {gv.a.x, gv.a.y, gv.a.z, gv.l.x, gv.l.y, gv.l.z};
#pragma unroll
      for (int k = 0; k < 6; k++) {
        finish_dof<R, ST>(M, scr, L, o + k, gqv[k] - dt * (qbv[k] + M.spring[o + k] * lamv[k]),
                          gvpv[k] + gvv[k] - dt * (vbv[k] + (M.damping[o + k] + dt * M.spring[o + k]) * lamv[k]), lamv[k]);
      }
    }
  }
}

// group load of dL/dx', the step's input state and action (B1..B3 and the clipping read them from the scratch)
template <class R, int ST, bool CONTACT>
NB2_HD void bwd_load(const Nb2ModelDev<R>& M, R* scr0, const float* st0, const float* act0, const float* gnext0, int nworlds, int tid, int nthr) {
  const int n = M.ndof, n2 = 2 * n;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(M.nb, n, M.nslots, M.nfree, SLOTW);
  WordScatter<R, ST> sg{scr0, n2, L.oGQ, M.magic_n2, nullptr};  // oGV = oGQ + n
  group_read(gnext0, nworlds * n2, tid, nthr, sg);
  WordScatter<R, ST> sx{scr0, n2, L.oSt, M.magic_n2, nullptr};
  group_read(st0, nworlds * n2, tid, nthr, sx);
  WordScatter<R, ST> sa{scr0, M.na, L.oAct, M.magic_na, nullptr};
  group_read(act0, nworlds * M.na, tid, nthr, sa);
}
struct NanGather { NB2_HD float operator()(int) const { return nanf(""); } };
template <class F> struct AddTo { F f; const float* dst; NB2_HD float operator()(int idx) const { return dst[idx] + f(idx); } };
// group store of the (already clipped) gradients: [oQb, oVb] are adjacent, dL/daction sits in oAct
template <class R, int ST, bool CONTACT>
NB2_HD void bwd_store(const Nb2ModelDev<R>& M, const R* scr0, float* gstate0, float* gaction0,
                      bool cd_error, int nworlds, int tid, int nthr, bool accumulate_state = false) {
  const int n = M.ndof, n2 = 2 * n, na = M.na;
  constexpr int SLOTW = CONTACT ? 42 : 18;
  const BwdLayout L = bwd_layout(M.nb, n, M.nslots, M.nfree, SLOTW);
  if (cd_error) {  // unsupported contact configuration for the backward: fail loudly, never silently wrong
    group_write(gstate0, nworlds * n2, tid, nthr, NanGather());
    group_write(gaction0, nworlds * na, tid, nthr, NanGather());
    return;
  }
  WordGather<R, ST> gs{scr0, n2, L.oQb, M.magic_n2};  // oVb = oQb + n
  if (accumulate_state) {  // rollouts: dL/dx_t = (loss gradient already in the buffer) + clipped back-propagated part
    AddTo<WordGather<R, ST>> acc{gs, gstate0};
    group_write(gstate0, nworlds * n2, tid, nthr, acc);
  } else group_write(gstate0, nworlds * n2, tid, nthr, gs);
  WordGather<R, ST> ga{scr0, na, L.oAct, M.magic_na};
  group_write(gaction0, nworlds * na, tid, nthr, ga);
}

// Stages of the cooperative backward (see world_forward_stage for the trunk/limb split):
//   0 group load of g_next and the input state (bwd_load) | barrier
//   1 B1 limbs (leaf->root)            | barrier
//   2 B1 trunk      3 B2 trunk         | barrier (after 3)
//   4 B2 limbs      5 B3 limbs      6 assemble limbs | barrier (after 6)
//   7 B3 trunk      8 assemble trunk   | barrier
//   9 clip + group store (bwd_store)
#define NB2_BWD_STAGES 10
#define NB2_BWD_SYNC_MASK 0x14Bu        /* after stages 0, 1, 3, 6, 8 */
#define NB2_BWD_SYNC_MASK_1LANE 0x101u  /* lanes == 1: after the group load and before the group store */
// The fused contact backward (k_cstep_bwd, and the host harness that emulates it) walks stages 1..8 in this order over
// NB2_CBWD_ITERS iterations: B1 limbs, B1 trunk, B2 trunk, B2 limbs | contact adjoint (before iteration 4) | B3 limbs, B3 trunk |
// iterations 6, 7: the SECOND B3 over limbs and trunk of a world in which restitution was active (see contact_backward) |
// assembly limbs, trunk.
#define NB2_CBWD_ITERS 10
struct CBwdIter { int stage; bool second; };
NB2_HD constexpr CBwdIter cbwd_iter(int it) {
  return {(it < 4) ? it + 1 : (it == 4 || it == 6) ? 5 : (it == 5 || it == 7) ? 7 : (it == 8) ? 6 : 8, static_cast<bool>((it == 6) | (it == 7))};
}
template <class R, int ST, bool CONTACT = false>
NB2_HD void world_backward_stage(const Nb2ModelDev<R>& M, R* scr, const R* sv, size_t B, int lane, int stage, float* gI = nullptr, const R* bt = nullptr,
                                 size_t gIB = 0, const BwdContactData<ST>* cdp = nullptr, const double* wi = nullptr, size_t wiB = 0,
                                 double* gIa = nullptr) {
  const float* st = nullptr;  // the passes read the state from the scratch (oSt)
  BwdContactData<ST> cd;
  if (CONTACT && cdp) cd = *cdp; else { cd.active = 0; cd.error = 0; cd.inj_of_body = nullptr; }
  // stages 1..8; pass: 1 = B1, 2 = B2, 3 = B3, 4 = assemble
  const int pass = (stage == 1 || stage == 2) ? 1 : (stage == 3 || stage == 4) ? 2 : (stage == 5 || stage == 7) ? 3 : 4;
  const bool trunk = (stage == 2) | (stage == 3) | (stage == 7) | (stage == 8);
  if (trunk && lane != 0) return;
  const int nr = trunk ? M.trunk_n : M.limb_n[lane];
  for (int rr = 0; rr < nr; rr++) {
    const int r = (pass == 1 || pass == 3) ? nr - 1 - rr : rr;
    const int lo = trunk ? M.trunk_lo[r] : M.limb_lo[lane][r], hi = trunk ? M.trunk_hi[r] : M.limb_hi[lane][r];
    if (pass == 1) bwd_B1<R, ST, CONTACT>(M, scr, st, sv, B, lo, hi, bt);
    else if (pass == 2) bwd_B2<R, ST, CONTACT>(M, scr, st, sv, B, lo, hi, bt);
    else if (pass == 3) bwd_B3<R, ST, CONTACT>(M, scr, st, sv, B, cd, lo, hi, gI, bt, gIB ? gIB : B, wi, wiB, gIa);
    else bwd_assemble<R, ST, CONTACT>(M, scr, st, cd, lo, hi);
  }
}

}  // namespace nb2
