// =====================================================================================
// TEST INFRASTRUCTURE ONLY.  fp64 CPU oracle for the differentiable timestep.
//
// A plain-C++ (no Eigen) restatement of the reference's algorithm for one world:
//   World::step                      dart/simulation/World.cpp:221-254, :307-333
//   Skeleton::computeForwardDynamics dart/dynamics/Skeleton.cpp:13296-13314 (ABA)
//   BodyNode::update{ArtInertia,BiasForce,AccelerationFD}  dart/dynamics/BodyNode.cpp:2046-2185
//   GenericJoint::*Dynamic           dart/dynamics/detail/GenericJoint.hpp:2168-2185, 2276-2301,
//                                    2395-2421, 2554-2571, 2656-2676
//   joint kinematics                 RevoluteJoint.cpp:141-152,203-211; PrismaticJoint.cpp:139-145,188-196;
//                                    FreeJoint.cpp:65-81,922-929,1027-1061 (DART_USE_IDENTITY_JACOBIAN build)
//   BackpropSnapshot::backprop       dart/neural/BackpropSnapshot.cpp:121-194, clip :425-479, action map :404-417
//
// The five step Jacobians (posPos, velPos, posVel, velVel, forceVel; BackpropSnapshot.cpp:159-178) are
// obtained here by forward-mode automatic differentiation (dual numbers) of the restated forward step,
// i.e. they are the exact derivatives the reference's analytic formulas compute (the reference verifies its
// formulas against finite differences of the same step at 1e-8, unittests/GradientTestUtils.hpp:637-680).
//
// Parity status: the reference cannot be built in this container (Eigen/ccd/assimp absent).  What its test-suite holds as literal
// vectors for this path IS pinned: the 8 LCP instances of unittests/unit/test_LCPUtils.cpp (tests/test_lcp.py) and the contact sets of
// unittests/unit/test_DARTCollide.cpp (box-box face-face annotation, sphere / capsule-end vs box: tests/test_golden_collide.py); the LCP
// stage is bit-compared with the reference's ODE dSolveLCP compiled from a reference tree (oracle/Makefile -> oracle/_ref/libodelcp.so).
// For the dynamics and the gradients the reference ships property tests only (analytic-vs-FD, unittests/GradientTestUtils.hpp): there
// value-level parity is UNPINNED and the oracle is held by the same properties (tests/test_oracle.py).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this library.
// =====================================================================================
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "spatial.hpp"
#include "contact.hpp"
#include "lcp_chain.hpp"

namespace orc {

enum { WELD = 0, REVOLUTE = 1, PRISMATIC = 2, FREE = 3 };

struct Model {
  int nb = 0, ndof = 0;
  std::vector<int> parent, jtype, dof_off, mobile;
  std::vector<double> axis, Tpj, Tcj, mass, com, moment;
  std::vector<double> damping, spring, rest, pos_lo, pos_hi, vel_lo, vel_hi, force_lo, force_hi;
  double gravity[3] = {0, 0, -9.81};
  double dt = 1e-3;
  std::vector<int> action_map;
  // contact stage
  std::vector<int> skel_id, shape_body, shape_type;
  std::vector<double> shape_dims, shape_T, friction, restitution;
  bool penetration_correction = false;
  double clip_depth = 0.03, fallback_cfm = 1e-4;
  std::vector<int> has_dofs_above;  // BodyNode::getNumDependentGenCoords() > 0
  std::vector<int> self_collision, adjacent_check;  // per body: Skeleton::isEnabledSelfCollisionCheck / isEnabledAdjacentBodyCheck of its skeleton
  std::vector<int> limit_enforced;  // per body: Joint::isPositionLimitEnforced of its parent joint (1-dof joints; constraint/JointLimitConstraint.cpp)
  std::vector<int> rigid_root;      // first ancestor reached through weld joints only (bodies with the same one cannot move against each other)
};

template <class S> static Iso<S> iso_from12(const double* t) {
  Iso<S> T;
  for (int i = 0; i < 9; i++) T.R.m[i] = S(t[i]);
  for (int i = 0; i < 3; i++) T.p[i] = S(t[9 + i]);
  return T;
}

// spatial inertia tensor (Inertia::computeSpatialTensor, dart/dynamics/Inertia.cpp:1368-1383)
template <class S> static Mat6<S> spatial_tensor(const Model& M, int i) {
  const double* mo = &M.moment[6 * i];
  double m = M.mass[i];
  Vec3<double> c = v3<double>(M.com[3 * i], M.com[3 * i + 1], M.com[3 * i + 2]);
  Mat3<double> C = skew(c), CT = transpose(C), CCt = mul(C, CT);
  double I[9] = {mo[0], mo[3], mo[4], mo[3], mo[1], mo[5], mo[4], mo[5], mo[2]};
  Mat6<S> G = zero66<S>();
  for (int r = 0; r < 3; r++) for (int cc = 0; cc < 3; cc++) {
    G(r, cc) = S(I[3 * r + cc] + m * CCt(r, cc));
    G(3 + r, cc) = S(m * CT(r, cc));
    G(r, 3 + cc) = S(m * C(r, cc));
    G(3 + r, 3 + cc) = S(r == cc ? m : 0.0);
  }
  return G;
}

template <class S> struct BodyState {
  Iso<S> T;       // parent body <- this body  (Joint::getRelativeTransform)
  Iso<S> W;       // world <- this body
  Mat6<S> G;      // spatial inertia
  Vec6<S> Scol[6];  // joint Jacobian columns (body frame)
  int k = 0;      // dofs
  Vec6<S> V, eta; // spatial velocity, partial acceleration
  Mat6<S> AI;     // articulated inertia
  Vec6<S> pA;     // bias force
  S psi[36];      // inverse projected articulated inertia (k x k)
  S u[6];         // total force
  Vec6<S> A;      // spatial acceleration
};

template <class S> static void invert_spd(const S* Min, int k, S* out) {
  // Gauss-Jordan with partial pivoting on a small k x k matrix (k in {1,6});
  // the reference uses math::inverse<ConfigSpaceT> (1/x for R1, LDLT-based inverse for SE3)
  S a[36], b[36];
  for (int i = 0; i < k * k; i++) a[i] = Min[i];
  for (int i = 0; i < k; i++) for (int j = 0; j < k; j++) b[i * k + j] = S(i == j ? 1.0 : 0.0);
  for (int c = 0; c < k; c++) {
    int piv = c; double best = std::fabs(val(a[c * k + c]));
    for (int r = c + 1; r < k; r++) if (std::fabs(val(a[r * k + c])) > best) { best = std::fabs(val(a[r * k + c])); piv = r; }
    if (piv != c) for (int j = 0; j < k; j++) { S t = a[c * k + j]; a[c * k + j] = a[piv * k + j]; a[piv * k + j] = t; t = b[c * k + j]; b[c * k + j] = b[piv * k + j]; b[piv * k + j] = t; }
    S inv = S(1.0) / a[c * k + c];
    for (int j = 0; j < k; j++) { a[c * k + j] = a[c * k + j] * inv; b[c * k + j] = b[c * k + j] * inv; }
    for (int r = 0; r < k; r++) if (r != c) {
      S f = a[r * k + c];
      for (int j = 0; j < k; j++) { a[r * k + j] = a[r * k + j] - f * a[c * k + j]; b[r * k + j] = b[r * k + j] - f * b[c * k + j]; }
    }
  }
  for (int i = 0; i < k * k; i++) out[i] = b[i];
}

// FreeJoint::integratePositionsExplicit, identity-Jacobian branch (FreeJoint.cpp:922-929)
template <class S> static void free_integrate(const S* q, const S* v, double dt, S* out) {
  Mat3<S> R = expMapRot(v3<S>(q[0], q[1], q[2]));
  Mat3<S> E = expMapRot(v3<S>(v[0] * dt, v[1] * dt, v[2] * dt));
  Vec3<S> w = logMap(mul(R, E));
  Vec3<S> p = v3<S>(q[3], q[4], q[5]) + mul(R, v3<S>(v[3] * dt, v[4] * dt, v[5] * dt));
  for (int i = 0; i < 3; i++) { out[i] = w[i]; out[3 + i] = p[i]; }
}

// One contact-free World::step.  q,v,tau: [ndof] -> qn, vn.  (World.cpp:221-254,307-333)
template <class S> static std::vector<BodyState<S>>& workspace(int nb) {
  // per-thread reusable workspace: a fresh ~1 MB vector per call would hit mmap/munmap and serialise threads
  static thread_local std::vector<BodyState<S>> B;
  if ((int)B.size() < nb) B.resize(nb);
  return B;
}

// kinematics, root -> leaf: joint transforms, world transforms, body-frame spatial velocities (Frame.cpp:144-160, GenericJoint.hpp:1803-1823)
template <class S>
static void kinematics_pass(const Model& M, const S* q, const S* v, std::vector<BodyState<S>>& B) {
  const int nb = M.nb;
  // ---- kinematics, root -> leaf (Frame.cpp:144-160, GenericJoint.hpp:1803-1823)
  for (int i = 0; i < nb; i++) {
    BodyState<S>& b = B[i];
    const int o = M.dof_off[i];
    Iso<S> Tpj = iso_from12<S>(&M.Tpj[12 * i]), Tcj = iso_from12<S>(&M.Tcj[12 * i]);
    Vec3<S> ax = v3<S>(S(M.axis[3 * i]), S(M.axis[3 * i + 1]), S(M.axis[3 * i + 2]));
    Iso<S> Q = iso_identity<S>();
    b.k = 0;
    switch (M.jtype[i]) {
      case REVOLUTE: {  // RevoluteJoint.cpp:203-211 (T), :141-152 (S = AdTAngular(T_cj, axis))
        b.k = 1;
        Q.R = expMapRot(ax * q[o]);
        b.Scol[0] = AdT(Tcj, v6(ax, v3<S>(S(0.0), S(0.0), S(0.0))));
        break;
      }
      case PRISMATIC: {  // PrismaticJoint.cpp:188-196, :139-145
        b.k = 1;
        Q.p = ax * q[o];
        b.Scol[0] = AdT(Tcj, v6(v3<S>(S(0.0), S(0.0), S(0.0)), ax));
        break;
      }
      case FREE: {  // FreeJoint.cpp:74-81, 1027-1061: T = Tpj * [expMapRot(q0..2), q3..5] * Tcj^-1, S = Ad[Tcj]
        b.k = 6;
        Q.R = expMapRot(v3<S>(q[o], q[o + 1], q[o + 2]));
        Q.p = v3<S>(q[o + 3], q[o + 4], q[o + 5]);
        for (int c = 0; c < 6; c++) { Vec6<S> e = zero6<S>(); e[c] = S(1.0); b.Scol[c] = AdT(Tcj, e); }
        break;
      }
      default: break;  // WELD
    }
    b.T = mul(mul(Tpj, Q), inverse(Tcj));
    const int p = M.parent[i];
    b.W = (p >= 0) ? mul(B[p].W, b.T) : b.T;
    Vec6<S> Sv = zero6<S>();
    for (int c = 0; c < b.k; c++) Sv = Sv + b.Scol[c] * v[o + c];
    b.V = (p >= 0) ? AdInvT(b.T, B[p].V) + Sv : Sv;
    b.eta = ad(b.V, Sv);  // dS = 0 for these joint types in this build
    b.G = spatial_tensor<S>(M, i);
  }
}

// Skeleton::computeForwardDynamics for every mobile skeleton: fills B (transforms, velocities, articulated
// inertias, psi) and the joint accelerations qdd.
template <class S>
static void aba_pass(const Model& M, const S* q, const S* v, const S* tau, std::vector<BodyState<S>>& B, std::vector<S>& qdd) {
  const int nb = M.nb;
  const double dt = M.dt;
  kinematics_pass<S>(M, q, v, B);
  // ---- articulated inertia + bias force, leaf -> root (BodyNode.cpp:2046-2114)
  static thread_local std::vector<std::vector<int>> kids;
  if ((int)kids.size() < nb) kids.resize(nb);
  for (int i = 0; i < nb; i++) kids[i].clear();
  for (int i = 0; i < nb; i++) if (M.parent[i] >= 0) kids[M.parent[i]].push_back(i);
  Vec3<S> g = v3<S>(S(M.gravity[0]), S(M.gravity[1]), S(M.gravity[2]));
  for (int i = nb - 1; i >= 0; i--) {
    BodyState<S>& b = B[i];
    if (!M.mobile[i]) continue;
    b.AI = b.G;
    for (int c : kids[i]) {
      BodyState<S>& ch = B[c];
      Mat6<S> PI = ch.AI;
      if (ch.k > 0) {  // GenericJoint.hpp:2168-2185 ; weld child: no projection (ZeroDofJoint.cpp:828-835)
        Vec6<S> AIS[6];
        for (int a = 0; a < ch.k; a++) AIS[a] = mul(ch.AI, ch.Scol[a]);
        for (int r = 0; r < 6; r++) for (int cc = 0; cc < 6; cc++) {
          S acc = S(0.0);
          for (int a = 0; a < ch.k; a++) for (int e = 0; e < ch.k; e++) acc = acc + AIS[a][r] * ch.psi[a * ch.k + e] * AIS[e][cc];
          PI(r, cc) = PI(r, cc) - acc;
        }
      }
      b.AI = b.AI + transformInertia(inverse(ch.T), PI);
    }
    if (b.k > 0) {  // updateInvProjArtInertiaDynamic (GenericJoint.hpp:2276-2301)
      S proj[36];
      for (int a = 0; a < b.k; a++) { Vec6<S> AIa = mul(b.AI, b.Scol[a]); for (int e = 0; e < b.k; e++) proj[e * b.k + a] = dot(b.Scol[e], AIa); }
      invert_spd(proj, b.k, b.psi);
    }
    // bias force (BodyNode.cpp:2076-2104): -dad(V, G V) - Fext - G * AdInvRLinear(W, g)
    Vec6<S> Fg = mul(b.G, v6(v3<S>(S(0.0), S(0.0), S(0.0)), mulT(b.W.R, g)));
    b.pA = zero6<S>() - dad(b.V, mul(b.G, b.V)) - Fg;
    for (int c : kids[i]) {
      BodyState<S>& ch = B[c];
      Vec6<S> inner = ch.eta;  // addChildBiasForceToDynamic (GenericJoint.hpp:2395-2421)
      if (ch.k > 0) {
        for (int a = 0; a < ch.k; a++) { S s = S(0.0); for (int e = 0; e < ch.k; e++) s = s + ch.psi[a * ch.k + e] * ch.u[e]; inner = inner + ch.Scol[a] * s; }
      }
      Vec6<S> beta = ch.pA + mul(ch.AI, inner);
      b.pA = b.pA + dAdInvT(ch.T, beta);
    }
    // total force (GenericJoint.hpp:2554-2571): tau - K (q - q0 + v dt) - D v - S^T (AI eta + pA)
    Vec6<S> bodyForce = mul(b.AI, b.eta) + b.pA;
    const int o = M.dof_off[i];
    for (int a = 0; a < b.k; a++) {
      S spring = S(-M.spring[o + a]) * (q[o + a] - S(M.rest[o + a]) + v[o + a] * dt);
      S damp = S(-M.damping[o + a]) * v[o + a];
      b.u[a] = tau[o + a] + spring + damp - dot(b.Scol[a], bodyForce);
    }
  }
  // ---- accelerations, root -> leaf (BodyNode.cpp:2159-2185, GenericJoint.hpp:2656-2676, Frame.cpp:254-271)
  qdd.assign(M.ndof, S(0.0));
  for (int i = 0; i < nb; i++) {
    BodyState<S>& b = B[i];
    if (!M.mobile[i]) { b.A = zero6<S>(); continue; }
    const int p = M.parent[i], o = M.dof_off[i];
    Vec6<S> Ap = (p >= 0) ? AdInvT(b.T, B[p].A) : zero6<S>();
    Vec6<S> AIAp = mul(b.AI, Ap);
    Vec6<S> Sa = zero6<S>();
    for (int a = 0; a < b.k; a++) {
      S acc = S(0.0);
      for (int e = 0; e < b.k; e++) acc = acc + b.psi[a * b.k + e] * (b.u[e] - dot(b.Scol[e], AIAp));
      qdd[o + a] = acc;
      Sa = Sa + b.Scol[a] * acc;
    }
    b.A = Ap + Sa + b.eta;
  }
}

// v+ = v + dt qdd (GenericJoint.hpp:1410-1414); q+ = q (+) dt v with the PRE-step velocity (World.cpp:307-322)
template <class S>
static void integrate(const Model& M, const S* q, const S* v, const S* vnew_mobile, S* qn, S* vn) {
  const int nb = M.nb;
  const double dt = M.dt;
  for (int i = 0; i < nb; i++) {
    const int o = M.dof_off[i];
    const int k = (M.jtype[i] == FREE) ? 6 : (M.jtype[i] == WELD ? 0 : 1);
    if (M.jtype[i] == FREE) free_integrate(&q[o], &v[o], dt, &qn[o]);
    else for (int a = 0; a < k; a++) qn[o + a] = q[o + a] + v[o + a] * dt;
    for (int a = 0; a < k; a++) vn[o + a] = M.mobile[i] ? vnew_mobile[o + a] : v[o + a];
  }
}

// One contact-free World::step.  q,v,tau: [ndof] -> qn, vn.  (World.cpp:221-254,307-333)
template <class S>
static void step_nocontact(const Model& M, const S* q, const S* v, const S* tau, S* qn, S* vn, S* qdd_out = nullptr) {
  std::vector<BodyState<S>>& B = workspace<S>(M.nb);
  static thread_local std::vector<S> qdd, vstar;
  aba_pass<S>(M, q, v, tau, B, qdd);
  vstar.assign(M.ndof, S(0.0));
  for (int i = 0; i < M.ndof; i++) vstar[i] = v[i] + qdd[i] * M.dt;
  integrate<S>(M, q, v, vstar.data(), qn, vn);
  if (qdd_out) for (int i = 0; i < M.ndof; i++) qdd_out[i] = qdd[i];
}

// ====================================================================================
// contact stage (double only): ConstraintSolver::solve + integrateVelocitiesFromImpulses
// ====================================================================================
struct ContactRows {
  int nc = 0, m = 0;
  std::vector<Contact<double>> contacts;
  std::vector<int> row_contact, row_off;        // row -> contact index ; contact -> first row
  std::vector<Vec6<double>> JA, JB;             // per row, body-frame wrench on body A / body B
  std::vector<int> reactA, reactB;              // per contact
  std::vector<double> b, lo, hi, restitution;   // per row
  std::vector<int> findex;
  int unsupported = 0;
  std::vector<int> limit_body, limit_side;      // active joint-limit rows appended after the contacts: body whose joint it is, +1 lower / -1 upper
};

static bool is_reactive(const Model& M, int body) { return M.mobile[body] && M.has_dofs_above[body]; }

// active joint-limit rows (JointLimitConstraint::update, JointLimitConstraint.cpp:150-240): 1-dof joints of mobile skeletons whose position
// sits on or beyond a limit; joints in skeleton / tree order as ConstraintSolver::updateConstraints visits them (:642-695)
static void active_limits(const Model& M, const double* q, std::vector<int>& body, std::vector<int>& side) {
  body.clear(); side.clear();
  if (M.limit_enforced.empty()) return;
  for (int i = 0; i < M.nb; i++) {
    if (!M.limit_enforced[i] || !M.mobile[i] || (M.jtype[i] != REVOLUTE && M.jtype[i] != PRISMATIC)) continue;
    const int d = M.dof_off[i];
    if (q[d] - M.pos_lo[d] <= 0.0) { body.push_back(i); side.push_back(+1); }
    else if (q[d] - M.pos_hi[d] >= 0.0) { body.push_back(i); side.push_back(-1); }
  }
}
// the row of a joint-limit constraint as a pair of body-frame wrenches: a unit impulse on the joint (applyUnitImpulse, :258-283) is S on the
// child and its reaction on the parent; with them the generic formulas give b = -(JA.V_A + JB.V_B) = -qdot (getInformation :243-256: the
// "bouncing velocity" is +-allowance * erp / dt with allowance 0, i.e. zero), lo / hi = [0, inf) on a lower limit, (-inf, 0] on an upper one
template <class S>
static void limit_row_wrenches(const Model& M, const std::vector<BodyState<S>>& B, int i, Vec6<S>& JA, Vec6<S>& JB, int& bodyB, bool& reactB) {
  JA = B[i].Scol[0];
  const int p = M.parent[i];
  if (p >= 0) { JB = zero6<S>() - dAdInvT(B[i].T, JA); bodyB = p; reactB = is_reactive(M, p); }
  else { JB = zero6<S>(); bodyB = i; reactB = false; }
}

// impulse-ABA: body impulses imp[i] (body frame) -> joint velocity changes dqd (Skeleton.cpp:13421-13456, 13552-13556,
// BodyNode.cpp:2117-2138, 2188-2215, GenericJoint.hpp:2482-2498, 2607-2613, 2713-2725)
template <class S>
static void impulse_response(const Model& M, std::vector<BodyState<S>>& B, const std::vector<Vec6<S>>& imp,
                             std::vector<S>& dqd, std::vector<Vec6<S>>& dV) {
  const int nb = M.nb;
  static thread_local std::vector<Vec6<S>> pI;
  static thread_local std::vector<S> uI;
  pI.assign(nb, zero6<S>()); uI.assign(M.ndof, S(0.0));
  dqd.assign(M.ndof, S(0.0)); dV.assign(nb, zero6<S>());
  std::vector<std::vector<int>> kids(nb);
  for (int i = 0; i < nb; i++) if (M.parent[i] >= 0) kids[M.parent[i]].push_back(i);
  for (int i = nb - 1; i >= 0; i--) {
    if (!M.mobile[i]) continue;
    BodyState<S>& b = B[i];
    pI[i] = zero6<S>() - imp[i];
    for (int c : kids[i]) {
      BodyState<S>& ch = B[c];
      Vec6<S> beta = pI[c];
      if (ch.k > 0) {
        Vec6<S> Su = zero6<S>();
        const int oc = M.dof_off[c];
        for (int a = 0; a < ch.k; a++) { S sacc = S(0.0); for (int e = 0; e < ch.k; e++) sacc = sacc + ch.psi[a * ch.k + e] * uI[oc + e]; Su = Su + ch.Scol[a] * sacc; }
        beta = beta + mul(ch.AI, Su);
      }
      pI[i] = pI[i] + dAdInvT(ch.T, beta);
    }
    const int o = M.dof_off[i];
    for (int a = 0; a < b.k; a++) uI[o + a] = -dot(b.Scol[a], pI[i]);
  }
  for (int i = 0; i < nb; i++) {
    if (!M.mobile[i]) continue;
    BodyState<S>& b = B[i];
    const int p = M.parent[i], o = M.dof_off[i];
    Vec6<S> Vp = (p >= 0) ? AdInvT(b.T, dV[p]) : zero6<S>();
    Vec6<S> AIVp = mul(b.AI, Vp);
    Vec6<S> Sd = zero6<S>();
    for (int a = 0; a < b.k; a++) {
      S acc = S(0.0);
      for (int e = 0; e < b.k; e++) acc = acc + b.psi[a * b.k + e] * (uI[o + e] - dot(b.Scol[e], AIVp));
      dqd[o + a] = acc;
      Sd = Sd + b.Scol[a] * acc;
    }
    dV[i] = Vp + Sd;
  }
}

template <class S> static void tangent_basis(const Vec3<S>& n, Vec3<S>& t1, Vec3<S>& t2) {  // ContactConstraint.cpp:734-795
  Vec3<S> z = v3<S>(S(0.0), S(0.0), S(1.0)), x = v3<S>(S(1.0), S(0.0), S(0.0)), y = v3<S>(S(0.0), S(1.0), S(0.0));
  Vec3<S> t = cross(z, n);
  if (val(dot(t, t)) < 1e-12) { t = cross(x, n); if (val(dot(t, t)) < 1e-12) { t = cross(y, n); if (val(dot(t, t)) < 1e-12) t = cross(z, n); } }
  t1 = t * (S(1.0) / sqrt(dot(t, t)));
  t2 = cross(n, t1);
}

template <class S>
static void collide_raw(const Model& M, const std::vector<BodyState<S>>& B, std::vector<Contact<S>>& raw, int& unsupported) {
  const int ns = (int)M.shape_body.size();
  const double clip = M.clip_depth;
  std::vector<Iso<S>> Tw(ns);
  for (int s = 0; s < ns; s++) Tw[s] = mul(B[M.shape_body[s]].W, iso_from12<S>(&M.shape_T[12 * s]));
  for (int i = 0; i + 1 < ns; i++) for (int j = i + 1; j < ns; j++) {
    const int bi = M.shape_body[i], bj = M.shape_body[j];
    if (bi == bj) continue;                                   // CollisionFilter.cpp:128-129
    if (!M.mobile[bi] && !M.mobile[bj]) continue;             // :137-138
    if (M.skel_id[bi] == M.skel_id[bj]) {                       // BodyNodeCollisionFilter::ignoresCollision (:140-150)
      if (M.self_collision.empty() || !M.self_collision[bi]) continue;   // self-collision checking is off by default
      if (!M.adjacent_check[bi] && (M.parent[bi] == bj || M.parent[bj] == bi)) continue;  // areAdjacentBodies (:155-170)
      if (M.rigid_root[bi] == M.rigid_root[bj]) continue;       // welded together: no relative motion (dropped on the device side too)
    }
    const int ti = M.shape_type[i], tj = M.shape_type[j];
    Vec3<S> di = v3<S>(S(M.shape_dims[3 * i]), S(M.shape_dims[3 * i + 1]), S(M.shape_dims[3 * i + 2]));
    Vec3<S> dj = v3<S>(S(M.shape_dims[3 * j]), S(M.shape_dims[3 * j + 1]), S(M.shape_dims[3 * j + 2]));
    if (ti == SH_BOX && tj == SH_BOX) collide_box_box(di, Tw[i], dj, Tw[j], clip, bi, bj, i, j, raw);
    else if (ti == SH_BOX && tj == SH_SPHERE) collide_box_sphere(di, Tw[i], dj[0], Tw[j], clip, CLIP_BOTH, bi, bj, i, j, raw);
    else if (ti == SH_SPHERE && tj == SH_BOX) collide_sphere_box(di[0], Tw[i], dj, Tw[j], clip, bi, bj, i, j, raw);
    else if ((ti == SH_BOX && tj == SH_CAPSULE) || (ti == SH_CAPSULE && tj == SH_BOX)) {
      const bool boxFirst = (ti == SH_BOX);
      const int cs = boxFirst ? j : i, bs = boxFirst ? i : j;
      const double r = M.shape_dims[3 * cs], h = M.shape_dims[3 * cs + 1];
      Vec3<S> bdim = boxFirst ? di : dj;
      // which end sphere is deeper inside / closer to the box? (stands in for ccdMPRPenetration's `pos`, DARTCollide.cpp:4455-4491)
      double depth_end[2];
      Iso<S> Tend[2];
      for (int e = 0; e < 2; e++) {
        Iso<S> off = iso_identity<S>(); off.p = v3<S>(S(0.0), S(0.0), S(e == 0 ? h / 2 : -h / 2));
        Tend[e] = mul(Tw[cs], off);
        Vec3<S> pl = apply(inverse(Tw[bs]), Tend[e].p);
        double q[3] = {val(pl[0]), val(pl[1]), val(pl[2])}, plv[3] = {q[0], q[1], q[2]};
        bool inside = true;
        for (int k = 0; k < 3; k++) { double hk = 0.5 * val(bdim[k]); if (q[k] < -hk) { q[k] = -hk; inside = false; } if (q[k] > hk) { q[k] = hk; inside = false; } }
        if (inside) { double mn = 1e300; for (int k = 0; k < 3; k++) mn = std::min(mn, 0.5 * val(bdim[k]) - std::fabs(plv[k])); depth_end[e] = mn + r; }
        else { double d2 = 0; for (int k = 0; k < 3; k++) d2 += (plv[k] - q[k]) * (plv[k] - q[k]); depth_end[e] = r - std::sqrt(d2); }
      }
      if (std::max(depth_end[0], depth_end[1]) < 0) continue;  // no overlap: MPR reports no intersection
      if (std::fabs(depth_end[0] - depth_end[1]) < 1e-9) { unsupported++; continue; }  // side-on "pipe" contact: needs MPR + createCapsuleMeshContact
      const int e = depth_end[0] > depth_end[1] ? 0 : 1;
      const int half = (e == 0) ? CLIP_TOP : CLIP_BOTTOM;
      if (boxFirst) collide_box_sphere(bdim, Tw[bs], S(r), Tend[e], clip, half, bi, bj, i, j, raw);
      else collide_sphere_box(S(r), Tend[e], bdim, Tw[bs], clip, bi, bj, i, j, raw);
    } else if (ti == SH_SPHERE && tj == SH_SPHERE) collide_sphere_sphere(di[0], Tw[i], dj[0], Tw[j], clip, bi, bj, i, j, raw);
    else if (ti == SH_CAPSULE && tj == SH_CAPSULE) collide_capsule_capsule(M.shape_dims[3 * i + 1], di[0], Tw[i], M.shape_dims[3 * j + 1], dj[0], Tw[j], clip, bi, bj, i, j, raw);
    else if (ti == SH_SPHERE && tj == SH_CAPSULE) collide_sphere_capsule(di[0], Tw[i], M.shape_dims[3 * j + 1], dj[0], Tw[j], clip, true, bi, bj, i, j, raw);
    else if (ti == SH_CAPSULE && tj == SH_SPHERE) collide_sphere_capsule(dj[0], Tw[j], M.shape_dims[3 * i + 1], di[0], Tw[i], clip, false, bi, bj, i, j, raw);
    else { unsupported++; }
  }
}

static void collide_world(const Model& M, const std::vector<BodyState<double>>& B, ContactRows& R) {
  const double clip = M.clip_depth;
  std::vector<Contact<double>> raw;
  collide_raw<double>(M, B, raw, R.unsupported);
  // ConstraintSolver::updateConstraints filtering (:576-601)
  for (auto& c : raw) {
    if (dot(c.normal, c.normal) < 1e-12) continue;
    if (c.depth < 0.0) continue;
    if (c.depth > clip) continue;
    if (!(is_reactive(M, c.bodyA) || is_reactive(M, c.bodyB))) continue;  // ContactConstraint::update / isActive
    R.contacts.push_back(c);
  }
  R.nc = (int)R.contacts.size();
}

struct ContactStepInfo {
  ContactRows rows;
  orc::Mat A;
  std::vector<double> x, vstar;
  std::vector<int> mapping;
  int status = 0;
};

static void step_contact(const Model& M, const double* q, const double* v, const double* tau, const double* x_warm, int m_warm,
                         double* qn, double* vn, ContactStepInfo& info) {
  const int nb = M.nb, n = M.ndof;
  std::vector<BodyState<double>>& B = workspace<double>(nb);
  std::vector<double> qdd;
  aba_pass<double>(M, q, v, tau, B, qdd);
  std::vector<double>& vs = info.vstar;
  vs.assign(n, 0.0);
  for (int i = 0; i < nb; i++) { const int o = M.dof_off[i]; for (int a = 0; a < B[i].k; a++) vs[o + a] = M.mobile[i] ? v[o + a] + qdd[o + a] * M.dt : v[o + a]; }
  // body velocities at the unconstrained velocity v* (positions unchanged)
  for (int i = 0; i < nb; i++) {
    BodyState<double>& b = B[i];
    Vec6<double> Sv = zero6<double>();
    for (int c = 0; c < b.k; c++) Sv = Sv + b.Scol[c] * vs[M.dof_off[i] + c];
    b.V = (M.parent[i] >= 0) ? AdInvT(b.T, B[M.parent[i]].V) + Sv : Sv;
  }
  ContactRows& R = info.rows;
  collide_world(M, B, R);
  bool bounce_active = false;  // a restitution term raised some b_i (status bit 1024, informational)
  // ---- rows (ContactConstraint ctor + getInformation)
  for (int ci = 0; ci < R.nc; ci++) {
    const Contact<double>& c = R.contacts[ci];
    const double mu = std::min(M.friction[c.bodyA], M.friction[c.bodyB]);
    const bool fric = mu > 1e-3;
    const double e = M.restitution[c.bodyA] * M.restitution[c.bodyB];
    const bool bounce = e > 1e-3;
    Vec3<double> dirs[3]; dirs[0] = c.normal;
    if (fric) tangent_basis<double>(c.normal, dirs[1], dirs[2]);
    const Iso<double>&WA = B[c.bodyA].W, &WB = B[c.bodyB].W;
    Vec3<double> pA = apply(inverse(WA), c.point), pB = apply(inverse(WB), c.point);
    const int dim = fric ? 3 : 1, off = R.m;
    R.row_off.push_back(off);
    R.reactA.push_back(is_reactive(M, c.bodyA)); R.reactB.push_back(is_reactive(M, c.bodyB));
    for (int k = 0; k < dim; k++) {
      Vec3<double> dA = mulT(WA.R, dirs[k]), dB = mulT(WB.R, neg(dirs[k]));
      Vec6<double> JA = v6(cross(pA, dA), dA), JB = v6(cross(pB, dB), dB);
      R.JA.push_back(JA); R.JB.push_back(JB); R.row_contact.push_back(ci);
      double rel = -(dot(JA, B[c.bodyA].V) + dot(JB, B[c.bodyB].V));  // getRelVelocity (:687-695)
      R.b.push_back(rel);
      R.restitution.push_back(k == 0 && bounce ? e : 0.0);
      if (k == 0) { R.lo.push_back(0.0); R.hi.push_back(HUGE_VAL); R.findex.push_back(-1); }
      else { R.lo.push_back(-mu); R.hi.push_back(mu); R.findex.push_back(off); }
    }
    // bouncing velocity (ContactConstraint.cpp:395-442): ERP 0.01, max ERV 1e-3, allowance 0
    double bv = c.depth - 0.0;
    if (bv < 0) bv = 0; else { bv *= 0.01 * (1.0 / M.dt); if (bv > 1e-3) bv = 1e-3; }
    if (!M.penetration_correction) bv = 0;
    else if (bv > 0) bounce_active = true;
    if (bounce) { double rv = R.b[off] * e; if (rv > 1e-1) { if (rv > bv) { bv = rv; if (bv > 1e2) bv = 1e2; bounce_active = true; } } }
    R.b[off] += bv;
    R.m += dim;
  }
  // ---- joint-limit rows after the contact rows (ConstraintSolver.cpp:642-695)
  active_limits(M, q, R.limit_body, R.limit_side);
  for (size_t l = 0; l < R.limit_body.size(); l++) {
    const int i = R.limit_body[l];
    Vec6<double> JA, JB; int bodyB; bool reactB;
    limit_row_wrenches<double>(M, B, i, JA, JB, bodyB, reactB);
    Contact<double> c; c.point = v3<double>(0.0, 0.0, 0.0); c.normal = c.point; c.depth = 0.0; c.bodyA = i; c.bodyB = bodyB; c.shapeA = c.shapeB = -1;
    c.type = R.limit_side[l] > 0 ? 100 : 101;
    R.contacts.push_back(c); R.nc++;
    R.row_off.push_back(R.m); R.reactA.push_back(is_reactive(M, i)); R.reactB.push_back(reactB);
    R.JA.push_back(JA); R.JB.push_back(JB); R.row_contact.push_back(R.nc - 1);
    R.b.push_back(-(dot(JA, B[i].V) + (reactB ? dot(JB, B[bodyB].V) : 0.0)));
    R.restitution.push_back(0.0);
    if (R.limit_side[l] > 0) { R.lo.push_back(0.0); R.hi.push_back(HUGE_VAL); } else { R.lo.push_back(-HUGE_VAL); R.hi.push_back(0.0); }
    R.findex.push_back(-1);
    R.m += 1;
  }
  const int m = R.m;
  if (m == 0) { integrate<double>(M, q, v, vs.data(), qn, vn); info.status = 0; return; }
  // ---- A by impulse tests (BoxedLcpConstraintSolver.cpp:190-349): upper blocks measured, lower mirrored
  orc::Mat A(m, m);
  std::vector<Vec6<double>> imp(nb), dV;
  std::vector<double> dqd;
  for (int r = 0; r < m; r++) {
    const int ci = R.row_contact[r];
    const Contact<double>& c = R.contacts[ci];
    for (auto& x : imp) x = zero6<double>();
    if (R.reactA[ci]) imp[c.bodyA] = imp[c.bodyA] + R.JA[r];
    if (R.reactB[ci]) imp[c.bodyB] = imp[c.bodyB] + R.JB[r];
    impulse_response<double>(M, B, imp, dqd, dV);
    for (int s = 0; s < m; s++) {
      const int cj = R.row_contact[s];
      if (cj < ci) { A(r, s) = A(s, r); continue; }
      const Contact<double>& d = R.contacts[cj];
      double a = 0;
      if (R.reactA[cj]) a += dot(R.JA[s], dV[d.bodyA]);
      if (R.reactB[cj]) a += dot(R.JB[s], dV[d.bodyB]);
      A(r, s) = a;
    }
  }
  info.A = A;
  // ---- warm start (:202-208, :334-337)
  orc::Vec x0(m, 0.0);
  if (m_warm == m && x_warm) for (int i = 0; i < m; i++) x0[i] = x_warm[i];
  else x0 = orc::guess_solution(A, R.b, R.findex);
  orc::ChainResult CR = orc::solve_chain(A, R.b, R.lo, R.hi, R.findex, x0, R.restitution, M.fallback_cfm);
  info.x = CR.x; info.mapping = CR.mapping; info.status = CR.status | (R.unsupported ? 128 : 0) | (bounce_active ? 1024 : 0);
  // ---- apply impulses (ConstraintSolver.cpp:813-823, ContactConstraint.cpp:630-684) and update velocities
  for (auto& x : imp) x = zero6<double>();
  for (int r = 0; r < m; r++) {
    const int ci = R.row_contact[r];
    const Contact<double>& c = R.contacts[ci];
    if (R.reactA[ci]) imp[c.bodyA] = imp[c.bodyA] + R.JA[r] * CR.x[r];
    if (R.reactB[ci]) imp[c.bodyB] = imp[c.bodyB] + R.JB[r] * CR.x[r];
  }
  impulse_response<double>(M, B, imp, dqd, dV);
  std::vector<double> vplus(n);
  for (int i = 0; i < n; i++) vplus[i] = vs[i] + dqd[i];
  integrate<double>(M, q, v, vplus.data(), qn, vn);
}

// ====================================================================================
// contact stage with a FIXED classification, scalar-generic: what BackpropSnapshot differentiates
// (dart/neural/BackpropSnapshot.cpp:980-1107): v+ = v* + M^-1 (A_c + A_ub E) f_c ,  f_c = Q^+ b_c ,
// Q = A_c^T M^-1 (A_c + A_ub E) + cfm I , with the clamping / upper-bound sets and E taken from the forward pass.
// Rank-deficient Q (redundant contacts on one rigid body): the velocity update only depends on the generalized impulse,
// which is the same for every solution of Q f = b when Q is symmetric (no upper-bound rows), so the derivative is taken
// through a maximal independent subset of clamping rows chosen on the primal values.
// ====================================================================================
template <class S> static bool solve_dense(int n, std::vector<S>& A, std::vector<S>& b) {  // Gaussian elimination, partial pivoting on values
  for (int c = 0; c < n; c++) {
    int piv = c; double best = std::fabs(val(A[c * n + c]));
    for (int r = c + 1; r < n; r++) if (std::fabs(val(A[r * n + c])) > best) { best = std::fabs(val(A[r * n + c])); piv = r; }
    if (best == 0) return false;
    if (piv != c) { for (int j = 0; j < n; j++) std::swap(A[c * n + j], A[piv * n + j]); std::swap(b[c], b[piv]); }
    S inv = S(1.0) / A[c * n + c];
    for (int r = c + 1; r < n; r++) {
      S f = A[r * n + c] * inv;
      for (int j = c; j < n; j++) A[r * n + j] = A[r * n + j] - f * A[c * n + j];
      b[r] = b[r] - f * b[c];
    }
  }
  for (int r = n - 1; r >= 0; r--) { S acc = b[r]; for (int j = r + 1; j < n; j++) acc = acc - A[r * n + j] * b[j]; b[r] = acc / A[r * n + r]; }
  return true;
}

struct FixedSets {  // from the primal (double) forward pass
  int nc_expected = 0, m = 0;
  std::vector<int> cl, ub, ub_normal_pos;  // row indices; for each ub row the position (in cl) of its normal row
  std::vector<double> ub_E;                // +-mu
  std::vector<int> keep;                   // independent subset of cl (positions in cl)
  double cfm = 0;
  bool ok = true;
  std::vector<int> limit_body, limit_side;  // the active joint-limit rows of the forward pass (frozen like the labels)
};

static FixedSets make_fixed_sets(const ContactStepInfo& info) {
  FixedSets F;
  const ContactRows& R = info.rows;
  F.nc_expected = R.nc; F.m = R.m;
  F.limit_body = R.limit_body; F.limit_side = R.limit_side;
  if (R.m == 0) return F;
  std::vector<int> clpos(R.m, -1);
  for (int j = 0; j < R.m; j++) if (info.mapping[j] == orc::CLAMPING) { clpos[j] = (int)F.cl.size(); F.cl.push_back(j); }
  for (int j = 0; j < R.m; j++) if (info.mapping[j] >= 0) {
    const int fp = info.mapping[j];
    F.ub.push_back(j); F.ub_normal_pos.push_back(clpos[fp]);
    const double up = info.x[fp] * R.hi[j], low = info.x[fp] * R.lo[j];
    F.ub_E.push_back((std::fabs(info.x[j] - up) < std::fabs(info.x[j] - low)) ? R.hi[j] : R.lo[j]);
  }
  for (int j = 0; j < R.m; j++) if (info.mapping[j] == orc::ILLEGAL) F.ok = false;
  F.cfm = (info.status & 8) ? -1.0 : 0.0;  // resolved by the caller (model's fallback cfm)
  const int nCl = (int)F.cl.size();
  // independent subset: pivoted Cholesky on the primal clamping block (symmetric, un-regularised case only; with the
  // fallback cfm on the diagonal Q is non-singular and every clamping row takes part, as in the reference)
  if (F.ub.empty() && !(info.status & 8)) {
    std::vector<double> G((size_t)nCl * nCl), L((size_t)nCl * nCl, 0.0);
    for (int r = 0; r < nCl; r++) for (int c = 0; c < nCl; c++) G[r * nCl + c] = info.A(F.cl[r], F.cl[c]);
    std::vector<int> perm(nCl); for (int i = 0; i < nCl; i++) perm[i] = i;
    double dmax = 0; for (int i = 0; i < nCl; i++) dmax = std::max(dmax, G[i * nCl + i]);
    for (int k = 0; k < nCl; k++) {
      int piv = -1; double best = dmax * 1e-10;
      for (int i = k; i < nCl; i++) { int pi = perm[i]; double d = G[pi * nCl + pi]; for (int j = 0; j < k; j++) d -= L[pi * nCl + j] * L[pi * nCl + j]; if (d > best) { best = d; piv = i; } }
      if (piv < 0) break;
      std::swap(perm[k], perm[piv]);
      const int pk = perm[k]; const double lkk = std::sqrt(best);
      L[pk * nCl + k] = lkk;
      for (int i = k + 1; i < nCl; i++) { int pi = perm[i]; double sacc = G[pi * nCl + pk]; for (int j = 0; j < k; j++) sacc -= L[pi * nCl + j] * L[pk * nCl + j]; L[pi * nCl + k] = sacc / lkk; }
      F.keep.push_back(pk);
    }
    std::sort(F.keep.begin(), F.keep.end());
  } else {
    for (int i = 0; i < nCl; i++) F.keep.push_back(i);
  }
  return F;
}

// v* -> v+ through the contact stage with the sets of F.  B must come from aba_pass<S> at (q, v, tau); vs = v*.
template <class S>
static bool contact_velocity_fixed(const Model& M, std::vector<BodyState<S>>& B, const std::vector<S>& vs, const FixedSets& F,
                                   double cfm, std::vector<S>& vplus) {
  const int nb = M.nb, n = M.ndof;
  vplus = vs;
  if (F.m == 0 || F.cl.empty()) return true;
  for (int i = 0; i < nb; i++) {
    BodyState<S>& b = B[i];
    Vec6<S> Sv = zero6<S>();
    for (int c = 0; c < b.k; c++) Sv = Sv + b.Scol[c] * vs[M.dof_off[i] + c];
    b.V = (M.parent[i] >= 0) ? AdInvT(b.T, B[M.parent[i]].V) + Sv : Sv;
  }
  std::vector<Contact<S>> raw, cs;
  int unsupported = 0;
  collide_raw<S>(M, B, raw, unsupported);
  for (auto& c : raw) {
    if (val(dot(c.normal, c.normal)) < 1e-12) continue;
    if (val(c.depth) < 0.0 || val(c.depth) > M.clip_depth) continue;
    if (!(is_reactive(M, c.bodyA) || is_reactive(M, c.bodyB))) continue;
    cs.push_back(c);
  }
  if ((int)cs.size() + (int)F.limit_body.size() != F.nc_expected) return false;  // the perturbation-free structure must be reproduced
  // rows of every contact (same construction as step_contact)
  std::vector<Vec6<S>> JA, JB; std::vector<S> bvec; std::vector<int> rowc;
  for (int ci = 0; ci < (int)cs.size(); ci++) {
    const Contact<S>& c = cs[ci];
    const double mu = std::min(M.friction[c.bodyA], M.friction[c.bodyB]);
    const bool fric = mu > 1e-3;
    const double e = M.restitution[c.bodyA] * M.restitution[c.bodyB];
    const bool bounce = e > 1e-3;
    Vec3<S> dirs[3]; dirs[0] = c.normal;
    if (fric) tangent_basis<S>(c.normal, dirs[1], dirs[2]);
    const Iso<S>&WA = B[c.bodyA].W, &WB = B[c.bodyB].W;
    Vec3<S> pA = apply(inverse(WA), c.point), pB = apply(inverse(WB), c.point);
    const int dim = fric ? 3 : 1, off = (int)bvec.size();
    for (int k = 0; k < dim; k++) {
      Vec3<S> dA = mulT(WA.R, dirs[k]), dB = mulT(WB.R, neg(dirs[k]));
      Vec6<S> ja = v6(cross(pA, dA), dA), jb = v6(cross(pB, dB), dB);
      JA.push_back(ja); JB.push_back(jb); rowc.push_back(ci);
      bvec.push_back(zero6<S>()[0] - (dot(ja, B[c.bodyA].V) + dot(jb, B[c.bodyB].V)));
    }
    S bv = c.depth;
    if (val(bv) < 0) bv = S(0.0); else { bv = bv * (0.01 * (1.0 / M.dt)); if (val(bv) > 1e-3) bv = S(1e-3); }
    if (!M.penetration_correction) bv = S(0.0);
    if (bounce) { S rv = bvec[off] * e; if (val(rv) > 1e-1) { if (val(rv) > val(bv)) { bv = rv; if (val(bv) > 1e2) bv = S(1e2); } } }
    bvec[off] = bvec[off] + bv;
  }
  // joint-limit rows, frozen at the forward pass's active set
  std::vector<int> lim_bodyB; std::vector<char> lim_reactB;
  const int ncs_real = (int)cs.size();
  for (size_t l = 0; l < F.limit_body.size(); l++) {
    const int i = F.limit_body[l];
    Vec6<S> ja, jb; int bodyB; bool reactB;
    limit_row_wrenches<S>(M, B, i, ja, jb, bodyB, reactB);
    Contact<S> c; c.bodyA = i; c.bodyB = bodyB; c.shapeA = c.shapeB = -1; c.type = 100; c.depth = S(0.0);
    c.point = v3<S>(S(0.0), S(0.0), S(0.0)); c.normal = c.point;
    cs.push_back(c);
    JA.push_back(ja); JB.push_back(jb); rowc.push_back((int)cs.size() - 1);
    S rel = zero6<S>()[0] - dot(ja, B[i].V);
    if (reactB) rel = rel - dot(jb, B[bodyB].V);
    bvec.push_back(rel);
  }
  (void)ncs_real;
  if ((int)bvec.size() != F.m) return false;
  auto response = [&](int r, std::vector<S>& dqd, std::vector<Vec6<S>>& dV) {
    std::vector<Vec6<S>> imp(nb, zero6<S>());
    const Contact<S>& c = cs[rowc[r]];
    if (is_reactive(M, c.bodyA)) imp[c.bodyA] = imp[c.bodyA] + JA[r];
    if (is_reactive(M, c.bodyB)) imp[c.bodyB] = imp[c.bodyB] + JB[r];
    impulse_response<S>(M, B, imp, dqd, dV);
  };
  auto measure = [&](int s2, const std::vector<Vec6<S>>& dV) {
    const Contact<S>& d = cs[rowc[s2]];
    S a = S(0.0);
    if (is_reactive(M, d.bodyA)) a = a + dot(JA[s2], dV[d.bodyA]);
    if (is_reactive(M, d.bodyB)) a = a + dot(JB[s2], dV[d.bodyB]);
    return a;
  };
  const int nk = (int)F.keep.size(), nUb = (int)F.ub.size();
  // Q[r, c] = A(cl_r, cl_c) + sum_u A(cl_r, ub_u) E(u, c)   restricted to the kept rows / columns
  std::vector<S> Q((size_t)nk * nk, S(0.0)), rhs(nk);
  std::vector<S> dqd; std::vector<Vec6<S>> dV;
  for (int c = 0; c < nk; c++) {
    // column c: impulse along P e_c = J_cl[c]^T + sum_{u: normal(u) == c} E_u J_ub[u]^T
    std::vector<Vec6<S>> imp(nb, zero6<S>());
    auto add_row = [&](int r, const S& coef) {
      const Contact<S>& cc = cs[rowc[r]];
      if (is_reactive(M, cc.bodyA)) imp[cc.bodyA] = imp[cc.bodyA] + JA[r] * coef;
      if (is_reactive(M, cc.bodyB)) imp[cc.bodyB] = imp[cc.bodyB] + JB[r] * coef;
    };
    add_row(F.cl[F.keep[c]], S(1.0));
    for (int u = 0; u < nUb; u++) if (F.ub_normal_pos[u] == F.keep[c]) add_row(F.ub[u], S(F.ub_E[u]));
    impulse_response<S>(M, B, imp, dqd, dV);
    for (int r = 0; r < nk; r++) Q[(size_t)r * nk + c] = measure(F.cl[F.keep[r]], dV);
    Q[(size_t)c * nk + c] = Q[(size_t)c * nk + c] + S(cfm);
  }
  for (int r = 0; r < nk; r++) rhs[r] = bvec[F.cl[F.keep[r]]];
  if (!solve_dense<S>(nk, Q, rhs)) return false;
  std::vector<Vec6<S>> imp(nb, zero6<S>());
  for (int c = 0; c < nk; c++) {
    auto add_row = [&](int r, const S& coef) {
      const Contact<S>& cc = cs[rowc[r]];
      if (is_reactive(M, cc.bodyA)) imp[cc.bodyA] = imp[cc.bodyA] + JA[r] * coef;
      if (is_reactive(M, cc.bodyB)) imp[cc.bodyB] = imp[cc.bodyB] + JB[r] * coef;
    };
    add_row(F.cl[F.keep[c]], rhs[c]);
    for (int u = 0; u < nUb; u++) if (F.ub_normal_pos[u] == F.keep[c]) add_row(F.ub[u], rhs[c] * F.ub_E[u]);
  }
  impulse_response<S>(M, B, imp, dqd, dV);
  for (int i = 0; i < n; i++) vplus[i] = vs[i] + dqd[i];
  return true;
}

template <class S>
static bool step_contact_fixed(const Model& M, const S* q, const S* v, const S* tau, const FixedSets& F, double cfm, S* qn, S* vn) {
  std::vector<BodyState<S>>& B = workspace<S>(M.nb);
  static thread_local std::vector<S> qdd;
  aba_pass<S>(M, q, v, tau, B, qdd);
  std::vector<S> vs(M.ndof, S(0.0)), vplus;
  for (int i = 0; i < M.nb; i++) { const int o = M.dof_off[i]; for (int a = 0; a < B[i].k; a++) vs[o + a] = M.mobile[i] ? v[o + a] + qdd[o + a] * M.dt : v[o + a]; }
  if (!contact_velocity_fixed<S>(M, B, vs, F, cfm, vplus)) return false;
  integrate<S>(M, q, v, vplus.data(), qn, vn);
  return true;
}

// Jacobian of the contact step for the classification found by the forward pass at (q, v, tau, x_warm)
static int step_jacobian_contact(const Model& M, const double* q, const double* v, const double* tau, const double* x_warm, int m_warm, double* J) {
  const int n = M.ndof, cols = 3 * n;
  ContactStepInfo info;
  std::vector<double> qn0(n), vn0(n);
  step_contact(M, q, v, tau, x_warm, m_warm, qn0.data(), vn0.data(), info);
  FixedSets F = make_fixed_sets(info);
  const double cfm = (info.status & 8) ? M.fallback_cfm : 0.0;
  if (!F.ok) return -2;
  // consistency: the fixed-set recomputation must reproduce the forward result
  {
    std::vector<double> qn1(n), vn1(n);
    if (!step_contact_fixed<double>(M, q, v, tau, F, cfm, qn1.data(), vn1.data())) return -3;
    double err = 0, ref = 0; for (int i = 0; i < n; i++) { err = std::max(err, std::fabs(vn1[i] - vn0[i])); ref = std::max(ref, std::fabs(vn0[i])); }
    if (err > 1e-7 * std::max(1.0, ref) && !(info.status & 16)) return -4;
  }
  constexpr int N = 12;
  typedef Dual<N> D;
  std::vector<D> dq(n), dv(n), dtau(n), qn(n), vn(n);
  for (int c0 = 0; c0 < cols; c0 += N) {
    for (int i = 0; i < n; i++) { dq[i] = D(q[i]); dv[i] = D(v[i]); dtau[i] = D(tau[i]); }
    for (int k = 0; k < N && c0 + k < cols; k++) {
      int c = c0 + k;
      if (c < n) dq[c].d[k] = 1.0; else if (c < 2 * n) dv[c - n].d[k] = 1.0; else dtau[c - 2 * n].d[k] = 1.0;
    }
    if (!step_contact_fixed<D>(M, dq.data(), dv.data(), dtau.data(), F, cfm, qn.data(), vn.data())) return -5;
    for (int k = 0; k < N && c0 + k < cols; k++) {
      int c = c0 + k;
      for (int r = 0; r < n; r++) { J[(size_t)r * cols + c] = qn[r].d[k]; J[(size_t)(n + r) * cols + c] = vn[r].d[k]; }
    }
  }
  return info.status;
}

// J = d[qn; vn] / d[q; v; tau]  row-major [2n x 3n]
static void step_jacobian(const Model& M, const double* q, const double* v, const double* tau, double* J) {
  constexpr int N = 12;
  typedef Dual<N> D;
  const int n = M.ndof, cols = 3 * n;
  std::vector<D> dq(n), dv(n), dtau(n), qn(n), vn(n);
  for (int c0 = 0; c0 < cols; c0 += N) {
    for (int i = 0; i < n; i++) { dq[i] = D(q[i]); dv[i] = D(v[i]); dtau[i] = D(tau[i]); }
    for (int k = 0; k < N && c0 + k < cols; k++) {
      int c = c0 + k;
      if (c < n) dq[c].d[k] = 1.0; else if (c < 2 * n) dv[c - n].d[k] = 1.0; else dtau[c - 2 * n].d[k] = 1.0;
    }
    step_nocontact<D>(M, dq.data(), dv.data(), dtau.data(), qn.data(), vn.data());
    for (int k = 0; k < N && c0 + k < cols; k++) {
      int c = c0 + k;
      for (int r = 0; r < n; r++) { J[(size_t)r * cols + c] = qn[r].d[k]; J[(size_t)(n + r) * cols + c] = vn[r].d[k]; }
    }
  }
}


// ---- IKMapping (neural/IKMapping.cpp:146-237): mapped positions / velocities of raw body nodes.  type 0 SPATIAL [log R; p | omega; v],
// 1 LINEAR, 2 ANGULAR, 3 COM of the skeleton of body `body` (Skeleton::getCOM = sum m_i W_i c_i / sum m_i).
template <class S> static Vec3<S> ang_of(const Vec6<S>& V) { return v3<S>(V[0], V[1], V[2]); }
template <class S> static Vec3<S> lin_of(const Vec6<S>& V) { return v3<S>(V[3], V[4], V[5]); }
template <class S>
static void ik_map(const Model& M, const S* q, const S* v, int nent, const int* type, const int* body, const int* skel_of_body, S* pos, S* vel) {
  std::vector<BodyState<S>> B(M.nb);
  kinematics_pass<S>(M, q, v, B);
  int cp = 0;
  for (int e = 0; e < nent; e++) {
    if (type[e] == 3) {
      S mt = S(0.0); Vec3<S> c = v3<S>(S(0.0), S(0.0), S(0.0)), cv = c;
      for (int i = 0; i < M.nb; i++) {
        if (skel_of_body[i] != skel_of_body[body[e]]) continue;
        Vec3<S> lc = v3<S>(S(M.com[3 * i]), S(M.com[3 * i + 1]), S(M.com[3 * i + 2]));
        Vec3<S> wc = mul(B[i].W.R, lc) + B[i].W.p;
        Vec3<S> om = mul(B[i].W.R, ang_of(B[i].V)), vl = mul(B[i].W.R, lin_of(B[i].V));
        Vec3<S> vc = vl + cross(om, mul(B[i].W.R, lc));  // BodyNode::getCOMLinearVelocity
        mt = mt + S(M.mass[i]);
        c = c + wc * S(M.mass[i]); cv = cv + vc * S(M.mass[i]);
      }
      for (int k = 0; k < 3; k++) { pos[cp + k] = c[k] / mt; vel[cp + k] = cv[k] / mt; }
      cp += 3;
      continue;
    }
    const BodyState<S>& b = B[body[e]];
    Vec3<S> phi = logMap(b.W.R), om = mul(b.W.R, ang_of(b.V)), vl = mul(b.W.R, lin_of(b.V));
    if (type[e] != 1) { for (int k = 0; k < 3; k++) { pos[cp + k] = phi[k]; vel[cp + k] = om[k]; } cp += 3; }
    if (type[e] != 2) { for (int k = 0; k < 3; k++) { pos[cp + k] = b.W.p[k]; vel[cp + k] = vl[k]; } cp += 3; }
  }
}

}  // namespace orc

// =====================================================================================
// C interface (ctypes)
// =====================================================================================
using orc::Model;
extern "C" {

void* orc_model_create(int nb, int ndof, const int* parent, const int* jtype, const int* dof_off, const int* mobile,
                       const double* axis, const double* Tpj, const double* Tcj, const double* mass, const double* com,
                       const double* moment, const double* damping, const double* spring, const double* rest,
                       const double* pos_lo, const double* pos_hi, const double* vel_lo, const double* vel_hi,
                       const double* force_lo, const double* force_hi, const double* gravity, double dt, int na,
                       const int* action_map) {
  Model* M = new Model();
  M->nb = nb; M->ndof = ndof;
  M->parent.assign(parent, parent + nb); M->jtype.assign(jtype, jtype + nb);
  M->dof_off.assign(dof_off, dof_off + nb); M->mobile.assign(mobile, mobile + nb);
  M->axis.assign(axis, axis + 3 * nb); M->Tpj.assign(Tpj, Tpj + 12 * nb); M->Tcj.assign(Tcj, Tcj + 12 * nb);
  M->mass.assign(mass, mass + nb); M->com.assign(com, com + 3 * nb); M->moment.assign(moment, moment + 6 * nb);
  M->damping.assign(damping, damping + ndof); M->spring.assign(spring, spring + ndof); M->rest.assign(rest, rest + ndof);
  M->pos_lo.assign(pos_lo, pos_lo + ndof); M->pos_hi.assign(pos_hi, pos_hi + ndof);
  M->vel_lo.assign(vel_lo, vel_lo + ndof); M->vel_hi.assign(vel_hi, vel_hi + ndof);
  M->force_lo.assign(force_lo, force_lo + ndof); M->force_hi.assign(force_hi, force_hi + ndof);
  for (int i = 0; i < 3; i++) M->gravity[i] = gravity[i];
  M->dt = dt;
  M->action_map.assign(action_map, action_map + na);
  return M;
}

void orc_model_destroy(void* h) { delete (Model*)h; }

// state = [q; v] (2n), action (na) -> next_state (2n).   World::setState/setAction/step/getState
void orc_step(void* h, const double* state, const double* action, double* next_state, double* qdd /*nullable*/) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];  // World.cpp:2061-2086
  orc::step_nocontact<double>(M, state, state + n, tau.data(), next_state, next_state + n, qdd);
}

// float-precision run of the same restatement (used only to *measure* fp32 sensitivity in tests)
void orc_step_f32(void* h, const double* state, const double* action, double* next_state) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  std::vector<float> q(n), v(n), tau(n, 0.f), qn(n), vn(n);
  for (int i = 0; i < n; i++) { q[i] = (float)state[i]; v[i] = (float)state[n + i]; }
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = (float)action[i];
  orc::step_nocontact<float>(M, q.data(), v.data(), tau.data(), qn.data(), vn.data());
  for (int i = 0; i < n; i++) { next_state[i] = qn[i]; next_state[n + i] = vn[i]; }
}

// IKMapping: mapped pos / vel (dim each) and the Jacobians d pos/d q, d vel/d qdot (row-major [dim x n]) by dual numbers
// (the reference builds them from Skeleton::getWorldPositionJacobian / getWorldJacobian, IKMapping.cpp:371-476)
void orc_ik(void* h, const double* state, int nent, const int* type, const int* body, const int* skel_of_body, int dim, double* pos, double* vel,
            double* Jpos, double* Jvel) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  orc::ik_map<double>(M, state, state + n, nent, type, body, skel_of_body, pos, vel);
  if (!Jpos && !Jvel) return;
  constexpr int N = 12;
  typedef orc::Dual<N> D;
  std::vector<D> q(n), v(n), p(dim), w(dim);
  for (int pass = 0; pass < 2; pass++) {
    double* J = pass ? Jvel : Jpos;
    if (!J) continue;
    for (int c0 = 0; c0 < n; c0 += N) {
      for (int i = 0; i < n; i++) { q[i] = D(state[i]); v[i] = D(state[n + i]); }
      for (int k = 0; k < N && c0 + k < n; k++) (pass ? v : q)[c0 + k].d[k] = 1.0;
      orc::ik_map<D>(M, q.data(), v.data(), nent, type, body, skel_of_body, p.data(), w.data());
      for (int k = 0; k < N && c0 + k < n; k++) for (int r = 0; r < dim; r++) J[(size_t)r * n + c0 + k] = (pass ? w : p)[r].d[k];
    }
  }
}

// Jacobians wrt full tau (n columns), row-major: J[2n x 3n] = d[q+;v+]/d[q;v;tau]
void orc_jacobian(void* h, const double* state, const double* action, double* J) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];
  orc::step_jacobian(M, state, state + n, tau.data(), J);
}

// BackpropSnapshot::backpropState: grad_next_state (2n) -> grad_state (2n), grad_action (na)
void orc_backprop(void* h, const double* state, const double* action, const double* grad_next, double* grad_state,
                  double* grad_action) {
  const Model& M = *(Model*)h;
  const int n = M.ndof, cols = 3 * n;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];
  std::vector<double> J((size_t)2 * n * cols);
  orc::step_jacobian(M, state, state + n, tau.data(), J.data());
  std::vector<double> g(cols, 0.0);
  for (int r = 0; r < 2 * n; r++) for (int c = 0; c < cols; c++) g[c] += J[(size_t)r * cols + c] * grad_next[r];
  // clipLossGradientsToBounds (BackpropSnapshot.cpp:425-479): exact-equality tests against the pre-step state
  for (int j = 0; j < n; j++) {
    double qj = state[j], vj = state[n + j], fj = tau[j];
    if (qj == M.pos_lo[j] && g[j] > 0) g[j] = 0;
    if (qj == M.pos_hi[j] && g[j] < 0) g[j] = 0;
    if (vj == M.vel_lo[j] && g[n + j] > 0) g[n + j] = 0;
    if (vj == M.vel_hi[j] && g[n + j] < 0) g[n + j] = 0;
    if (fj == M.force_lo[j] && g[2 * n + j] > 0) g[2 * n + j] = 0;
    if (fj == M.force_hi[j] && g[2 * n + j] < 0) g[2 * n + j] = 0;
  }
  for (int j = 0; j < 2 * n; j++) grad_state[j] = g[j];
  for (size_t i = 0; i < M.action_map.size(); i++) grad_action[i] = g[2 * n + M.action_map[i]];  // :404-417
}

// ---- contact stage -----------------------------------------------------------------
void orc_model_set_contact(void* h, const int* skel_id, int ns, const int* shape_body, const int* shape_type,
                           const double* shape_dims, const double* shape_T, const double* friction,
                           const double* restitution, int penetration_correction, double clip_depth, double fallback_cfm) {
  Model& M = *(Model*)h;
  M.skel_id.assign(skel_id, skel_id + M.nb);
  M.shape_body.assign(shape_body, shape_body + ns); M.shape_type.assign(shape_type, shape_type + ns);
  M.shape_dims.assign(shape_dims, shape_dims + 3 * ns); M.shape_T.assign(shape_T, shape_T + 12 * ns);
  M.friction.assign(friction, friction + M.nb); M.restitution.assign(restitution, restitution + M.nb);
  M.penetration_correction = penetration_correction != 0; M.clip_depth = clip_depth; M.fallback_cfm = fallback_cfm;
  M.has_dofs_above.assign(M.nb, 0);
  M.rigid_root.assign(M.nb, 0);
  for (int i = 0; i < M.nb; i++) {
    int k = (M.jtype[i] == orc::FREE) ? 6 : (M.jtype[i] == orc::WELD ? 0 : 1);
    M.has_dofs_above[i] = (k > 0) || (M.parent[i] >= 0 && M.has_dofs_above[M.parent[i]]);
    M.rigid_root[i] = (M.jtype[i] == orc::WELD && M.parent[i] >= 0) ? M.rigid_root[M.parent[i]] : i;
  }
}
void orc_model_set_limits(void* h, const int* limit_enforced) {
  Model& M = *(Model*)h;
  M.limit_enforced.assign(limit_enforced, limit_enforced + M.nb);
}
void orc_model_set_self_collision(void* h, const int* self_collision, const int* adjacent_check) {
  Model& M = *(Model*)h;
  M.self_collision.assign(self_collision, self_collision + M.nb);
  M.adjacent_check.assign(adjacent_check, adjacent_check + M.nb);
}

// One World::step with the contact stage.  x_warm/m_warm: cached LCP solution (BoxedLcpConstraintSolver mX) or m_warm=-1.
// Outputs (caller-sized with max_rows / max_contacts): returns the LCP dimension m, or -1 if buffers are too small.
int orc_step_contact(void* h, const double* state, const double* action, const double* x_warm, int m_warm, double* next_state,
                     int max_contacts, int max_rows, int* nc_out, double* contact_point, double* contact_normal,
                     double* contact_depth, int* contact_bodies, int* contact_type, double* A_out, double* b_out, double* lo_out,
                     double* hi_out, int* findex_out, double* x_out, int* mapping_out, int* status_out, double* vstar_out) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];
  orc::ContactStepInfo info;
  orc::step_contact(M, state, state + n, tau.data(), x_warm, m_warm, next_state, next_state + n, info);
  const orc::ContactRows& R = info.rows;
  if (R.nc > max_contacts || R.m > max_rows) return -1;
  *nc_out = R.nc;
  for (int c = 0; c < R.nc; c++) {
    for (int k = 0; k < 3; k++) { contact_point[3 * c + k] = R.contacts[c].point[k]; contact_normal[3 * c + k] = R.contacts[c].normal[k]; }
    contact_depth[c] = R.contacts[c].depth; contact_bodies[2 * c] = R.contacts[c].bodyA; contact_bodies[2 * c + 1] = R.contacts[c].bodyB;
    contact_type[c] = R.contacts[c].type;
  }
  for (int r = 0; r < R.m; r++) {
    b_out[r] = R.b[r]; lo_out[r] = R.lo[r]; hi_out[r] = R.hi[r]; findex_out[r] = R.findex[r];
    x_out[r] = info.x[r]; mapping_out[r] = info.mapping[r];
    for (int c = 0; c < R.m; c++) A_out[(size_t)r * R.m + c] = info.A(r, c);
  }
  *status_out = info.status;
  if (vstar_out) for (int i = 0; i < n; i++) vstar_out[i] = info.vstar[i];
  return R.m;
}

// raw LCP chain on caller data (tests: literal instances of unittests/unit/test_LCPUtils.cpp, comparison with dSolveLCP)
int orc_solve_chain(int n, const double* A, const double* b, const double* lo, const double* hi, const int* findex,
                    const double* x0, int have_x0, double fallback_cfm, double* x_out, int* mapping_out) {
  orc::Mat Am(n, n); orc::Vec bv(b, b + n), lov(lo, lo + n), hiv(hi, hi + n), rest(n, 0.0);
  std::vector<int> fi(findex, findex + n);
  for (int i = 0; i < n * n; i++) Am.a[i] = A[i];
  orc::Vec x0v = have_x0 ? orc::Vec(x0, x0 + n) : orc::guess_solution(Am, bv, fi);
  orc::ChainResult R = orc::solve_chain(Am, bv, lov, hiv, fi, x0v, rest, fallback_cfm);
  for (int i = 0; i < n; i++) { x_out[i] = R.x[i]; mapping_out[i] = R.mapping[i]; }
  return R.status;
}
int orc_lcp_valid(int n, const double* A, const double* x, const double* b, const double* hi, const double* lo, const int* findex) {
  orc::Mat Am(n, n); for (int i = 0; i < n * n; i++) Am.a[i] = A[i];
  return orc::lcp_valid(Am, orc::Vec(x, x + n), orc::Vec(b, b + n), orc::Vec(hi, hi + n), orc::Vec(lo, lo + n), std::vector<int>(findex, findex + n), false) ? 1 : 0;
}
// the Dantzig restatement alone (A row-major n x n, clobbers nothing of the caller's)
int orc_dantzig(int n, const double* A, const double* b, const double* lo, const double* hi, const int* findex, int early, double* x_out) {
  orc::Problem P; P.A = orc::Mat(n, n); for (int i = 0; i < n * n; i++) P.A.a[i] = A[i];
  P.x.assign(n, 0.0); P.b.assign(b, b + n); P.lo.assign(lo, lo + n); P.hi.assign(hi, hi + n); P.fi.assign(findex, findex + n);
  bool ok = orc::run_dantzig(P, early != 0);
  for (int i = 0; i < n; i++) x_out[i] = P.x[i];
  return ok ? 1 : 0;
}
void orc_pinv_solve(int m, int n, const double* Q, const double* b, double* x) {
  orc::Mat Qm(m, n); for (int i = 0; i < m * n; i++) Qm.a[i] = Q[i];
  orc::Vec r = orc::pinv_solve(Qm, orc::Vec(b, b + m));
  for (int i = 0; i < n; i++) x[i] = r[i];
}

// Jacobian / VJP of the contact step (classification frozen at the forward solution).  Returns the forward status (>=0)
// or a negative error (-2 illegal rows, -3/-5 structure changed, -4 fixed-set recomputation disagrees with the forward).
int orc_jacobian_contact(void* h, const double* state, const double* action, const double* x_warm, int m_warm, double* J) {
  const Model& M = *(Model*)h;
  const int n = M.ndof;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];
  return orc::step_jacobian_contact(M, state, state + n, tau.data(), x_warm, m_warm, J);
}
int orc_backprop_contact(void* h, const double* state, const double* action, const double* x_warm, int m_warm, const double* grad_next,
                         double* grad_state, double* grad_action) {
  const Model& M = *(Model*)h;
  const int n = M.ndof, cols = 3 * n;
  std::vector<double> tau(n, 0.0);
  for (size_t i = 0; i < M.action_map.size(); i++) tau[M.action_map[i]] = action[i];
  std::vector<double> J((size_t)2 * n * cols);
  int rc = orc::step_jacobian_contact(M, state, state + n, tau.data(), x_warm, m_warm, J.data());
  if (rc < 0) return rc;
  std::vector<double> g(cols, 0.0);
  for (int r = 0; r < 2 * n; r++) for (int c = 0; c < cols; c++) g[c] += J[(size_t)r * cols + c] * grad_next[r];
  for (int j = 0; j < n; j++) {
    double qj = state[j], vj = state[n + j], fj = tau[j];
    if (qj == M.pos_lo[j] && g[j] > 0) g[j] = 0;
    if (qj == M.pos_hi[j] && g[j] < 0) g[j] = 0;
    if (vj == M.vel_lo[j] && g[n + j] > 0) g[n + j] = 0;
    if (vj == M.vel_hi[j] && g[n + j] < 0) g[n + j] = 0;
    if (fj == M.force_lo[j] && g[2 * n + j] > 0) g[2 * n + j] = 0;
    if (fj == M.force_hi[j] && g[2 * n + j] < 0) g[2 * n + j] = 0;
  }
  for (int j = 0; j < 2 * n; j++) grad_state[j] = g[j];
  for (size_t i = 0; i < M.action_map.size(); i++) grad_action[i] = g[2 * n + M.action_map[i]];
  return rc;
}

}  // extern "C"
