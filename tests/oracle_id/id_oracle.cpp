// TEST INFRASTRUCTURE ONLY.  fp64 oracle of the contact-free inverse dynamics, built on the step oracle (oracle/nb_oracle.cpp, compiled
// into this library as it stands): the same model, kinematics and spatial algebra, the force balance of its ABA solved for tau.
//   a = (v' - v) / dt ;  tau = S^T f + K (q - q0 + v dt) + D v   with  f_i = G A_i - dad(V_i, G V_i) - G [0; W_i^T g] + sum_c X*_c f_c,
//   A_i = X^-1 A_p + S a + eta   (reference parametrisation: welds kept, dense 6x6 inertias; dofs of immobile skeletons get 0).
// Templated on the scalar like aba_pass, so that dual numbers give its Jacobians.
#include "../../oracle/nb_oracle.cpp"

namespace orc {
template <class S>
static void inverse_dynamics(const Model& M, const S* q, const S* v, const S* vnext, S* tau) {
  const int nb = M.nb;
  std::vector<BodyState<S>>& B = workspace<S>(nb);
  kinematics_pass<S>(M, q, v, B);
  Vec3<S> g = v3<S>(S(M.gravity[0]), S(M.gravity[1]), S(M.gravity[2]));
  static thread_local std::vector<Vec6<S>> f;
  f.assign(nb, zero6<S>());
  for (int i = 0; i < nb; i++) {
    BodyState<S>& b = B[i];
    if (!M.mobile[i]) { b.A = zero6<S>(); continue; }
    const int p = M.parent[i], o = M.dof_off[i];
    Vec6<S> A = (p >= 0) ? AdInvT(b.T, B[p].A) : zero6<S>();
    for (int a = 0; a < b.k; a++) A = A + b.Scol[a] * ((vnext[o + a] - v[o + a]) / S(M.dt));
    b.A = A + b.eta;
    f[i] = mul(b.G, b.A) - dad(b.V, mul(b.G, b.V)) - mul(b.G, v6(v3<S>(S(0.0), S(0.0), S(0.0)), mulT(b.W.R, g)));
  }
  for (int d = 0; d < M.ndof; d++) tau[d] = S(0.0);
  for (int i = nb - 1; i >= 0; i--) {
    if (!M.mobile[i]) continue;
    const BodyState<S>& b = B[i];
    const int o = M.dof_off[i];
    for (int a = 0; a < b.k; a++)
      tau[o + a] = dot(b.Scol[a], f[i]) + S(M.spring[o + a]) * (q[o + a] - S(M.rest[o + a]) + v[o + a] * M.dt) + S(M.damping[o + a]) * v[o + a];
    if (M.parent[i] >= 0) f[M.parent[i]] = f[M.parent[i]] + dAdInvT(b.T, f[i]);
  }
}
}  // namespace orc

extern "C" {
// state [q; v] (2n), next_vel (n) -> tau (n); J (nullable): d tau / d[q; v; v'] row-major [n x 3n] by dual numbers.  h: a model of
// this library's orc_model_create.
void orc_inverse_dynamics(void* h, const double* state, const double* next_vel, double* tau, double* J) {
  const Model& M = *(Model*)h;
  const int n = M.ndof, cols = 3 * n;
  orc::inverse_dynamics<double>(M, state, state + n, next_vel, tau);
  if (!J) return;
  constexpr int N = 12;
  typedef orc::Dual<N> D;
  std::vector<D> dq(n), dv(n), dvn(n), dtau(n);
  for (int c0 = 0; c0 < cols; c0 += N) {
    for (int i = 0; i < n; i++) { dq[i] = D(state[i]); dv[i] = D(state[n + i]); dvn[i] = D(next_vel[i]); }
    for (int k = 0; k < N && c0 + k < cols; k++) {
      const int c = c0 + k;
      if (c < n) dq[c].d[k] = 1.0; else if (c < 2 * n) dv[c - n].d[k] = 1.0; else dvn[c - 2 * n].d[k] = 1.0;
    }
    orc::inverse_dynamics<D>(M, dq.data(), dv.data(), dvn.data(), dtau.data());
    for (int k = 0; k < N && c0 + k < cols; k++)
      for (int r = 0; r < n; r++) J[(size_t)r * cols + c0 + k] = dtau[r].d[k];
  }
}
}
