// TEST INFRASTRUCTURE ONLY.  fp64 oracle of the multiple-contact inverse dynamics, built on the contact inverse-dynamics oracle
// (cid_oracle.cpp, compiled into this library as it stands).  It follows the definition, not the device's closed form:
//   J_i = [Ad(W_j) S_j] over the joints j on the path from contact body i to the world (reference parametrisation, welds kept), p_i the
//   world position of body i's own frame; the wrenches minimise sum_i |Gamma(p_i)^-1 (w_i - g_i)|^2 subject to the root rows
//   sum_i J_i[:, root]^T w_i = tau_ID[root], solved through the full KKT system by a general dense solve (solve_dense, partial pivoting);
//   tau = tau_ID - sum_i J_i^T w_i.
// Templated on the scalar, so that dual numbers give its Jacobians.
#include "cid_oracle.cpp"

namespace orc {
template <class S>
static void multiple_contact_inverse_dynamics(const Model& M, int k, const int* body, const S* q, const S* v, const S* vnext, const S* guess,
                                              S* tau, S* wrench) {
  const int n = M.ndof, m = 6 * k + 6;
  inverse_dynamics<S>(M, q, v, vnext, tau);  // tau_ID; its kinematics are still in the workspace
  const std::vector<BodyState<S>>& B = workspace<S>(M.nb);
  std::vector<std::vector<Vec6<S>>> J(k, std::vector<Vec6<S>>(n, zero6<S>()));
  int root = 0;
  std::vector<S> A((size_t)m * m, S(0.0)), b(m, S(0.0));
  for (int i = 0; i < k; i++) {
    for (int j = body[i]; j >= 0; j = M.parent[j]) {
      root = j;
      for (int a = 0; a < B[j].k; a++) J[i][M.dof_off[j] + a] = AdT(B[j].W, B[j].Scol[a]);
    }
    // Q_i = Gi^T Gi with Gi = Gamma(p_i)^-1 = [[I, -[p]x], [0, I]]
    const Mat3<S> P = skew(B[body[i]].W.p);
    S Gi[36];
    for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Gi[r * 6 + c] = S(r == c ? 1.0 : 0.0);
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) Gi[r * 6 + 3 + c] = S(0.0) - P(r, c);
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) {
        S s = S(0.0);
        for (int t = 0; t < 6; t++) s = s + Gi[t * 6 + r] * Gi[t * 6 + c];
        A[(size_t)(6 * i + r) * m + 6 * i + c] = s;
      }
    for (int r = 0; r < 6; r++) {
      S s = S(0.0);
      for (int c = 0; c < 6; c++) s = s + A[(size_t)(6 * i + r) * m + 6 * i + c] * guess[6 * i + c];
      b[6 * i + r] = s;
    }
  }
  const int o = M.dof_off[root];
  for (int i = 0; i < k; i++)
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) A[(size_t)(6 * k + r) * m + 6 * i + c] = A[(size_t)(6 * i + c) * m + 6 * k + r] = J[i][o + r][c];
  for (int r = 0; r < 6; r++) b[6 * k + r] = tau[o + r];
  solve_dense(m, A, b);
  for (int c = 0; c < 6 * k; c++) wrench[c] = b[c];
  for (int d = 0; d < n; d++) {
    S s = S(0.0);
    for (int i = 0; i < k; i++)
      for (int c = 0; c < 6; c++) s = s + J[i][d][c] * wrench[6 * i + c];
    tau[d] = tau[d] - s;
  }
}
}  // namespace orc

extern "C" {
// k raw body indices (welds kept) under one 6-dof root.  state [q; v] (2n), next_vel (n), guess [k][6] (nullable: 0) -> tau (n), wrench
// [k][6]; J (nullable): d [tau; wrench] / d [q; v; v'; guess] row-major [(n + 6k) x (3n + 6k)] by dual numbers.
void orc_multiple_contact_inverse_dynamics(void* h, int k, const int* body, const double* state, const double* next_vel, const double* guess,
                                           double* tau, double* wrench, double* J) {
  const Model& M = *(Model*)h;
  const int n = M.ndof, cols = 3 * n + 6 * k;
  std::vector<double> g(6 * k, 0.0);
  if (guess) g.assign(guess, guess + 6 * k);
  orc::multiple_contact_inverse_dynamics<double>(M, k, body, state, state + n, next_vel, g.data(), tau, wrench);
  if (!J) return;
  constexpr int N = 12;
  typedef orc::Dual<N> D;
  std::vector<D> dq(n), dv(n), dvn(n), dg(6 * k), dtau(n), dw(6 * k);
  for (int c0 = 0; c0 < cols; c0 += N) {
    for (int i = 0; i < n; i++) { dq[i] = D(state[i]); dv[i] = D(state[n + i]); dvn[i] = D(next_vel[i]); }
    for (int i = 0; i < 6 * k; i++) dg[i] = D(g[i]);
    for (int t = 0; t < N && c0 + t < cols; t++) {
      const int c = c0 + t;
      if (c < n) dq[c].d[t] = 1.0; else if (c < 2 * n) dv[c - n].d[t] = 1.0; else if (c < 3 * n) dvn[c - 2 * n].d[t] = 1.0; else dg[c - 3 * n].d[t] = 1.0;
    }
    orc::multiple_contact_inverse_dynamics<D>(M, k, body, dq.data(), dv.data(), dvn.data(), dg.data(), dtau.data(), dw.data());
    for (int t = 0; t < N && c0 + t < cols; t++) {
      for (int r = 0; r < n; r++) J[(size_t)r * cols + c0 + t] = dtau[r].d[t];
      for (int r = 0; r < 6 * k; r++) J[(size_t)(n + r) * cols + c0 + t] = dw[r].d[t];
    }
  }
}
}
