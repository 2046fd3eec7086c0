// TEST INFRASTRUCTURE ONLY.  fp64 oracle of the contact inverse dynamics, built on the inverse-dynamics oracle (id_oracle.cpp, compiled into
// this library as it stands).  It follows the definition, not the device's shortcut:
//   J_c = [Ad(W_j) S_j] over the joints j on the path from the contact body to the world (reference parametrisation, welds kept; the
//   columns of every other joint are 0): q-dot -> spatial velocity of the contact body in world axes about the world origin;
//   the wrench solves the root rows  J_c[:, root]^T w = tau_ID[root]  by a general dense solve (Gauss-Jordan, partial pivoting);
//   tau = tau_ID - J_c^T w.
// Templated on the scalar, so that dual numbers give its Jacobians.
#include "id_oracle.cpp"

namespace orc {
template <class S>
static void contact_inverse_dynamics(const Model& M, int body, const S* q, const S* v, const S* vnext, S* tau, S* wrench) {
  const int n = M.ndof;
  inverse_dynamics<S>(M, q, v, vnext, tau);  // tau_ID; its kinematics are still in the workspace
  const std::vector<BodyState<S>>& B = workspace<S>(M.nb);
  std::vector<Vec6<S>> J(n, zero6<S>());  // column d of J_c
  int root = body;
  for (int i = body; i >= 0; i = M.parent[i]) {
    root = i;
    for (int a = 0; a < B[i].k; a++) J[M.dof_off[i] + a] = AdT(B[i].W, B[i].Scol[a]);
  }
  const int o = M.dof_off[root];
  S A[36], b[6];
  for (int r = 0; r < 6; r++) {
    for (int c = 0; c < 6; c++) A[r * 6 + c] = J[o + r][c];
    b[r] = tau[o + r];
  }
  for (int c = 0; c < 6; c++) {
    int piv = c;
    for (int r = c + 1; r < 6; r++) if (std::fabs(val(A[r * 6 + c])) > std::fabs(val(A[piv * 6 + c]))) piv = r;
    for (int j = 0; j < 6; j++) std::swap(A[c * 6 + j], A[piv * 6 + j]);
    std::swap(b[c], b[piv]);
    for (int r = 0; r < 6; r++) {
      if (r == c) continue;
      const S f = A[r * 6 + c] / A[c * 6 + c];
      for (int j = 0; j < 6; j++) A[r * 6 + j] = A[r * 6 + j] - f * A[c * 6 + j];
      b[r] = b[r] - f * b[c];
    }
  }
  for (int c = 0; c < 6; c++) wrench[c] = b[c] / A[c * 6 + c];
  for (int d = 0; d < n; d++) {
    S s = S(0.0);
    for (int c = 0; c < 6; c++) s = s + J[d][c] * wrench[c];
    tau[d] = tau[d] - s;
  }
}
}  // namespace orc

extern "C" {
// body: raw body index (welds kept) under a 6-dof root.  state [q; v] (2n), next_vel (n) -> tau (n), wrench (6); J (nullable):
// d [tau; wrench] / d [q; v; v'] row-major [(n + 6) x 3n] by dual numbers.
void orc_contact_inverse_dynamics(void* h, int body, const double* state, const double* next_vel, double* tau, double* wrench, double* J) {
  const Model& M = *(Model*)h;
  const int n = M.ndof, cols = 3 * n;
  orc::contact_inverse_dynamics<double>(M, body, state, state + n, next_vel, tau, wrench);
  if (!J) return;
  constexpr int N = 12;
  typedef orc::Dual<N> D;
  std::vector<D> dq(n), dv(n), dvn(n), dtau(n), dw(6);
  for (int c0 = 0; c0 < cols; c0 += N) {
    for (int i = 0; i < n; i++) { dq[i] = D(state[i]); dv[i] = D(state[n + i]); dvn[i] = D(next_vel[i]); }
    for (int k = 0; k < N && c0 + k < cols; k++) {
      const int c = c0 + k;
      if (c < n) dq[c].d[k] = 1.0; else if (c < 2 * n) dv[c - n].d[k] = 1.0; else dvn[c - 2 * n].d[k] = 1.0;
    }
    orc::contact_inverse_dynamics<D>(M, body, dq.data(), dv.data(), dvn.data(), dtau.data(), dw.data());
    for (int k = 0; k < N && c0 + k < cols; k++) {
      for (int r = 0; r < n; r++) J[(size_t)r * cols + c0 + k] = dtau[r].d[k];
      for (int r = 0; r < 6; r++) J[(size_t)(n + r) * cols + c0 + k] = dw[r].d[k];
    }
  }
}
}
