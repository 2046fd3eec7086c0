// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the dense-Jacobian program of constrained forward dynamics (csrc/nb2_cfd.cuh
// cfdj_world, §6p), as k_cfdj runs it: one world at a time in a poisoned working set, each stage's 32 lanes one after the other (reversed
// for odd worlds), so that a missing barrier shows up as a poisoned read.  The row-slot count (8 or 1, as the kernels) is a run-time choice.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_cfd.cuh"

namespace {
constexpr int NL = 32;

template <class R, int ST>
int run(const nb2_model_desc* d, int k, int point, const int32_t* body, const double* T, int B, const R* state, const R* tau, const R* off,
        int off_pw, const double* wi, double rho, R* qdd, R* wrench, R* const* J) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::fd_identity_actions(M);
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(k, point, body, T);
  const int n = M.ndof, m = k * (point ? 3 : 6);
  const size_t nn = (size_t)n * n, mn = (size_t)m * n;
  std::vector<R> ws((size_t)nb2::cfdj_layout(M.nb, M.ndof, M.nslots, M.nfree, m, ST).total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    nb2::CfdRows<R> io{};
    io.state = state + (size_t)w * 2 * n; io.tau = tau + (size_t)w * n; io.off = off ? off + (off_pw ? (size_t)w * k * 3 : 0) : nullptr;
    io.qdd = qdd + (size_t)w * n; io.wrench = wrench + (size_t)w * m;
    io.wi = wi ? wi + w : nullptr; io.wiB = (size_t)B;
    io.rho = (R)rho;
    const nb2::CfdJacRows<R> out{J[0] + w * nn, J[1] + w * nn, J[2] + w * nn, J[3] + w * mn, J[4] + w * mn, J[5] + w * mn};
    auto stage = [&](auto&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l, NL); };
    nb2::cfdj_world<R, ST>(M, N, io, out, ws.data(), stage);
  }
  return 0;
}
template <class R>
int run_st(int slots, const nb2_model_desc* d, int k, int point, const int32_t* body, const double* T, int B, const void* state, const void* tau,
           const void* off, int off_pw, const double* wi, double rho, void* qdd, void* wrench, void* const* J) {
  R* Jr[6];
  for (int i = 0; i < 6; i++) Jr[i] = (R*)J[i];
  auto f = slots == 8 ? run<R, 8> : run<R, 1>;
  return f(d, k, point, body, T, B, (const R*)state, (const R*)tau, (const R*)off, off_pw, wi, rho, (R*)qdd, (R*)wrench, Jr);
}
}  // namespace

extern "C" {
// qdd [B][n], wrench [B][m] and the six blocks J = {dqdd/dq, dqdd/dqdot, dqdd/dtau [B][n][n], dwrench/dq, dwrench/dqdot, dwrench/dtau
// [B][m][n]}.  Rows in double if fp64, else float; wi: word-major per-world inertia or NULL.
int emul_constrained_forward_dynamics_jacobians(const nb2_model_desc* d, int slots, int k, int point, const int32_t* body, const double* T, int B,
                                                const void* state, const void* tau, const void* off, int off_pw, const double* wi, double rho,
                                                void* qdd, void* wrench, void* const* J, int fp64) {
  auto f = fp64 ? run_st<double> : run_st<float>;
  return f(slots, d, k, point, body, T, B, state, tau, off, off_pw, wi, rho, qdd, wrench, J);
}
}
