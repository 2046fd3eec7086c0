// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the dense-Jacobian program of impulse dynamics (csrc/nb2_imp.cuh impj_world, §6r),
// as k_impj runs it: one world at a time in a poisoned working set, each stage's 32 lanes one after the other (reversed for odd worlds), so
// that a missing barrier shows up as a poisoned read.  The row-slot count (8 or 1, as the kernels) is a run-time choice.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_imp.cuh"

namespace {
constexpr int NL = 32;

template <class R, int ST>
int run(const nb2_model_desc* d, int k, int point, const int32_t* body, const double* T, int B, const R* state, const R* off, int off_pw,
        const double* wi, double e, double rho, R* vel, R* imp, R* const* J) {
  Nb2ModelDev<R> F; std::string err;
  if (!nb2_fill_model(*d, F, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::fd_identity_actions(F);
  const Nb2ModelDev<R> M = nb2::imp_model(F);
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(k, point, body, T);
  const int n = M.ndof, m = k * (point ? 3 : 6);
  const size_t nn = (size_t)n * n, mn = (size_t)m * n;
  std::vector<R> ws((size_t)nb2::cfdj_layout(M.nb, M.ndof, M.nslots, M.nfree, m, ST).total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    nb2::ImpRows<R> io{};
    io.state = state + (size_t)w * 2 * n; io.off = off ? off + (off_pw ? (size_t)w * k * 3 : 0) : nullptr;
    io.vel = vel + (size_t)w * n; io.imp = imp + (size_t)w * m;
    io.wi = wi ? wi + w : nullptr; io.wiB = (size_t)B;
    io.rho = (R)rho; io.e = (R)e;
    const nb2::ImpJacRows<R> out{J[0] + w * nn, J[1] + w * nn, J[2] + w * mn, J[3] + w * mn};
    auto stage = [&](auto&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l, NL); };
    nb2::impj_world<R, ST>(M, N, io, out, ws.data(), stage);
  }
  return 0;
}
template <class R>
int run_st(int slots, const nb2_model_desc* d, int k, int point, const int32_t* body, const double* T, int B, const void* state, const void* off,
           int off_pw, const double* wi, double e, double rho, void* vel, void* imp, void* const* J) {
  R* Jr[4];
  for (int i = 0; i < 4; i++) Jr[i] = (R*)J[i];
  auto f = slots == 8 ? run<R, 8> : run<R, 1>;
  return f(d, k, point, body, T, B, (const R*)state, (const R*)off, off_pw, wi, e, rho, (R*)vel, (R*)imp, Jr);
}
}  // namespace

extern "C" {
// vel [B][n], imp [B][m] and the four blocks J = {dvel/dq, dvel/dqdot- [B][n][n], dimp/dq, dimp/dqdot- [B][m][n]}.  Rows in double if fp64,
// else float; wi: word-major per-world inertia or NULL.
int emul_impulse_dynamics_jacobians(const nb2_model_desc* d, int slots, int k, int point, const int32_t* body, const double* T, int B,
                                    const void* state, const void* off, int off_pw, const double* wi, double e, double rho, void* vel,
                                    void* imp, void* const* J, int fp64) {
  auto f = fp64 ? run_st<double> : run_st<float>;
  return f(slots, d, k, point, body, T, B, state, off, off_pw, wi, e, rho, vel, imp, J);
}
}
