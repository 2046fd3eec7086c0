// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the constrained forward-dynamics program (csrc/nb2_cfd.cuh §6o), as k_cfd runs
// it: one world at a time in a poisoned working set, each stage's 32 lanes one after the other (reversed for odd worlds), so that a missing
// barrier shows up as a poisoned read.  The row-slot count (8 or 1) is a run-time choice, to check that the rounds give the same results.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_cfd.cuh"

namespace {
constexpr int NL = 32;

template <class R, int ST>
int run(const nb2_model_desc* d, int bwd, int k, int point, const int32_t* body, const double* T, int B, const R* state, const R* tau,
        const R* off, int off_pw, const double* wi, double rho, R* qdd, R* wrench, const R* gqdd, const R* gw, R* gstate, R* gtau, R* goff,
        double* gI) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::fd_identity_actions(M);
  nb2::CfdNodes<R> N;
  N.k = k; N.point = point;
  for (int e = 0; e < k; e++) { N.body[e] = body[e]; for (int c = 0; c < 12; c++) N.T[e][c] = (R)T[12 * e + c]; }
  const int n = M.ndof, m = k * (point ? 3 : 6);
  std::vector<R> ws((size_t)nb2::cfd_layout(M, m, ST).total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    nb2::CfdRows<R> io;
    io.state = state + (size_t)w * 2 * n; io.tau = tau + (size_t)w * n; io.off = off ? off + (off_pw ? (size_t)w * k * 3 : 0) : nullptr;
    io.qdd = bwd ? nullptr : qdd + (size_t)w * n; io.wrench = bwd ? nullptr : wrench + (size_t)w * m;
    io.gqdd = bwd ? gqdd + (size_t)w * n : nullptr; io.gw = bwd ? gw + (size_t)w * m : nullptr;
    io.gstate = bwd ? gstate + (size_t)w * 2 * n : nullptr; io.gtau = bwd ? gtau + (size_t)w * n : nullptr;
    io.goff = bwd && goff ? goff + (size_t)w * k * 3 : nullptr; io.gI = bwd && gI ? gI + w : nullptr;
    io.wi = wi ? wi + w : nullptr; io.wiB = (size_t)B;
    io.rho = (R)rho;
    auto stage = [&](auto&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l, NL); };
    if (bwd) nb2::cfd_world<R, ST, true>(M, N, io, ws.data(), stage);
    else nb2::cfd_world<R, ST, false>(M, N, io, ws.data(), stage);
  }
  return 0;
}
template <class R>
int run_st(int slots, const nb2_model_desc* d, int bwd, int k, int point, const int32_t* body, const double* T, int B, const void* state,
           const void* tau, const void* off, int off_pw, const double* wi, double rho, void* qdd, void* wrench, const void* gqdd, const void* gw,
           void* gstate, void* gtau, void* goff, double* gI) {
  auto f = slots == 8 ? run<R, 8> : run<R, 1>;
  return f(d, bwd, k, point, body, T, B, (const R*)state, (const R*)tau, (const R*)off, off_pw, wi, rho, (R*)qdd, (R*)wrench, (const R*)gqdd,
           (const R*)gw, (R*)gstate, (R*)gtau, (R*)goff, gI);
}
}  // namespace

extern "C" {
// bwd = 0: qdd [B][n], wrench [B][m]; bwd = 1: gstate [B][2n], gtau [B][n], goff [B][k][3] (or NULL), gI [10 nb][B] (or NULL).  Rows in
// double if fp64, else float; wi: word-major per-world inertia or NULL.
int emul_constrained_forward_dynamics(const nb2_model_desc* d, int bwd, int slots, int k, int point, const int32_t* body, const double* T, int B,
                                      const void* state, const void* tau, const void* off, int off_pw, const double* wi, double rho, void* qdd,
                                      void* wrench, const void* gqdd, const void* gw, void* gstate, void* gtau, void* goff, double* gI,
                                      int fp64) {
  auto f = fp64 ? run_st<double> : run_st<float>;
  return f(slots, d, bwd, k, point, body, T, B, state, tau, off, off_pw, wi, rho, qdd, wrench, gqdd, gw, gstate, gtau, goff, gI);
}
}
