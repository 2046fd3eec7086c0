// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the impulse-dynamics program (csrc/nb2_imp.cuh §6q), as k_imp runs it: one world at
// a time in a poisoned working set, each stage's 32 lanes one after the other (reversed for odd worlds), so that a missing barrier shows up
// as a poisoned read.  The row-slot count (8 or 1) is a run-time choice, to check that the rounds give the same results.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_imp.cuh"

namespace {
constexpr int NL = 32;

template <class R, int ST>
int run(const nb2_model_desc* d, int bwd, int k, int point, const int32_t* body, const double* T, int B, const R* state, const R* off,
        int off_pw, const double* wi, double e, double rho, R* vel, R* imp, const R* gvel, const R* gimp, R* gstate, R* goff, double* gI) {
  Nb2ModelDev<R> F; std::string err;
  if (!nb2_fill_model(*d, F, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::fd_identity_actions(F);
  const Nb2ModelDev<R> M = nb2::imp_model(F);
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(k, point, body, T);
  const int n = M.ndof, m = k * (point ? 3 : 6);
  std::vector<R> ws((size_t)nb2::cfd_layout(M, m, ST).total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    nb2::ImpRows<R> io;
    io.state = state + (size_t)w * 2 * n; io.off = off ? off + (off_pw ? (size_t)w * k * 3 : 0) : nullptr;
    io.vel = bwd ? nullptr : vel + (size_t)w * n; io.imp = bwd ? nullptr : imp + (size_t)w * m;
    io.gvel = bwd ? gvel + (size_t)w * n : nullptr; io.gimp = bwd ? gimp + (size_t)w * m : nullptr;
    io.gstate = bwd ? gstate + (size_t)w * 2 * n : nullptr;
    io.goff = bwd && goff ? goff + (size_t)w * k * 3 : nullptr; io.gI = bwd && gI ? gI + w : nullptr;
    io.wi = wi ? wi + w : nullptr; io.wiB = (size_t)B;
    io.rho = (R)rho; io.e = (R)e;
    auto stage = [&](auto&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l, NL); };
    if (bwd) nb2::imp_world<R, ST, true>(M, N, io, ws.data(), stage);
    else nb2::imp_world<R, ST, false>(M, N, io, ws.data(), stage);
  }
  return 0;
}
template <class R>
int run_st(int slots, const nb2_model_desc* d, int bwd, int k, int point, const int32_t* body, const double* T, int B, const void* state,
           const void* off, int off_pw, const double* wi, double e, double rho, void* vel, void* imp, const void* gvel, const void* gimp,
           void* gstate, void* goff, double* gI) {
  auto f = slots == 8 ? run<R, 8> : run<R, 1>;
  return f(d, bwd, k, point, body, T, B, (const R*)state, (const R*)off, off_pw, wi, e, rho, (R*)vel, (R*)imp, (const R*)gvel, (const R*)gimp,
           (R*)gstate, (R*)goff, gI);
}
}  // namespace

extern "C" {
// bwd = 0: vel [B][n], imp [B][m]; bwd = 1: gstate [B][2n], goff [B][k][3] (or NULL), gI [10 nb][B] (or NULL).  Rows in double if fp64,
// else float; wi: word-major per-world inertia or NULL.
int emul_impulse_dynamics(const nb2_model_desc* d, int bwd, int slots, int k, int point, const int32_t* body, const double* T, int B,
                          const void* state, const void* off, int off_pw, const double* wi, double e, double rho, void* vel, void* imp,
                          const void* gvel, const void* gimp, void* gstate, void* goff, double* gI, int fp64) {
  auto f = fp64 ? run_st<double> : run_st<float>;
  return f(slots, d, bwd, k, point, body, T, B, state, off, off_pw, wi, e, rho, vel, imp, gvel, gimp, gstate, goff, gI);
}
}
