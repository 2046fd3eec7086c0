// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the dense dynamics-Jacobian stage functions (csrc/nb2_djac.cuh), as k_dj runs them:
// one world at a time in a poisoned working set, the forward stages over NT virtual lanes, the row rounds of ST slots.  Lanes of a stage
// run in reverse order for odd worlds (and the row slots of a round always in reverse), so that a missing barrier shows up as a poisoned
// read.  The slot count ST is a run-time choice here (4, 8, 16 or 32), to check that the rounds give the same rows.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_djac.cuh"

template <class R, int ST, bool FD>
static void run_dj_world(const Nb2ModelDev<R>& M, int B, size_t w, const R* state, const R* x, const double* winertia, R* out, R* J1, R* J2, R* J3) {
  const int n = M.ndof;
  const size_t nn = (size_t)n * n;
  std::vector<R> ws((size_t)nb2::dj_layout(M, FD, ST).total, R(1e30));
  const R* s = state + w * 2 * n;
  const double* wi = winertia ? winertia + w : nullptr;
  const bool rev = w & 1;
  for (int t = 0; t < NT; t++) nb2::dj_load<R>(M, ws.data(), s, x + w * n, rev ? NT - 1 - t : t, NT);
  for (int sg = 1; sg < nb2::dj_fwd_stages<FD>() - 1; sg++)
    for (int l = 0; l < M.lanes; l++) nb2::dj_forward_stage<R, FD>(M, ws.data(), rev ? M.lanes - 1 - l : l, sg, wi, (size_t)B);
  for (int t = 0; t < NT; t++) nb2::dj_store_out<R>(M, ws.data(), out + w * n, t, NT);
  for (int r0 = 0; r0 < n; r0 += ST) {
    const int nrows = (n - r0 < ST) ? n - r0 : ST;
    for (int t = nrows - 1; t >= 0; t--) nb2::dj_row<R, ST, FD>(M, ws.data(), s, r0 + t, t, wi, (size_t)B);
    for (int t = 0; t < NT; t++) nb2::dj_rows_store<R, ST, FD>(M, ws.data(), r0, nrows, J1 + w * nn, J2 + w * nn, J3 + w * nn, t, NT);
  }
}
template <class R, bool FD>
static int run_dj(const nb2_model_desc* d, int slots, int B, const R* state, const R* x, const double* winertia, R* out, R* J1, R* J2, R* J3) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  if (FD) nb2::fd_identity_actions(M);
  for (int w = 0; w < B; w++) {
    switch (slots) {
      case 32: run_dj_world<R, 32, FD>(M, B, w, state, x, winertia, out, J1, J2, J3); break;
      case 16: run_dj_world<R, 16, FD>(M, B, w, state, x, winertia, out, J1, J2, J3); break;
      case 8: run_dj_world<R, 8, FD>(M, B, w, state, x, winertia, out, J1, J2, J3); break;
      case 4: run_dj_world<R, 4, FD>(M, B, w, state, x, winertia, out, J1, J2, J3); break;
      default: return -1;
    }
  }
  return 0;
}
extern "C" {
// fd: forward dynamics (x = tau), else inverse dynamics (x = next_vel); rows and blocks in double if fp64, else float; winertia may be NULL
int emul_dynamics_jacobians(const nb2_model_desc* d, int fd, int slots, int B, const void* state, const void* x, void* out, void* J1, void* J2, void* J3,
                            int fp64, const double* winertia) {
  if (fp64) {
    auto f = fd ? run_dj<double, true> : run_dj<double, false>;
    return f(d, slots, B, (const double*)state, (const double*)x, winertia, (double*)out, (double*)J1, (double*)J2, (double*)J3);
  }
  auto f = fd ? run_dj<float, true> : run_dj<float, false>;
  return f(d, slots, B, (const float*)state, (const float*)x, winertia, (float*)out, (float*)J1, (float*)J2, (float*)J3);
}
}
