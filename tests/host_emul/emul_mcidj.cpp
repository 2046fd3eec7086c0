// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the dense contact-inverse-dynamics Jacobian stage functions (csrc/nb2_mcidj.cuh),
// as k_mcidj runs them: one world at a time in a poisoned working set, the load and forward stages over NT virtual lanes, the row rounds of
// ST slots.  Lanes of a stage run in reverse order for odd worlds (and the row slots of a round always in reverse), so that a missing
// barrier shows up as a poisoned read.  The slot count ST is a run-time choice here (4, 8, 16 or 32), to check that the rounds give the
// same rows.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_mcidj.cuh"

template <class R, int ST>
static void run_mcidj_world(const Nb2ModelDev<R>& M, const nb2::McidBodies<R>& b, int B, size_t w, const R* state, const R* next_vel,
                            const R* guess, const double* winertia, R* tau, R* wrench, R* const* J) {
  const int n = M.ndof, m = 6 * b.k, rows = n + m;
  const size_t nn = (size_t)n * n, mn = (size_t)m * n, mm = (size_t)m * m;
  std::vector<R> ws((size_t)nb2::mcidj_layout(M, b.k, ST).total, R(1e30));
  const R* s = state + w * 2 * n;
  const R* g = guess ? guess + w * m : nullptr;
  const double* wi = winertia ? winertia + w : nullptr;
  const bool rev = w & 1;
  const nb2::McidjRows<R> out{J[0] + w * nn, J[1] + w * nn, J[2] + w * nn, J[3] ? J[3] + w * mn : nullptr,
                              J[4] + w * mn, J[5] + w * mn, J[6] + w * mn, J[7] ? J[7] + w * mm : nullptr};
  for (int i = 0; i < NT; i++) {
    const int t = rev ? NT - 1 - i : i;
    nb2::dj_load<R>(M, ws.data(), s, next_vel + w * n, t, NT);
    nb2::mcidj_load_guess<R, ST>(M, b.k, ws.data(), g, t, NT);
  }
  for (int sg = 1; sg < NB2_ID_FWD_STAGES - 1; sg++)
    for (int l = 0; l < M.lanes; l++) nb2::dj_forward_stage<R, false>(M, ws.data(), rev ? M.lanes - 1 - l : l, sg, wi, (size_t)B);
  nb2::mcidj_forward<R, ST>(M, b, ws.data(), s, g != nullptr);
  for (int t = 0; t < NT; t++) nb2::mcidj_store_out<R, ST>(M, b.k, ws.data(), tau + w * n, wrench + w * m, rev ? NT - 1 - t : t, NT);
  for (int r0 = 0; r0 < rows; r0 += ST) {
    const int nrows = (rows - r0 < ST) ? rows - r0 : ST;
    for (int t = nrows - 1; t >= 0; t--) nb2::mcidj_row<R, ST>(M, b, ws.data(), s, g != nullptr, r0 + t, t, wi, (size_t)B);
    for (int t = 0; t < NT; t++) nb2::mcidj_rows_store<R, ST>(M, b.k, ws.data(), r0, nrows, out, rev ? NT - 1 - t : t, NT);
  }
}
template <class R>
static int run_mcidj(const nb2_model_desc* d, int slots, int B, int k, const int32_t* body, const double* point, const R* state,
                     const R* next_vel, const R* guess, const double* winertia, R* tau, R* wrench, R* const* J) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::McidBodies<R> b;
  if (nb2::mcid_bodies(M, k, body, point, &b) < 0) return -2;
  for (int w = 0; w < B; w++) {
    switch (slots) {
      case 32: run_mcidj_world<R, 32>(M, b, B, w, state, next_vel, guess, winertia, tau, wrench, J); break;
      case 16: run_mcidj_world<R, 16>(M, b, B, w, state, next_vel, guess, winertia, tau, wrench, J); break;
      case 8: run_mcidj_world<R, 8>(M, b, B, w, state, next_vel, guess, winertia, tau, wrench, J); break;
      case 4: run_mcidj_world<R, 4>(M, b, B, w, state, next_vel, guess, winertia, tau, wrench, J); break;
      default: return -1;
    }
  }
  return 0;
}
extern "C" {
// body [k]: canonical body indices, point [k][3]: each body's origin in its canonical frame; rows in double if fp64, else float; guess
// [B][k][6] may be NULL; J: the eight blocks of nb2_multiple_contact_inverse_dynamics_jacobians (J[3], J[7] may be NULL); winertia may be NULL
int emul_contact_inverse_dynamics_jacobians(const nb2_model_desc* d, int slots, int B, int k, const int32_t* body, const double* point,
                                            const void* state, const void* next_vel, const void* guess, void* tau, void* wrench, void* const* J,
                                            int fp64, const double* winertia) {
  if (fp64)
    return run_mcidj<double>(d, slots, B, k, body, point, (const double*)state, (const double*)next_vel, (const double*)guess, winertia,
                             (double*)tau, (double*)wrench, (double* const*)J);
  return run_mcidj<float>(d, slots, B, k, body, point, (const float*)state, (const float*)next_vel, (const float*)guess, winertia, (float*)tau,
                          (float*)wrench, (float* const*)J);
}
}
