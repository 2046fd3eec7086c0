// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the inverse-dynamics device functions (csrc/nb2_dyn.cuh id_*), as k_id_fwd /
// k_id_bwd run them: the step harness (emul.cpp, compiled into this library as it stands) with its group size G, its NT virtual threads
// for the group load / store, its scratch poisoning and the reversed lane order of odd worlds.
#include "emul.cpp"

// inverse dynamics (k_id_fwd / k_id_bwd): rows in the arithmetic type, same group / lane emulation as run_fwd / run_bwd
template <class R>
static int run_id_fwd(const nb2_model_desc* d, int B, const R* state, const R* next_vel, R* tau, R* saved, const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  std::vector<R> scr((size_t)nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree).total * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);
    for (int sg = 0; sg < NB2_ID_FWD_STAGES; sg++) {
      if (sg == 0) { for (int t = NT - 1; t >= 0; t--) nb2::id_load<R, G>(M, scr.data(), state + (size_t)g0 * 2 * M.ndof, next_vel + (size_t)g0 * M.ndof, nw, t, NT); continue; }
      if (sg == NB2_ID_FWD_STAGES - 1) { for (int t = 0; t < NT; t++) nb2::id_store<R, G>(M, scr.data(), tau + (size_t)g0 * M.ndof, nw, t, NT); continue; }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::id_forward_stage<R, G>(M, scr.data() + slot, saved ? saved + w : nullptr, (size_t)B, saved != nullptr, lane, sg, nullptr,
                                      winertia ? winertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
template <class R>
static int run_id_bwd(const nb2_model_desc* d, int B, const R* state, const R* saved, const R* gtau, R* gstate, R* gnext, double* ginertia,
                      const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  std::vector<R> scr((size_t)nb2::id_bwd_words(M.nb, M.ndof, M.nslots, M.nfree) * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);
    for (int sg = 0; sg < NB2_ID_BWD_STAGES; sg++) {
      if (sg == 0) { for (int t = NT - 1; t >= 0; t--) nb2::id_bwd_load<R, G>(M, scr.data(), state + (size_t)g0 * 2 * M.ndof, gtau + (size_t)g0 * M.ndof, nw, t, NT); continue; }
      if (sg == NB2_ID_BWD_STAGES - 1) {
        for (int t = 0; t < NT; t++) nb2::id_bwd_store<R, G>(M, scr.data(), gstate + (size_t)g0 * 2 * M.ndof, gnext + (size_t)g0 * M.ndof, nw, t, NT);
        continue;
      }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::id_backward_stage<R, G>(M, scr.data() + slot, saved + w, (size_t)B, lane, sg, nullptr, winertia ? winertia + w : nullptr, (size_t)B,
                                       ginertia ? ginertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
extern "C" {
// rows and the saved stream in the arithmetic type (double if fp64, float otherwise); ginertia: fp64 [10*nb][B] (may be NULL)
int emul_inverse_dynamics(const nb2_model_desc* d, int B, const void* state, const void* next_vel, void* tau, void* saved, int fp64, const double* winertia) {
  return fp64 ? run_id_fwd<double>(d, B, (const double*)state, (const double*)next_vel, (double*)tau, (double*)saved, winertia)
              : run_id_fwd<float>(d, B, (const float*)state, (const float*)next_vel, (float*)tau, (float*)saved, winertia);
}
int emul_inverse_dynamics_backward(const nb2_model_desc* d, int B, const void* state, const void* saved, const void* gtau, void* gstate, void* gnext,
                                   double* ginertia, int fp64, const double* winertia) {
  return fp64 ? run_id_bwd<double>(d, B, (const double*)state, (const double*)saved, (const double*)gtau, (double*)gstate, (double*)gnext, ginertia, winertia)
              : run_id_bwd<float>(d, B, (const float*)state, (const float*)saved, (const float*)gtau, (float*)gstate, (float*)gnext, ginertia, winertia);
}
}
