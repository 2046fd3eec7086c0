// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the forward-dynamics device functions (csrc/nb2_dyn.cuh fd_*, world_forward_stage
// with the FD pass 3), as k_fd_fwd / k_fd_bwd run them: the step harness (emul.cpp, compiled into this library as it stands) with its group
// size G, its NT virtual threads for the group load / store, its scratch poisoning and the reversed lane order of odd worlds.
#include "emul.cpp"

// the kernels' model: the descriptor's, with an identity action map (tau per dof)
template <class R> static bool fd_model(const nb2_model_desc* d, Nb2ModelDev<R>* M) {
  std::string err;
  if (!nb2_fill_model(*d, *M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return false; }
  nb2::fd_identity_actions(*M);
  return true;
}
// q, qdot rows `qs` / `vs` words apart, as k_fd_fwd reads them
template <class R>
static int run_fd_fwd(const nb2_model_desc* d, int B, const R* q, int qs, const R* v, int vs, const R* tau, R* qdd, R* saved, const double* winertia) {
  Nb2ModelDev<R> M;
  if (!fd_model(d, &M)) return -1;
  std::vector<R> scr((size_t)nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree).total * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);
    for (int sg = 0; sg < NB2_FWD_STAGES; sg++) {
      if (sg == 0) {
        for (int t = NT - 1; t >= 0; t--)
          nb2::fd_load<R, G>(M, scr.data(), q + (size_t)g0 * qs, qs, v + (size_t)g0 * vs, vs, tau + (size_t)g0 * M.ndof, nw, t, NT);
        continue;
      }
      if (sg == NB2_FWD_STAGES - 1) { for (int t = 0; t < NT; t++) nb2::fd_store<R, G>(M, scr.data(), qdd + (size_t)g0 * M.ndof, nw, t, NT); continue; }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::world_forward_stage<R, G, true>(M, scr.data() + slot, saved ? saved + w : nullptr, (size_t)B, saved != nullptr, lane, sg, nullptr, nullptr,
                                               winertia ? winertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
template <class R>
static int run_fd_bwd(const nb2_model_desc* d, int B, const R* state, const R* saved, const R* gqdd, R* gstate, R* gtau, double* ginertia,
                      const double* winertia) {
  Nb2ModelDev<R> M;
  if (!fd_model(d, &M)) return -1;
  std::vector<R> scr((size_t)nb2::bwd_layout(M.nb, M.ndof, M.nslots, M.nfree).total * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);
    for (int sg = 0; sg < NB2_BWD_STAGES; sg++) {
      if (sg == 0) { for (int t = NT - 1; t >= 0; t--) nb2::fd_bwd_load<R, G>(M, scr.data(), state + (size_t)g0 * 2 * M.ndof, gqdd + (size_t)g0 * M.ndof, nw, t, NT); continue; }
      if (sg == NB2_BWD_STAGES - 1) {
        for (int t = 0; t < NT; t++) nb2::fd_bwd_store<R, G>(M, scr.data(), gstate + (size_t)g0 * 2 * M.ndof, gtau + (size_t)g0 * M.ndof, nw, t, NT);
        continue;
      }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::fd_backward_stage<R, G>(M, scr.data() + slot, saved + w, (size_t)B, lane, sg, nullptr, winertia ? winertia + w : nullptr, (size_t)B,
                                       ginertia ? ginertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
extern "C" {
// rows and the saved stream in the arithmetic type (double if fp64, float otherwise); saved and winertia may be NULL
int emul_forward_dynamics(const nb2_model_desc* d, int B, const void* q, int qs, const void* v, int vs, const void* tau, void* qdd, void* saved, int fp64,
                          const double* winertia) {
  return fp64 ? run_fd_fwd<double>(d, B, (const double*)q, qs, (const double*)v, vs, (const double*)tau, (double*)qdd, (double*)saved, winertia)
              : run_fd_fwd<float>(d, B, (const float*)q, qs, (const float*)v, vs, (const float*)tau, (float*)qdd, (float*)saved, winertia);
}
// ginertia: fp64 [10*nb][B] (may be NULL)
int emul_forward_dynamics_backward(const nb2_model_desc* d, int B, const void* state, const void* saved, const void* gqdd, void* gstate, void* gtau,
                                   double* ginertia, int fp64, const double* winertia) {
  return fp64 ? run_fd_bwd<double>(d, B, (const double*)state, (const double*)saved, (const double*)gqdd, (double*)gstate, (double*)gtau, ginertia, winertia)
              : run_fd_bwd<float>(d, B, (const float*)state, (const float*)saved, (const float*)gqdd, (float*)gstate, (float*)gtau, ginertia, winertia);
}
}
