// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the contact inverse-dynamics device functions (csrc/nb2_dyn.cuh cid_*), in the
// order nb2_contact_inverse_dynamics / _backward launch them: the inverse-dynamics harness (emul_id.cpp, compiled into this library as it
// stands) for k_id_fwd / k_id_bwd, and one call per world for k_cid_fwd / k_cid_bwd.
#include "emul_id.cpp"

template <class R>
static int run_cid_fwd(const nb2_model_desc* d, int B, int body, const R* state, const R* next_vel, R* tau, R* wrench, R* saved,
                       const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::CidChain c;
  if (nb2::cid_chain(M, body, &c) < 0) return -2;
  if (int rc = run_id_fwd<R>(d, B, state, next_vel, tau, saved, winertia)) return rc;
  for (int w = 0; w < B; w++) nb2::cid_forward<R>(M, c, state + (size_t)w * 2 * M.ndof, tau + (size_t)w * M.ndof, wrench + (size_t)w * 6);
  return 0;
}
template <class R>
static int run_cid_bwd(const nb2_model_desc* d, int B, int body, const R* state, const R* saved, const R* wrench, const R* gtau, const R* gw,
                       R* gstate, R* gnext, double* ginertia, const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::CidChain c;
  if (nb2::cid_chain(M, body, &c) < 0) return -2;
  const size_t n = M.ndof;
  std::vector<R> seed((size_t)B * n, R(1e30));
  for (int w = 0; w < B; w++) nb2::cid_vjp<R>(M, c, state + w * 2 * n, wrench + (size_t)w * 6, gtau + w * n, gw + (size_t)w * 6, seed.data() + w * n, nullptr);
  if (int rc = run_id_bwd<R>(d, B, state, saved, seed.data(), gstate, gnext, ginertia, winertia)) return rc;
  for (int w = 0; w < B; w++) nb2::cid_vjp<R>(M, c, state + w * 2 * n, wrench + (size_t)w * 6, gtau + w * n, gw + (size_t)w * 6, nullptr, gstate + w * 2 * n);
  return 0;
}
extern "C" {
// body: canonical body index; rows in the arithmetic type (double if fp64, float otherwise); ginertia: fp64 [10*nb][B] (may be NULL)
int emul_contact_inverse_dynamics(const nb2_model_desc* d, int B, int body, const void* state, const void* next_vel, void* tau, void* wrench, void* saved,
                                  int fp64, const double* winertia) {
  return fp64 ? run_cid_fwd<double>(d, B, body, (const double*)state, (const double*)next_vel, (double*)tau, (double*)wrench, (double*)saved, winertia)
              : run_cid_fwd<float>(d, B, body, (const float*)state, (const float*)next_vel, (float*)tau, (float*)wrench, (float*)saved, winertia);
}
int emul_contact_inverse_dynamics_backward(const nb2_model_desc* d, int B, int body, const void* state, const void* saved, const void* wrench,
                                           const void* gtau, const void* gw, void* gstate, void* gnext, double* ginertia, int fp64, const double* winertia) {
  return fp64 ? run_cid_bwd<double>(d, B, body, (const double*)state, (const double*)saved, (const double*)wrench, (const double*)gtau, (const double*)gw,
                                    (double*)gstate, (double*)gnext, ginertia, winertia)
              : run_cid_bwd<float>(d, B, body, (const float*)state, (const float*)saved, (const float*)wrench, (const float*)gtau, (const float*)gw,
                                   (float*)gstate, (float*)gnext, ginertia, winertia);
}
}
