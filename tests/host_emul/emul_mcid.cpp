// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the multiple-contact inverse-dynamics device functions (csrc/nb2_dyn.cuh mcid_*),
// in the order nb2_multiple_contact_inverse_dynamics / _backward launch them: the inverse-dynamics harness (emul_id.cpp) for k_id_fwd /
// k_id_bwd, and one call per world for k_mcid_fwd / k_mcid_bwd.  One contact body runs the contact harness (emul_cid.cpp, compiled into
// this library as it stands) with a zero guess gradient, as the entry points do.
#include "emul_cid.cpp"

template <class R>
static int run_mcid_fwd(const nb2_model_desc* d, int B, int k, const int32_t* body, const double* point, const R* state, const R* next_vel,
                        const R* guess, R* tau, R* wrench, R* saved, const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::McidBodies<R> b;
  if (nb2::mcid_bodies(M, k, body, point, &b) < 0) return -2;
  if (k == 1) return run_cid_fwd<R>(d, B, body[0], state, next_vel, tau, wrench, saved, winertia);
  if (int rc = run_id_fwd<R>(d, B, state, next_vel, tau, saved, winertia)) return rc;
  const size_t n = M.ndof;
  for (int w = 0; w < B; w++)
    nb2::mcid_forward<R>(M, b, state + w * 2 * n, guess ? guess + (size_t)w * 6 * k : nullptr, tau + w * n, wrench + (size_t)w * 6 * k);
  return 0;
}
template <class R>
static int run_mcid_bwd(const nb2_model_desc* d, int B, int k, const int32_t* body, const double* point, const R* state, const R* saved,
                        const R* wrench, const R* guess, const R* gtau, const R* gw, R* gstate, R* gnext, double* ginertia, R* gguess,
                        const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::McidBodies<R> b;
  if (nb2::mcid_bodies(M, k, body, point, &b) < 0) return -2;
  const size_t n = M.ndof, kw = 6 * (size_t)k;
  if (k == 1) {
    if (gguess) for (int i = 0; i < B * 6; i++) gguess[i] = R(0);
    return run_cid_bwd<R>(d, B, body[0], state, saved, wrench, gtau, gw, gstate, gnext, ginertia, winertia);
  }
  std::vector<R> seed((size_t)B * n, R(1e30));
  for (int w = 0; w < B; w++)
    nb2::mcid_vjp<R>(M, b, state + w * 2 * n, wrench + w * kw, guess ? guess + w * kw : nullptr, gtau + w * n, gw + w * kw, seed.data() + w * n,
                     gguess ? gguess + w * kw : nullptr, nullptr);
  if (int rc = run_id_bwd<R>(d, B, state, saved, seed.data(), gstate, gnext, ginertia, winertia)) return rc;
  for (int w = 0; w < B; w++)
    nb2::mcid_vjp<R>(M, b, state + w * 2 * n, wrench + w * kw, guess ? guess + w * kw : nullptr, gtau + w * n, gw + w * kw, nullptr, nullptr,
                     gstate + w * 2 * n);
  return 0;
}
extern "C" {
// body [k]: canonical body indices, point [k][3]: each body's origin in its canonical frame; rows in the arithmetic type (double if fp64,
// float otherwise); guess / gguess [B][k][6] (may be NULL); ginertia: fp64 [10*nb][B] (may be NULL)
int emul_multiple_contact_inverse_dynamics(const nb2_model_desc* d, int B, int k, const int32_t* body, const double* point, const void* state,
                                           const void* next_vel, const void* guess, void* tau, void* wrench, void* saved, int fp64,
                                           const double* winertia) {
  return fp64 ? run_mcid_fwd<double>(d, B, k, body, point, (const double*)state, (const double*)next_vel, (const double*)guess, (double*)tau,
                                     (double*)wrench, (double*)saved, winertia)
              : run_mcid_fwd<float>(d, B, k, body, point, (const float*)state, (const float*)next_vel, (const float*)guess, (float*)tau,
                                    (float*)wrench, (float*)saved, winertia);
}
int emul_multiple_contact_inverse_dynamics_backward(const nb2_model_desc* d, int B, int k, const int32_t* body, const double* point,
                                                    const void* state, const void* saved, const void* wrench, const void* guess, const void* gtau,
                                                    const void* gw, void* gstate, void* gnext, double* ginertia, void* gguess, int fp64,
                                                    const double* winertia) {
  return fp64 ? run_mcid_bwd<double>(d, B, k, body, point, (const double*)state, (const double*)saved, (const double*)wrench,
                                     (const double*)guess, (const double*)gtau, (const double*)gw, (double*)gstate, (double*)gnext, ginertia,
                                     (double*)gguess, winertia)
              : run_mcid_bwd<float>(d, B, k, body, point, (const float*)state, (const float*)saved, (const float*)wrench, (const float*)guess,
                                    (const float*)gtau, (const float*)gw, (float*)gstate, (float*)gnext, ginertia, (float*)gguess, winertia);
}
}
