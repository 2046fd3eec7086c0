// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the energy-and-momentum device functions (csrc/nb2_energy.cuh §6m), as k_em_fwd /
// k_em_bwd run them: one world at a time, its 32 lanes stage by stage (the kernels' __syncwarp boundaries), the lanes of odd worlds in
// reversed order, the working set poisoned before every world.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_energy.cuh"

namespace {
constexpr int NL = 32;
template <class F> void lanes(int w, F&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l); }

template <class R>
int run(const nb2_model_desc* d, int B, const R* state, int root, const double* wi, R* kin, R* pot, R* mom, const R* gkin, const R* gpot,
        const R* gmom, R* gstate, double* gI) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  const bool bwd = gstate != nullptr;
  const nb2::EmLayout L = nb2::em_layout(M.nb, n, bwd);
  std::vector<R> ws(L.total);
  const R zero6[6] = {R(0), R(0), R(0), R(0), R(0), R(0)};
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    const R* q = state + (size_t)w * 2 * n;
    const double* wiw = wi ? wi + w : nullptr;
    lanes(w, [&](int l) { nb2::jcdb_init<R>(M, q, root, ws.data(), l, NL); });
    lanes(w, [&](int l) { nb2::jc_moments<R>(M, root, wiw, (size_t)B, ws.data(), l, NL); });
    lanes(w, [&](int l) { nb2::jcd_vel<R>(M, q + n, root, wiw, (size_t)B, true, ws.data(), l); });
    if (!bwd) {
      lanes(w, [&](int l) { nb2::em_bodies<R>(M, root, wiw, (size_t)B, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::em_sums<R>(M, q, root, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::em_store<R>(M, root, ws.data(), kin + w, pot + w, mom + (size_t)w * 6, l); });
    } else {
      const R gT = gkin ? gkin[w] : R(0), gU = gpot ? gpot[w] : R(0);
      const R* gh = gmom ? gmom + (size_t)w * 6 : zero6;
      lanes(w, [&](int l) { nb2::emb_bodies<R>(M, q, root, wiw, (size_t)B, gT, gU, gh, ws.data(), gI ? gI + w : nullptr, (size_t)B, l, NL); });
      lanes(w, [&](int l) { nb2::emb_reduce<R>(M, q, q + n, root, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jd_store_row<R>(n, ws.data() + L.oGq, gstate + (size_t)w * 2 * n, l, NL); });
    }
  }
  return 0;
}
}  // namespace

extern "C" {
// rows in the arithmetic type (double if fp64, float otherwise).  gstate == NULL: the forward into kin / pot / mom; else the backward.
int emul_energy_momentum(const nb2_model_desc* d, int B, const void* state, int root, const double* wi, void* kin, void* pot, void* mom,
                         const void* gkin, const void* gpot, const void* gmom, void* gstate, double* gI, int fp64) {
  return fp64 ? run<double>(d, B, (const double*)state, root, wi, (double*)kin, (double*)pot, (double*)mom, (const double*)gkin, (const double*)gpot,
                            (const double*)gmom, (double*)gstate, gI)
              : run<float>(d, B, (const float*)state, root, wi, (float*)kin, (float*)pot, (float*)mom, (const float*)gkin, (const float*)gpot,
                           (const float*)gmom, (float*)gstate, gI);
}
}
