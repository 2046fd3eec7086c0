// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the regressor device functions (csrc/nb2_reg.cuh §6n), as k_reg_id / k_reg_energy
// run them: one world at a time, its 32 lanes stage by stage (the kernels' __syncwarp boundaries), the lanes of odd worlds in reversed
// order, the working set poisoned before every world.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_reg.cuh"

namespace {
constexpr int NL = 32;
template <class F> void lanes(int w, F&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l); }

template <class R>
int run(const nb2_model_desc* d, int B, const R* state, const R* next_vel, R* Y, R* tp, R* YT, R* YU, R* spring) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof, row = 10 * M.nb;
  const bool energy = Y == nullptr;
  const nb2::RegLayout L = nb2::reg_layout(M, energy);
  std::vector<R> ws(L.total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    const R* s = state + (size_t)w * 2 * n;
    lanes(w, [&](int l) { nb2::dj_load<R>(M, ws.data(), s, energy ? s + n : next_vel + (size_t)w * n, l, NL); });
    for (int sg = 1; sg <= 2; sg++) lanes(w, [&](int l) { nb2::reg_kinematics<R>(M, ws.data(), l, sg); });
    lanes(w, [&](int l) { nb2::reg_poses<R>(M, ws.data(), l); });
    if (!energy) {
      lanes(w, [&](int l) { nb2::reg_axes<R>(M, ws.data(), tp + (size_t)w * n, l, NL); });
      for (int dd = 0; dd < n; dd++) {
        lanes(w, [&](int l) { nb2::reg_id_row<R>(M, ws.data(), dd, l, NL); });
        lanes(w, [&](int l) { nb2::reg_store<R>(ws.data() + L.oY, Y + ((size_t)w * n + dd) * row, row, l, NL); });
      }
    } else {
      lanes(w, [&](int l) { nb2::reg_energy_cols<R>(M, ws.data(), l, NL); });
      lanes(w, [&](int l) {
        nb2::reg_store<R>(ws.data() + L.oY, YT + (size_t)w * row, row, l, NL);
        nb2::reg_store<R>(ws.data() + L.oY + row, YU + (size_t)w * row, row, l, NL);
        nb2::reg_spring_energy<R>(M, ws.data(), spring + w, l);
      });
    }
  }
  return 0;
}
}  // namespace

extern "C" {
// rows in the arithmetic type (double if fp64, float otherwise).  Y != NULL: the ID regressor into Y / tp; else the energy regressor.
int emul_regressor(const nb2_model_desc* d, int B, const void* state, const void* next_vel, void* Y, void* tp, void* YT, void* YU, void* spring,
                   int fp64) {
  return fp64 ? run<double>(d, B, (const double*)state, (const double*)next_vel, (double*)Y, (double*)tp, (double*)YT, (double*)YU, (double*)spring)
              : run<float>(d, B, (const float*)state, (const float*)next_vel, (float*)Y, (float*)tp, (float*)YT, (float*)YU, (float*)spring);
}
}
