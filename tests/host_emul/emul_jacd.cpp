// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the Jacobian-derivative device functions (csrc/nb2_jac.cuh §6j), as
// k_jacd_point_fwd / k_jacd_point_bwd / k_jacd_com_fwd / k_jacd_com_bwd run them: one item at a time, its 32 lanes stage by stage (the
// kernels' __syncwarp boundaries), the lanes of odd worlds in reversed order, the working set poisoned before every item.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_jac.cuh"

namespace {
constexpr int NL = 32;
template <class F> void lanes(int w, F&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l); }

// state: [B][2n]; body: [k] canonical bodies (-1 static); T: [k][12] fp64; off: nullptr, [k][3] or [B][k][3] (off_pw) in R
template <class R>
int run_point(const nb2_model_desc* d, int B, const R* state, int k, const int* body, const double* T, const R* off, int off_pw, R* dJ,
              const R* gJ, R* gstate, R* goff) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  std::vector<R> Tn((size_t)k * 12);
  for (size_t i = 0; i < Tn.size(); i++) Tn[i] = (R)T[i];
  const size_t blk = (size_t)6 * n;
  for (int w = 0; w < B; w++) {
    const R* q = state + (size_t)w * 2 * n;
    auto o_of = [&](int e) -> const R* { return off ? off + ((off_pw ? (size_t)w * k : 0) + e) * 3 : nullptr; };
    if (dJ) {
      std::vector<R> ws(nb2::jpd_layout(n).total);
      for (int e = 0; e < k; e++) {
        for (auto& x : ws) x = R(1e30);
        lanes(w, [&](int l) { nb2::jp_zero<R>(M, ws.data(), l, NL); });
        lanes(w, [&](int l) { nb2::jpd_walk<R>(M, q, q + n, body[e], Tn.data() + 12 * e, o_of(e), ws.data(), l); });
        lanes(w, [&](int l) { nb2::jpd_columns<R>(M, body[e], ws.data(), l, NL); });
        for (size_t i = 0; i < blk; i++) dJ[((size_t)w * k + e) * blk + i] = ws[i];
      }
    } else {
      const nb2::JpdbLayout L = nb2::jpdb_layout(M.nb, n);
      std::vector<R> ws(L.total);
      for (auto& x : ws) x = R(1e30);
      lanes(w, [&](int l) { nb2::jpdb_init<R>(M, ws.data(), l, NL); });
      for (int e = 0; e < k; e++) {
        const R* g = gJ + ((size_t)w * k + e) * blk;
        lanes(w, [&](int l) { nb2::jpdb_walk<R>(M, q, q + n, body[e], Tn.data() + 12 * e, o_of(e), ws.data(), l); });
        lanes(w, [&](int l) { nb2::jpdb_terms<R>(M, body[e], g, ws.data(), l, NL); });
        lanes(w, [&](int l) { nb2::jpdb_reduce<R>(M, q, q + n, body[e], ws.data(), goff ? goff + ((size_t)w * k + e) * 3 : nullptr, l); });
      }
      lanes(w, [&](int l) { nb2::jd_store_row<R>(n, ws.data() + L.oGq, gstate + (size_t)w * 2 * n, l, NL); });
    }
  }
  return 0;
}
template <class R>
int run_com(const nb2_model_desc* d, int B, const R* state, int root, const double* wi, R* dJ, const R* gJ, R* gstate, double* gI) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  const bool bwd = dJ == nullptr;
  const nb2::JcdLayout L = nb2::jcd_layout(M.nb, n, bwd);
  std::vector<R> ws(L.total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    const R* q = state + (size_t)w * 2 * n;
    const double* wiw = wi ? wi + w : nullptr;
    if (!bwd) {
      lanes(w, [&](int l) { nb2::jc_init<R>(M, q, root, false, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jc_moments<R>(M, root, wiw, (size_t)B, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jcd_vel<R>(M, q + n, root, wiw, (size_t)B, false, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jcd_columns<R>(M, root, ws.data(), l, NL); });
      for (int i = 0; i < 3 * n; i++) dJ[(size_t)w * 3 * n + i] = ws[L.oCol + i];
    } else {
      lanes(w, [&](int l) { nb2::jcdb_init<R>(M, q, root, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jc_moments<R>(M, root, wiw, (size_t)B, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jcd_vel<R>(M, q + n, root, wiw, (size_t)B, true, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jcdb_terms<R>(M, root, gJ + (size_t)w * 3 * n, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jcdb_prefix<R>(M, root, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jcdb_bodies<R>(M, root, wiw, (size_t)B, ws.data(), gI ? gI + w : nullptr, (size_t)B, l, NL); });
      lanes(w, [&](int l) { nb2::jcdb_reduce<R>(M, q, q + n, root, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jd_store_row<R>(n, ws.data() + L.oGq, gstate + (size_t)w * 2 * n, l, NL); });
    }
  }
  return 0;
}
}  // namespace

extern "C" {
// rows in the arithmetic type (double if fp64, float otherwise).  dJ != NULL: the forward into dJ; else the backward of gJ.
int emul_world_jacobian_deriv(const nb2_model_desc* d, int B, const void* state, int k, const int* body, const double* T, const void* off,
                              int off_pw, void* dJ, const void* gJ, void* gstate, void* goff, int fp64) {
  return fp64 ? run_point<double>(d, B, (const double*)state, k, body, T, (const double*)off, off_pw, (double*)dJ, (const double*)gJ,
                                  (double*)gstate, (double*)goff)
              : run_point<float>(d, B, (const float*)state, k, body, T, (const float*)off, off_pw, (float*)dJ, (const float*)gJ, (float*)gstate,
                                 (float*)goff);
}
int emul_com_jacobian_deriv(const nb2_model_desc* d, int B, const void* state, int root, const double* wi, void* dJ, const void* gJ, void* gstate,
                            double* gI, int fp64) {
  return fp64 ? run_com<double>(d, B, (const double*)state, root, wi, (double*)dJ, (const double*)gJ, (double*)gstate, gI)
              : run_com<float>(d, B, (const float*)state, root, wi, (float*)dJ, (const float*)gJ, (float*)gstate, gI);
}
}
