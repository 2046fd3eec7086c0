// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the world-Jacobian device functions (csrc/nb2_jac.cuh), as k_jac_point_fwd /
// k_jac_point_bwd / k_jac_com_fwd / k_jac_com_bwd run them: one item at a time, its 32 lanes stage by stage (the kernels' __syncwarp
// boundaries), the lanes of odd worlds in reversed order, the working set poisoned before every item.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_jac.cuh"

namespace {
constexpr int NL = 32;
template <class F> void lanes(int w, F&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l); }

// body: [k] canonical bodies (-1 static); T: [k][12] fp64; off: nullptr, [k][3] or [B][k][3] (off_pw) in R
template <class R>
int run_point(const nb2_model_desc* d, int B, const R* pos, int k, const int* body, const double* T, const R* off, int off_pw, R* J,
              const R* gJ, R* gpos, R* goff) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  std::vector<R> Tn((size_t)k * 12);
  for (size_t i = 0; i < Tn.size(); i++) Tn[i] = (R)T[i];
  const size_t blk = (size_t)6 * n;
  for (int w = 0; w < B; w++) {
    const R* q = pos + (size_t)w * n;
    auto o_of = [&](int e) -> const R* { return off ? off + ((off_pw ? (size_t)w * k : 0) + e) * 3 : nullptr; };
    if (J) {
      std::vector<R> ws(nb2::jp_layout(n).total);
      for (int e = 0; e < k; e++) {
        for (auto& x : ws) x = R(1e30);
        lanes(w, [&](int l) { nb2::jp_zero<R>(M, ws.data(), l, NL); });
        lanes(w, [&](int l) { nb2::jp_walk<R>(M, q, body[e], Tn.data() + 12 * e, o_of(e), ws.data(), l); });
        lanes(w, [&](int l) { nb2::jp_columns<R>(M, body[e], ws.data(), l, NL); });
        for (size_t i = 0; i < blk; i++) J[((size_t)w * k + e) * blk + i] = ws[i];
      }
    } else {
      std::vector<R> ws(nb2::jpb_layout(M.nb, n).total);
      for (auto& x : ws) x = R(1e30);
      lanes(w, [&](int l) { nb2::jpb_init<R>(M, ws.data(), l, NL); });
      for (int e = 0; e < k; e++) {
        const R* g = gJ + ((size_t)w * k + e) * blk;
        lanes(w, [&](int l) { nb2::jpb_walk<R>(M, q, body[e], Tn.data() + 12 * e, o_of(e), ws.data(), l); });
        lanes(w, [&](int l) { nb2::jpb_terms<R>(M, body[e], g, ws.data(), l, NL); });
        lanes(w, [&](int l) { nb2::jpb_reduce<R>(M, q, body[e], ws.data(), goff ? goff + ((size_t)w * k + e) * 3 : nullptr, l); });
      }
      lanes(w, [&](int l) { nb2::jpb_store_row<R>(M, ws.data(), gpos + (size_t)w * n, l, NL); });
    }
  }
  return 0;
}
template <class R>
int run_com(const nb2_model_desc* d, int B, const R* pos, int root, const double* wi, R* J, const R* gJ, R* gpos, double* gI) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  const bool bwd = J == nullptr;
  std::vector<R> ws(nb2::jc_layout(M.nb, n, bwd).total);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    const R* q = pos + (size_t)w * n;
    const double* wiw = wi ? wi + w : nullptr;
    lanes(w, [&](int l) { nb2::jc_init<R>(M, q, root, bwd, ws.data(), l, NL); });
    lanes(w, [&](int l) { nb2::jc_moments<R>(M, root, wiw, (size_t)B, ws.data(), l, NL); });
    if (!bwd) {
      lanes(w, [&](int l) { nb2::jc_columns<R>(M, root, ws.data(), l, NL); });
      const int oc = nb2::jc_layout(M.nb, n, false).oCol;
      for (int i = 0; i < 3 * n; i++) J[(size_t)w * 3 * n + i] = ws[oc + i];
    } else {
      lanes(w, [&](int l) { nb2::jcb_terms<R>(M, root, gJ + (size_t)w * 3 * n, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::jcb_sums<R>(M, root, ws.data(), l); });
      lanes(w, [&](int l) { nb2::jcb_grads<R>(M, q, root, ws.data(), gI ? gI + w : nullptr, (size_t)B, l, NL); });
      lanes(w, [&](int l) { nb2::jcb_store_row<R>(M, ws.data(), gpos + (size_t)w * n, l, NL); });
    }
  }
  return 0;
}
}  // namespace

extern "C" {
// rows in the arithmetic type (double if fp64, float otherwise).  J != NULL: the forward into J; else the backward of gJ.
int emul_world_jacobian(const nb2_model_desc* d, int B, const void* pos, int k, const int* body, const double* T, const void* off, int off_pw,
                        void* J, const void* gJ, void* gpos, void* goff, int fp64) {
  return fp64 ? run_point<double>(d, B, (const double*)pos, k, body, T, (const double*)off, off_pw, (double*)J, (const double*)gJ, (double*)gpos,
                                  (double*)goff)
              : run_point<float>(d, B, (const float*)pos, k, body, T, (const float*)off, off_pw, (float*)J, (const float*)gJ, (float*)gpos,
                                 (float*)goff);
}
int emul_com_jacobian(const nb2_model_desc* d, int B, const void* pos, int root, const double* wi, void* J, const void* gJ, void* gpos, double* gI,
                      int fp64) {
  return fp64 ? run_com<double>(d, B, (const double*)pos, root, wi, (double*)J, (const double*)gJ, (double*)gpos, gI)
              : run_com<float>(d, B, (const float*)pos, root, wi, (float*)J, (const float*)gJ, (float*)gpos, gI);
}
}
