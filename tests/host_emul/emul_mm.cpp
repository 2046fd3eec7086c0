// DEVELOPMENT/TEST HARNESS ONLY — the host emulation of the mass-matrix device functions (csrc/nb2_mm.cuh), as k_mm_fwd / k_minv_fwd /
// k_mm_bwd run them: one world at a time, its 32 lanes stage by stage (the kernels' __syncwarp boundaries), the lanes of odd worlds in
// reversed order, the working set poisoned before every world.
#include "emul.cpp"
#include "../../nimblephysics_b200/csrc/nb2_mm.cuh"

namespace {
constexpr int NL = 32;
template <class F> void lanes(int w, F&& f) { for (int l = 0; l < NL; l++) f((w & 1) ? NL - 1 - l : l); }

// which: 0 M, 1 M^-1
template <class R>
int run_mm_fwd(const nb2_model_desc* d, int which, int B, const R* pos, const double* wi, R* out) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  const size_t words = which == 0 ? nb2::mm_layout(M.nb, n).total : nb2::minv_layout(M.nb, n, M.nslots, M.nfree, NL).total;
  const int oMat = which == 0 ? nb2::mm_layout(M.nb, n).oMat : nb2::minv_layout(M.nb, n, M.nslots, M.nfree, NL).oMat;
  std::vector<R> ws(words);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    const R* q = pos + (size_t)w * n;
    const double* wiw = wi ? wi + w : nullptr;
    if (which == 0) {
      lanes(w, [&](int l) { nb2::crba_init<R>(M, q, wiw, (size_t)B, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::crba_composite<R>(M, ws.data(), l); });
      lanes(w, [&](int l) { nb2::crba_columns<R>(M, ws.data(), l, NL); });
    } else {
      lanes(w, [&](int l) { nb2::minv_init<R>(M, q, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::minv_articulated<R>(M, ws.data(), wiw, (size_t)B, l, NL); });
      lanes(w, [&](int l) { nb2::minv_columns<R>(M, ws.data(), l, NL); });
    }
    for (int k = 0; k < n * n; k++) out[(size_t)w * n * n + k] = ws[oMat + k];
  }
  return 0;
}
// minv == nullptr: the M backward of grad; else the M^-1 backward
template <class R>
int run_mm_bwd(const nb2_model_desc* d, int B, const R* pos, const double* wi, const R* grad, const R* minv, R* gpos, double* gI) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  const int n = M.ndof;
  std::vector<R> ws(nb2::mminvb_words(M.nb, n, NL)), tmp((size_t)n * n);
  for (int w = 0; w < B; w++) {
    for (auto& x : ws) x = R(1e30);
    for (auto& x : tmp) x = R(1e30);
    const R* q = pos + (size_t)w * n;
    const double* wiw = wi ? wi + w : nullptr;
    double* gIw = gI ? gI + w : nullptr;
    if (minv) {
      lanes(w, [&](int l) { nb2::mminvb_load<R>(M, minv + (size_t)w * n * n, grad + (size_t)w * n * n, ws.data(), l, NL); });
      lanes(w, [&](int l) { nb2::mminvb_left<R>(M, ws.data(), tmp.data(), l, NL); });
      lanes(w, [&](int l) { nb2::mminvb_right<R>(M, ws.data(), tmp.data(), l, NL); });
    }
    lanes(w, [&](int l) { nb2::mmb_init<R>(M, q, minv ? nullptr : grad + (size_t)w * n * n, ws.data(), l, NL); });
    lanes(w, [&](int l) { nb2::mmb_root_frames<R>(M, ws.data(), l, NL); });
    for (int b = 0; b < M.nb; b++) {
      lanes(w, [&](int l) { nb2::mmb_body_chain<R>(M, ws.data(), b, l, NL); });
      lanes(w, [&](int l) { nb2::mmb_body_columns<R>(M, ws.data(), b, l, NL); });
      lanes(w, [&](int l) { nb2::mmb_body_forces<R>(M, ws.data(), b, wiw, (size_t)B, l, NL); });
      lanes(w, [&](int l) { nb2::mmb_body_reduce<R>(M, ws.data(), b, gIw, (size_t)B, l, NL); });
    }
    lanes(w, [&](int l) { nb2::mmb_free_q<R>(M, q, ws.data(), l, NL); });
    lanes(w, [&](int l) { nb2::mmb_store_row<R>(M, ws.data(), gpos + (size_t)w * n, l, NL); });
  }
  return 0;
}
}  // namespace

extern "C" {
// rows in the arithmetic type (double if fp64, float otherwise); wi: fp64 [10*nb][B] or NULL; gI: fp64 [10*nb][B] or NULL
int emul_mass_matrix(const nb2_model_desc* d, int inverse, int B, const void* pos, const double* wi, void* out, int fp64) {
  return fp64 ? run_mm_fwd<double>(d, inverse, B, (const double*)pos, wi, (double*)out)
              : run_mm_fwd<float>(d, inverse, B, (const float*)pos, wi, (float*)out);
}
int emul_mass_matrix_backward(const nb2_model_desc* d, int B, const void* pos, const double* wi, const void* grad, const void* minv, void* gpos,
                              double* gI, int fp64) {
  return fp64 ? run_mm_bwd<double>(d, B, (const double*)pos, wi, (const double*)grad, (const double*)minv, (double*)gpos, gI)
              : run_mm_bwd<float>(d, B, (const float*)pos, wi, (const float*)grad, (const float*)minv, (float*)gpos, gI);
}
}
