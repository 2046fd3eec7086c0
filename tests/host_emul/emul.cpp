// DEVELOPMENT/TEST HARNESS ONLY — compiles the per-world device functions (csrc/nb2_dyn.cuh) as host code so that
// the kernel math can be checked against the oracle in the GPU-less build container (tests/test_host_emul.py).
// Every runner takes an optional per-world canonical inertia table `winertia` (fp64, word-major [10*nb][B] as the *_pw
// entry points take it); NULL = the model's table (tests/test_per_world_mass.py).
// It is never loaded by the nimblephysics_b200 package: the product path has no CPU fallback.
#include <string>
#include <vector>

#include "../../nimblephysics_b200/csrc/nb2_dyn.cuh"
#include "../../nimblephysics_b200/csrc/nb2_host_model.h"

// The emulated "warp" holds a GROUP of up to G worlds (scratch stride G, like the device's 32/lanes worlds per warp) and
// NT virtual threads for the group load / store; the sweep stages run per (world slot, lane).  Lanes of odd worlds run in
// reverse order so that a missing barrier (a cross-lane dependency inside one stage) shows up as a poisoned read.
constexpr int G = 3, NT = 5;
template <class R>
static int run_fwd(const nb2_model_desc* d, int B, const float* state, const float* action, float* next, R* saved, const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::FwdLayout L = nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  std::vector<R> scr((size_t)L.total * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);  // poison: catches reads of never-written scratch
    for (int sg = 0; sg < NB2_FWD_STAGES; sg++) {
      if (sg == 0) { for (int t = NT - 1; t >= 0; t--) nb2::fwd_load<R, G>(M, scr.data(), state + (size_t)g0 * 2 * M.ndof, action + (size_t)g0 * M.na, nw, t, NT); continue; }
      if (sg == NB2_FWD_STAGES - 1) { for (int t = 0; t < NT; t++) nb2::fwd_store<R, G>(M, scr.data(), next + (size_t)g0 * 2 * M.ndof, nw, t, NT); continue; }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::world_forward_stage<R, G>(M, scr.data() + slot, saved ? saved + w : nullptr, (size_t)B, saved != nullptr, lane, sg, nullptr, nullptr,
                                         winertia ? winertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
template <class R>
static int run_bwd(const nb2_model_desc* d, int B, const float* state, const float* action, const R* saved,
                   const float* gnext, float* gstate, float* gaction, float* ginertia, const double* winertia) {
  Nb2ModelDev<R> M; std::string err;
  if (!nb2_fill_model(*d, M, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::BwdLayout L = nb2::bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  std::vector<R> scr((size_t)L.total * G);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int nw = (B - g0 < G) ? B - g0 : G;
    for (auto& x : scr) x = R(1e30);
    for (int sg = 0; sg < NB2_BWD_STAGES; sg++) {
      if (sg == 0) { for (int t = NT - 1; t >= 0; t--) nb2::bwd_load<R, G, false>(M, scr.data(), state + (size_t)g0 * 2 * M.ndof, action + (size_t)g0 * M.na, gnext + (size_t)g0 * 2 * M.ndof, nw, t, NT); continue; }
      if (sg == NB2_BWD_STAGES - 1) {
        for (int t = 0; t < NT; t++)
          nb2::bwd_store<R, G, false>(M, scr.data(), gstate + (size_t)g0 * 2 * M.ndof, gaction + (size_t)g0 * M.na, false, nw, t, NT);
        continue;
      }
      for (int slot = 0; slot < nw; slot++)
        for (int l = 0; l < M.lanes; l++) {
          const int w = g0 + slot, lane = (w & 1) ? M.lanes - 1 - l : l;
          nb2::world_backward_stage<R, G>(M, scr.data() + slot, saved + w, (size_t)B, lane, sg, ginertia ? ginertia + w : nullptr, nullptr, 0, nullptr,
                                          winertia ? winertia + w : nullptr, (size_t)B);
        }
    }
  }
  return 0;
}
// fused forward with the contact stage (fp64), as k_cstep_fwd runs it: ABA sweeps (every lane of the schedule), warp-cooperative
// contact stage on the world's scratch, store.  The saved stream is WORLD-MAJOR (word k of world w at saved[w * words + k]).
static nb2::cw::Dims contact_dims(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, int MC, int MR) {
  return nb2::cw::make_dims(M.nb, M.ndof, M.nfree, MC, MR, C.ncb, C.max_chain_dofs);
}
static int run_fwd_contact(const nb2_model_desc* d, int B, const float* state, const float* action, float* next, double* saved,
                           double* x_lcp, int* m_lcp, int* labels, int* status, int* nc, float* cinfo, double* crec, int small_mc, int reverse,
                           const double* winertia) {
  Nb2ModelDev<double> M; Nb2ContactDev C; std::string err;
  if (!nb2_fill_model(*d, M, err) || !nb2_fill_contact(*d, C, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::FwdLayout L = nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int words = nb2_saved_words(M.nb, M.ndof, M.nfree);
  const nb2::cw::Dims ds = contact_dims(M, C, small_mc, 3 * small_mc), db = contact_dims(M, C, NB2_MAX_CONTACTS, NB2_MAX_ROWS);
  std::vector<double> scr(L.total), wss(nb2::cw::ws_doubles(ds)), wsb(nb2::cw::ws_doubles(db));
  const size_t recd = nb2::cw::record_doubles(M.ndof);
  for (int w = 0; w < B; w++) {
    nb2::cw::cw_host_reverse() = reverse && (w & 1);
    for (auto& x : scr) x = 1e30;
    for (auto& x : wss) x = 1e30;
    for (auto& x : wsb) x = 1e30;
    const float* st = state + (size_t)w * 2 * M.ndof;
    nb2::cw::Ws ws0 = nb2::cw::carve(wss.data(), ds);
    nb2::fwd_load<double, 1>(M, scr.data(), st, action + (size_t)w * M.na, 1, 0, 1);
    for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++)
      for (int l = 0; l < M.lanes; l++) {
        const int lane = (w & 1) ? M.lanes - 1 - l : l;
        nb2::world_forward_stage<double, 1>(M, scr.data(), saved + (size_t)w * words, 1, true, lane, sg, nullptr, ws0.Iinv,
                                            winertia ? winertia + w : nullptr, (size_t)B);
      }
    nb2::cw::FwdIO io;
    io.x_io = x_lcp + (size_t)w * NB2_MAX_ROWS; io.m_io = m_lcp + w; io.labels = labels + (size_t)w * NB2_MAX_ROWS; io.status = status + w;
    io.nc = nc + w; io.cinfo = cinfo ? cinfo + (size_t)w * NB2_MAX_CONTACTS * 10 : nullptr; io.rec = crec ? crec + (size_t)w * recd : nullptr;
    int pc = 0; nb2::cw::BigPool pool{&pc, wsb.data(), wsb.size(), 1};
    nb2::cw::contact_forward(M, C, scr.data(), st, &ws0, ds, pool, db, ws0.Iinv, io);
    nb2::fwd_store<double, 1>(M, scr.data(), next + (size_t)w * 2 * M.ndof, 1, 0, 1);
  }
  nb2::cw::cw_host_reverse() = 0;
  return 0;
}
// fused backward with the contact stage, as k_cstep_bwd runs it: lambda sweeps (B1, B2) along the schedule, the warp-cooperative
// contact adjoint, reverse RNEA sweep (B3) + assembly with the contact injections, store.
static int run_bwd_contact(const nb2_model_desc* d, int B, const float* state, const float* action, const double* saved,
                           const double* crec, const float* gnext, float* gstate, float* gaction, float* ginertia, int* bstatus, int small_mc, int reverse,
                           const double* winertia) {
  Nb2ModelDev<double> M; Nb2ContactDev C; std::string err;
  if (!nb2_fill_model(*d, M, err) || !nb2_fill_contact(*d, C, err)) { fprintf(stderr, "emul: %s\n", err.c_str()); return -1; }
  nb2::BwdLayout L = nb2::bwd_layout(M.nb, M.ndof, M.nslots, M.nfree, 42);
  const int words = nb2_saved_words(M.nb, M.ndof, M.nfree);
  const nb2::cw::Dims ds = nb2::cw::make_dims(M.nb, M.ndof, M.nfree, small_mc, 3 * small_mc, C.ncb, C.max_chain_dofs, 1);
  const nb2::cw::Dims db = nb2::cw::make_dims(M.nb, M.ndof, M.nfree, NB2_MAX_CONTACTS, NB2_MAX_ROWS, C.ncb, C.max_chain_dofs, 1);
  std::vector<double> scr(L.total), wss(nb2::cw::ws_doubles(ds)), wsb(nb2::cw::ws_doubles(db));
  const size_t recd = nb2::cw::record_doubles(M.ndof);
  for (int w = 0; w < B; w++) {
    nb2::cw::cw_host_reverse() = reverse && (w & 1);
    for (auto& x : scr) x = 1e30;
    for (auto& x : wss) x = 1e30;
    for (auto& x : wsb) x = 1e30;
    const float* st = state + (size_t)w * 2 * M.ndof;
    const double* sv = saved + (size_t)w * words;
    nb2::bwd_load<double, 1, true>(M, scr.data(), st, action + (size_t)w * M.na, gnext + (size_t)w * 2 * M.ndof, 1, 0, 1);
    nb2::BwdContactData<1> cd; cd.active = 0; cd.error = 0; cd.inj_of_body = nullptr;
    nb2::cw::Ws wsd = nb2::cw::carve(wss.data(), ds);
    nb2::BwdContactData<1> c2 = cd;
    float* gI = ginertia ? ginertia + w : nullptr;
    for (int it = 0; it < NB2_CBWD_ITERS; it++) {  // the stage order of k_cstep_bwd
      const auto [sg, second] = nb2::cbwd_iter(it);
      if (it == 4) {
        int pc = 0; nb2::cw::BigPool pool{&pc, wsb.data(), wsb.size(), 1};
        cd = nb2::cw::contact_backward<true>(M, C, st, sv, &wsd, ds, pool, db, crec + (size_t)w * recd, scr.data(), L.oLam, L.oBody);
      }
      if (second && !cd.bounce) continue;
      if (it == 6) c2 = nb2::cw::bounce_pass2_begin(M, C, wsd, cd, scr.data(), L.oLam, L.oBody);
      if (it == 8 && cd.bounce) nb2::cw::bounce_pass2_end(M, wsd, scr.data(), L.oLam);
      for (int l = 0; l < M.lanes; l++) {
        const int lane = (w & 1) ? M.lanes - 1 - l : l;
        nb2::world_backward_stage<double, 1, true>(M, scr.data(), sv, 1, lane, sg, gI, nullptr, (size_t)B, second ? &c2 : &cd,
                                                   winertia ? winertia + w : nullptr, (size_t)B);
      }
    }
    nb2::bwd_store<double, 1, true>(M, scr.data(), gstate + (size_t)w * 2 * M.ndof, gaction + (size_t)w * M.na, cd.error != 0, 1, 0, 1);
    if (bstatus) bstatus[w] = cd.error;
  }
  nb2::cw::cw_host_reverse() = 0;
  return 0;
}
// warp-cooperative solve chain (csrc/nb2_cw.cuh) on a caller-supplied boxed LCP; reverse != 0 runs every CW_FOR backwards
static int run_cw_chain(int m, const double* A, const double* b, const double* lo, const double* hi, const int* fi, const double* x0, int have_x0,
                        double cfm, double* x_out, int* mapping_out, int reverse) {
  nb2::cw::cw_host_reverse() = reverse;
  const nb2::cw::Dims d = nb2::cw::make_dims(1, 1, 0, (m + 2) / 3 + 1, m > 3 ? m : 3, 1, 1);
  std::vector<double> wsb(nb2::cw::ws_doubles(d), 1e30);
  const nb2::cw::Ws ws = nb2::cw::carve(wsb.data(), d);
  const int ld = m | 1;
  for (int i = 0; i < m; i++) for (int j = 0; j < m; j++) ws.A[i * ld + j] = A[i * m + j];
  for (int i = 0; i < m; i++) { ws.b[i] = b[i]; ws.lo[i] = lo[i]; ws.hi[i] = hi[i]; ws.findex[i] = fi[i]; }
  const int status = nb2::cw::lcp_chain(m, ws, ws, cfm, have_x0 ? x0 : nullptr);
  for (int i = 0; i < m; i++) { x_out[i] = ws.x[i]; mapping_out[i] = ws.mapping[i]; }
  nb2::cw::cw_host_reverse() = 0;
  return status;
}
extern "C" {
int emul_cw_solve_chain(int m, const double* A, const double* b, const double* lo, const double* hi, const int* fi, const double* x0, int have_x0,
                        double cfm, double* x_out, int* mapping_out, int reverse) {
  return run_cw_chain(m, A, b, lo, hi, fi, x0, have_x0, cfm, x_out, mapping_out, reverse);
}
int emul_forward_contact(const nb2_model_desc* d, int B, const float* state, const float* action, float* next, double* saved,
                         double* x_lcp, int* m_lcp, int* labels, int* status, int* nc, float* cinfo, double* crec, int small_mc, int reverse,
                         const double* winertia) {
  return run_fwd_contact(d, B, state, action, next, saved, x_lcp, m_lcp, labels, status, nc, cinfo, crec, small_mc, reverse, winertia);
}
int emul_backward_contact(const nb2_model_desc* d, int B, const float* state, const float* action, const double* saved,
                          const double* crec, const float* gnext, float* gstate, float* gaction, float* ginertia, int* bstatus, int small_mc, int reverse,
                          const double* winertia) {
  return run_bwd_contact(d, B, state, action, saved, crec, gnext, gstate, gaction, ginertia, bstatus, small_mc, reverse, winertia);
}
int emul_contact_rec_doubles(const nb2_model_desc* d) { return (int)nb2::cw::record_doubles(d->ndof); }
int emul_saved_words(const nb2_model_desc* d) {
  int nfree = 0; for (int i = 0; i < d->nb; i++) nfree += d->jtype[i] == NB2_JT_FREE;
  return nb2_saved_words(d->nb, d->ndof, nfree);
}
int emul_forward(const nb2_model_desc* d, int B, const float* state, const float* action, float* next, void* saved, int fp64, const double* winertia) {
  return fp64 ? run_fwd<double>(d, B, state, action, next, (double*)saved, winertia) : run_fwd<float>(d, B, state, action, next, (float*)saved, winertia);
}
int emul_backward(const nb2_model_desc* d, int B, const float* state, const float* action, const void* saved,
                  const float* gnext, float* gstate, float* gaction, int fp64, float* ginertia, const double* winertia) {
  return fp64 ? run_bwd<double>(d, B, state, action, (const double*)saved, gnext, gstate, gaction, ginertia, winertia)
              : run_bwd<float>(d, B, state, action, (const float*)saved, gnext, gstate, gaction, ginertia, winertia);
}
}
