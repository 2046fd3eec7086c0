// Dense Jacobians of contact inverse dynamics, one to NB2_MAX_CONTACT_BODIES bodies, batched (DESIGN.md §6s):
//   (tau, w_1..w_k) = MCID(q, qdot, v'; g)   ->   d[tau; w]/dq, d[tau; w]/dqdot, d[tau; w]/dv' (v' held fixed in the first two), d[tau; w]/dg
// Row i of each block is the layer's vector-Jacobian product with the seed e_i on output i (n rows on tau, then 6k on the wrenches), formed
// exactly as nb2_multiple_contact_inverse_dynamics_backward forms it: mcid_vjp (cid_vjp for one body) turns the seed into the inverse-
// dynamics seed and dL/dg, the ID backward stages sweep that seed, and mcid_vjp / cid_vjp then ADD their direct q-term to the q row.
//
// ONE WARP PER WORLD, the k_dj shape (nb2_djac.cuh).  The world's working set sits in the block's shared memory (arithmetic type R):
//   dj_layout(ST) words        the ID forward scratch, the saved stream and ST slots of the ID backward's scratch, [word][slot]
//   wrench  6k words           the forward's wrenches (mcid_forward / cid_forward, run in place on the tau words of the forward scratch)
//   guess   6k words           the guesses (read only with k >= 2 and a guess)
//   ST row scratches, contiguous, cWords each:  g [n + 6k] (the seed e_row on [tau; w]), seed [n] (the ID backward's seed), gg [6k]
//                              (dL/dg), gq [n] (the q row, for the direct term): mcid_vjp takes contiguous vectors.
// Every function below is one stage: lanes exchange data only between stages (the kernel puts a __syncwarp there), so a host build can
// run a stage's lanes in any order.
#pragma once
#include "nb2_djac.cuh"

namespace nb2 {

struct McidjLayout { DjLayout D; int oW, oG, oC, cWords, total; };
NB2_HD McidjLayout mcidj_layout(int nb, int n, int nslots, int nfree, int k, int st) {
  McidjLayout L;
  L.D = dj_layout(nb, n, nslots, nfree, false, st);
  const int m = 6 * k;
  L.oW = L.D.total;
  L.oG = L.oW + m;
  L.oC = L.oG + m;
  L.cWords = 3 * n + 2 * m;
  L.total = L.oC + st * L.cWords;
  return L;
}
template <class R> NB2_HD McidjLayout mcidj_layout(const Nb2ModelDev<R>& M, int k, int st) { return mcidj_layout(M.nb, M.ndof, M.nslots, M.nfree, k, st); }

// the world's blocks: T_* [n][n] (T_g [n][6k]) for the tau rows, W_* [6k][n] (W_g [6k][6k]) for the wrench rows; T_g / W_g may be nullptr
template <class R> struct McidjRows { R *Tq, *Tqd, *Tn, *Tg, *Wq, *Wqd, *Wn, *Wg; };

// stage 0 (with dj_load), lanes over 6k: the world's guesses (nullptr: none) into their shared words
template <class R, int ST> NB2_HD void mcidj_load_guess(const Nb2ModelDev<R>& M, int k, R* ws, const R* guess, int lane, int nl) {
  if (!guess) return;
  const McidjLayout L = mcidj_layout(M, k, ST);
  for (int d = lane; d < 6 * k; d += nl) ws[L.oG + d] = guess[d];
}
// after the ID forward stages, one lane: the contact split, in place on tau_ID (guessed: the guesses were loaded).  state: the world's row.
template <class R, int ST> NB2_HD void mcidj_forward(const Nb2ModelDev<R>& M, const McidBodies<R>& b, R* ws, const R* state, bool guessed) {
  const McidjLayout L = mcidj_layout(M, b.k, ST);
  R* tau = ws + fwd_layout(M.nb, M.ndof, M.nslots, M.nfree).oAct;
  if (b.k == 1) cid_forward<R>(M, b.c[0], state, tau, ws + L.oW);
  else mcid_forward<R>(M, b, state, guessed ? ws + L.oG : nullptr, tau, ws + L.oW);
}
// lanes over dofs and wrench entries: the layer's outputs
template <class R, int ST> NB2_HD void mcidj_store_out(const Nb2ModelDev<R>& M, int k, const R* ws, R* tau, R* wrench, int lane, int nl) {
  const McidjLayout L = mcidj_layout(M, k, ST);
  dj_store_out<R>(M, ws, tau, lane, nl);
  for (int d = lane; d < 6 * k; d += nl) wrench[d] = ws[L.oW + d];
}

// row `row` (< n + 6k) on slot t: the contact VJP's seed, the ID backward stages over the schedule's lanes in order (as dj_row), then the
// contact VJP's direct q-term added to the q row.  state: the world's [q ; qdot] row.
template <class R, int ST>
NB2_HD void mcidj_row(const Nb2ModelDev<R>& M, const McidBodies<R>& b, R* ws, const R* state, bool guessed, int row, int t, const double* wi,
                      size_t wiB) {
  const McidjLayout L = mcidj_layout(M, b.k, ST);
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof, m = 6 * b.k;
  R* rb = ws + L.D.oB + t;
  const R* sv = ws + L.D.oS;
  R* g = ws + L.oC + (size_t)t * L.cWords;
  R *seed = g + n + m, *gg = seed + n, *gq = gg + m;
  const R* wr = ws + L.oW;
  const R* gs = guessed ? ws + L.oG : nullptr;
  for (int d = 0; d < n + m; d++) g[d] = (d == row) ? R(1) : R(0);
  if (b.k == 1) cid_vjp<R>(M, b.c[0], state, wr, g, g + n, seed, nullptr);
  else mcid_vjp<R>(M, b, state, wr, gs, g, g + n, seed, gg, nullptr);
  for (int d = 0; d < 2 * n; d++) rb[(size_t)(BL.oSt + d) * ST] = state[d];
  for (int d = 0; d < n; d++) rb[(size_t)(BL.oLam + d) * ST] = seed[d];
  for (int sg = 1; sg < NB2_ID_BWD_STAGES - 1; sg++)
    for (int l = 0; l < M.lanes; l++) id_backward_stage<R, ST>(M, rb, sv, 1, l, sg, nullptr, wi, wiB, nullptr, 0);
  for (int d = 0; d < n; d++) gq[d] = rb[(size_t)(BL.oQb + d) * ST];
  if (b.k == 1) cid_vjp<R>(M, b.c[0], state, wr, g, g + n, nullptr, gq);
  else mcid_vjp<R>(M, b, state, wr, gs, g, g + n, nullptr, nullptr, gq);
}
// lanes over the entries of rows r0 .. r0 + nrows - 1, slot-fastest (as dj_rows_store): row r < n goes to the T blocks, row n + i to the
// W blocks.  The q entries come from the slot's gq (ID backward + direct term), the others from the ID backward's scratch; with one body
// the guess blocks are zero (the guess is not read).
template <class R, int ST>
NB2_HD void mcidj_rows_store(const Nb2ModelDev<R>& M, int k, const R* ws, int r0, int nrows, const McidjRows<R>& J, int lane, int nl) {
  const McidjLayout L = mcidj_layout(M, k, ST);
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof, m = 6 * k;
  for (int idx = lane; idx < nrows * n; idx += nl) {
    const int j = idx / nrows, t = idx - j * nrows, r = r0 + t;
    const R* rb = ws + L.D.oB + t;
    const R* gq = ws + L.oC + (size_t)t * L.cWords + 2 * n + 2 * m;
    const bool tr = r < n;
    const size_t e = (size_t)(tr ? r : r - n) * n + j;
    (tr ? J.Tq : J.Wq)[e] = gq[j];
    (tr ? J.Tqd : J.Wqd)[e] = rb[(size_t)(BL.oVb + j) * ST];
    (tr ? J.Tn : J.Wn)[e] = rb[(size_t)(BL.oGQ + j) * ST];
  }
  if (!J.Tg && !J.Wg) return;
  for (int idx = lane; idx < nrows * m; idx += nl) {
    const int j = idx / nrows, t = idx - j * nrows, r = r0 + t;
    const R v = k == 1 ? R(0) : ws[L.oC + (size_t)t * L.cWords + 2 * n + m + j];
    R* dst = r < n ? J.Tg : J.Wg;
    if (dst) dst[(size_t)(r < n ? r : r - n) * m + j] = v;
  }
}

}  // namespace nb2
