// Dense Jacobians of contact-free inverse and forward dynamics, batched (DESIGN.md §6l):
//   ID:  tau = ID(q, qdot, v')           ->  dtau/dq, dtau/dqdot, dtau/dv'       (v' held fixed in the first two)
//   FD:  qdd = FD(q, qdot, tau)          ->  dqdd/dq, dqdd/dqdot, dqdd/dtau
// J[i][j] = d out_i / d in_j.  Row i of each triple is the vector-Jacobian product of the layer with the seed e_i, so the rows come from
// the existing backward sweeps (id_backward_stage / fd_backward_stage) seeded with the identity, on ONE forward and ONE saved stream.
//
// ONE WARP PER WORLD.  The world's working set sits in the block's shared memory (arithmetic type R):
//   forward scratch  fwd_layout words, stride 1                 (the step's / ID's forward passes, lanes of the model's schedule)
//   saved stream     nb2_saved_words, stride 1                  (what the backward sweeps read: every row reads the same words)
//   row scratch      ST slots of the backward's scratch, [word][slot]  (thread t < ST sweeps row r0 + t of the round starting at r0)
// The rows of one round run the same model-only control flow on different seeds, so a warp issues them as one instruction stream.
// Every function below is one stage: lanes exchange data only between stages (the kernels put a __syncwarp there), so a host build can
// run a stage's lanes in any order.
#pragma once
#include "nb2_dyn.cuh"

namespace nb2 {

struct DjLayout { int oF, oS, oB, rowWords, total; };  // total: words of the whole working set with ST row slots
NB2_HD DjLayout dj_layout(int nb, int n, int nslots, int nfree, bool fd, int st) {
  DjLayout L;
  L.oF = 0;
  L.oS = fwd_layout(nb, n, nslots, nfree).total;
  L.oB = L.oS + nb2_saved_words(nb, n, nfree);
  L.rowWords = fd ? bwd_layout(nb, n, nslots, nfree).total : id_bwd_words(nb, n, nslots, nfree);
  L.total = L.oB + st * L.rowWords;
  return L;
}
template <class R> NB2_HD DjLayout dj_layout(const Nb2ModelDev<R>& M, bool fd, int st) { return dj_layout(M.nb, M.ndof, M.nslots, M.nfree, fd, st); }

// stage 0, lanes over dofs: q, qdot and the second input x (ID: v', FD: tau) into the forward scratch
template <class R> NB2_HD void dj_load(const Nb2ModelDev<R>& M, R* ws, const R* state, const R* x, int lane, int nl) {
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof;
  for (int d = lane; d < n; d += nl) {
    ws[F.oQ + d] = state[d];
    ws[F.oV + d] = state[n + d];
    ws[F.oAct + d] = x[d];
  }
}
// forward stages 1 .. dj_fwd_stages() - 2 on lane `lane` of the model's schedule (lanes >= M.lanes idle): the ID / FD forward passes, which
// leave tau / qdd in the action words and write the saved stream.  FD needs M with an identity action map (fd_identity_actions).
template <bool FD> NB2_HD constexpr int dj_fwd_stages() { return FD ? NB2_FWD_STAGES : NB2_ID_FWD_STAGES; }
template <class R, bool FD>
NB2_HD void dj_forward_stage(const Nb2ModelDev<R>& M, R* ws, int lane, int stage, const double* wi, size_t wiB) {
  if (lane >= M.lanes) return;
  const DjLayout L = dj_layout(M, FD, 0);
  if (FD) world_forward_stage<R, 1, true>(M, ws + L.oF, ws + L.oS, 1, true, lane, stage, nullptr, nullptr, wi, wiB);
  else id_forward_stage<R, 1>(M, ws + L.oF, ws + L.oS, 1, true, lane, stage, nullptr, wi, wiB);
}
// lanes over dofs: the layer's own output (tau or qdd)
template <class R> NB2_HD void dj_store_out(const Nb2ModelDev<R>& M, const R* ws, R* out, int lane, int nl) {
  const FwdLayout F = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  for (int d = lane; d < M.ndof; d += nl) out[d] = ws[F.oAct + d];
}

// row sweep of slot t (row r0 + t < n): the backward's group load with the seed e_row, then every backward stage over the schedule's lanes
// in order (the slot's scratch is its own, so no barrier is needed inside).  state: the world's [q ; qdot] row.
template <class R, int ST, bool FD>
NB2_HD void dj_row(const Nb2ModelDev<R>& M, R* ws, const R* state, int row, int t, const double* wi, size_t wiB) {
  const DjLayout L = dj_layout(M, FD, ST);
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof, seed = FD ? BL.oGV : BL.oLam;
  R* rb = ws + L.oB + t;
  const R* sv = ws + L.oS;
  for (int d = 0; d < 2 * n; d++) rb[(size_t)(BL.oSt + d) * ST] = state[d];
  for (int d = 0; d < n; d++) rb[(size_t)(seed + d) * ST] = (d == row) ? R(1) : R(0);
  constexpr int stages = FD ? NB2_BWD_STAGES : NB2_ID_BWD_STAGES;
  for (int sg = 1; sg < stages - 1; sg++)
    for (int l = 0; l < M.lanes; l++) {
      if (FD) fd_backward_stage<R, ST>(M, rb, sv, 1, l, sg, nullptr, wi, wiB, nullptr, 0);
      else id_backward_stage<R, ST>(M, rb, sv, 1, l, sg, nullptr, wi, wiB, nullptr, 0);
    }
}
// lanes over the entries of rows r0 .. r0 + nrows - 1 of the world's three n x n blocks (J1 = d/dq, J2 = d/dqdot, J3 = d/dv' or d/dtau),
// slot-fastest so that the scratch reads of a warp fall in distinct banks
template <class R, int ST, bool FD>
NB2_HD void dj_rows_store(const Nb2ModelDev<R>& M, const R* ws, int r0, int nrows, R* J1, R* J2, R* J3, int lane, int nl) {
  const DjLayout L = dj_layout(M, FD, ST);
  const BwdLayout BL = bwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof, o3 = FD ? BL.oLam : BL.oGQ;
  for (int idx = lane; idx < nrows * n; idx += nl) {
    const int j = idx / nrows, t = idx - j * nrows;
    const R* rb = ws + L.oB + t;
    const size_t e = (size_t)(r0 + t) * n + j;
    J1[e] = rb[(size_t)(BL.oQb + j) * ST];
    J2[e] = rb[(size_t)(BL.oVb + j) * ST];
    J3[e] = rb[(size_t)(o3 + j) * ST];
  }
}

}  // namespace nb2
