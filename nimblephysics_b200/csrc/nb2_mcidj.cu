// Dense-Jacobian kernel of contact inverse dynamics (nb2_multiple_contact_inverse_dynamics_jacobians; DESIGN.md §6s), in a translation
// unit of its own (see nb2_mcidj.h).  The entry is in nb2_kernels.cu.
#include "nb2_mcidj.cuh"
#include "nb2_mcidj.h"

namespace {

// ONE WARP PER WORLD, one world per block (nb2_mcidj.cuh): the ID forward on the model's lane schedule, the contact split on one lane, the
// layer's outputs, then rounds of ST of the n + 6k rows, each swept by one thread and written out by the whole warp.
template <class R, int ST>
__global__ void __launch_bounds__(32)
k_mcidj(const __grid_constant__ Nb2ModelDev<R> M, const __grid_constant__ nb2::McidBodies<R> b, int B, const R* __restrict__ state,
        const R* __restrict__ next_vel, const R* __restrict__ guess, const double* __restrict__ winertia, R* __restrict__ tau,
        R* __restrict__ wrench, R* __restrict__ Tq, R* __restrict__ Tqd, R* __restrict__ Tn, R* __restrict__ Tg, R* __restrict__ Wq,
        R* __restrict__ Wqd, R* __restrict__ Wn, R* __restrict__ Wg) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int lane = threadIdx.x, n = M.ndof, m = 6 * b.k, rows = n + m;
  const size_t w = blockIdx.x, nn = (size_t)n * n, mn = (size_t)m * n, nm = (size_t)n * m, mm = (size_t)m * m;
  const R* s = state + w * 2 * n;
  const R* g = guess ? guess + w * m : nullptr;
  const double* wi = winertia ? winertia + w : nullptr;
  const nb2::McidjRows<R> J{Tq + w * nn, Tqd + w * nn, Tn + w * nn, Tg ? Tg + w * nm : nullptr,
                            Wq + w * mn, Wqd + w * mn, Wn + w * mn, Wg ? Wg + w * mm : nullptr};
  nb2::dj_load<R>(M, ws, s, next_vel + w * n, lane, 32);
  nb2::mcidj_load_guess<R, ST>(M, b.k, ws, g, lane, 32);
  __syncwarp();
#pragma unroll 1
  for (int sg = 1; sg < NB2_ID_FWD_STAGES - 1; sg++) {
    nb2::dj_forward_stage<R, false>(M, ws, lane, sg, wi, (size_t)B);
    __syncwarp();
  }
  if (lane == 0) nb2::mcidj_forward<R, ST>(M, b, ws, s, g != nullptr);
  __syncwarp();
  nb2::mcidj_store_out<R, ST>(M, b.k, ws, tau + w * n, wrench + w * m, lane, 32);
#pragma unroll 1
  for (int r0 = 0; r0 < rows; r0 += ST) {
    const int nrows = min(ST, rows - r0);
    if (lane < nrows) nb2::mcidj_row<R, ST>(M, b, ws, s, g != nullptr, r0 + lane, lane, wi, (size_t)B);
    __syncwarp();
    nb2::mcidj_rows_store<R, ST>(M, b.k, ws, r0, nrows, J, lane, 32);
    __syncwarp();
  }
}

template <class R, int ST>
cudaError_t launch(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, const nb2::McidBodies<R>& b, int B, const McidjArgs& a) {
  cudaError_t e = cudaFuncSetAttribute(k_mcidj<R, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_mcidj<R, ST><<<B, 32, smem, s>>>(M, b, B, (const R*)a.state, (const R*)a.next_vel, (const R*)a.guess, a.wi, (R*)a.tau, (R*)a.wrench,
                                      (R*)a.J[0], (R*)a.J[1], (R*)a.J[2], (R*)a.J[3], (R*)a.J[4], (R*)a.J[5], (R*)a.J[6], (R*)a.J[7]);
  return cudaGetLastError();
}

}  // namespace

int nb2_mcidj_slots(int nb, int n, int nslots, int nfree, int k, size_t word, size_t max_smem, size_t* smem) {
  int want = 4;
  while (want < 32 && want < n + 6 * k) want *= 2;
  for (int st = want; st >= 4; st /= 2) {
    const size_t bytes = (size_t)nb2::mcidj_layout(nb, n, nslots, nfree, k, st).total * word;
    if (bytes <= max_smem) { *smem = bytes; return st; }
  }
  return 0;
}
template <class R>
cudaError_t nb2_mcidj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const McidjArgs& a) {
  nb2::McidBodies<R> b;
  if (nb2::mcid_bodies(M, a.k, a.body, a.point, &b) < 0) return cudaErrorInvalidValue;  // the entry has checked the set
  switch (slots) {
    case 32: return launch<R, 32>(smem, s, M, b, B, a);
    case 16: return launch<R, 16>(smem, s, M, b, B, a);
    case 8: return launch<R, 8>(smem, s, M, b, B, a);
    default: return launch<R, 4>(smem, s, M, b, B, a);
  }
}
template cudaError_t nb2_mcidj_launch<float>(int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const McidjArgs&);
template cudaError_t nb2_mcidj_launch<double>(int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const McidjArgs&);
