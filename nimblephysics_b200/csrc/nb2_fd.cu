// Forward-dynamics kernels of libnb2.so (nb2_forward_dynamics_batch / _backward, nb2_forward_dynamics; DESIGN.md §6k), in a translation
// unit of their own (see nb2_fd.h).  The launch shape is chosen in nb2_kernels.cu.
#include "nb2_coop.cuh"
#include "nb2_fd.h"

namespace {

// ---- forward dynamics (nb2_forward_dynamics_batch / _backward, nb2_forward_dynamics): the group shape of the inverse-dynamics kernels, the step's
// passes and stages.  M is the model with an identity action map (fd_identity_actions): tau is per dof.  q and qdot are read through a row
// pointer and a row stride each, so state rows [q ; qdot] and separate position / velocity arrays are read in place.
template <class R, int K, int W>
__global__ void __launch_bounds__(GroupShape<K, W>::MAX_THREADS)
k_fd_fwd(const __grid_constant__ Nb2ModelDev<R> M, int B, const R* __restrict__ q, int qs, const R* __restrict__ v, int vs, const R* __restrict__ tau,
         R* __restrict__ qdd, R* __restrict__ saved, int words, const double* __restrict__ winertia) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  constexpr int ST = GroupShape<K, W>::ST, NT = GroupShape<K, W>::THREADS;
  const GroupPos<K, W> gp(B);
  const int nworlds = gp.nworlds;
  const bool valid = gp.valid();
  const size_t wg = nworlds > 0 ? gp.g0 : 0, w = wg + (valid ? gp.slot : 0);
  R* scr0 = reinterpret_cast<R*>(nb2_smem) + (size_t)gp.gb * words * ST;
  R* scr = scr0 + gp.slot;
  R* sv = saved ? saved + w : nullptr;
  const double* wi = winertia ? winertia + w : nullptr;
  constexpr unsigned sync_mask = (K > 1) ? NB2_FWD_SYNC_MASK : NB2_FWD_SYNC_MASK_1LANE;
#pragma unroll 1
  for (int sg = 0; sg < NB2_FWD_STAGES; sg++) {
    if (sg == 0) {
      if (nworlds > 0) nb2::fd_load<R, ST>(M, scr0, q + wg * qs, (size_t)qs, v + wg * vs, (size_t)vs, tau + wg * M.ndof, nworlds, gp.tid, NT);
    } else if (sg == NB2_FWD_STAGES - 1) { if (nworlds > 0) nb2::fd_store<R, ST>(M, scr0, qdd + wg * M.ndof, nworlds, gp.tid, NT); }
    else if (valid) nb2::world_forward_stage<R, ST, true>(M, scr, sv, (size_t)B, saved != nullptr, gp.lane, sg, nullptr, nullptr, wi, (size_t)B);
    if ((sync_mask >> sg) & 1u) group_sync<K>();
  }
}

template <class R, int K, int W>
__global__ void __launch_bounds__(GroupShape<K, W>::MAX_THREADS)
k_fd_bwd(const __grid_constant__ Nb2ModelDev<R> M, int B, const R* __restrict__ state, const R* __restrict__ saved, const R* __restrict__ gqdd,
         R* __restrict__ gstate, R* __restrict__ gtau, double* __restrict__ ginertia, int words, const double* __restrict__ winertia) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  constexpr int ST = GroupShape<K, W>::ST, NT = GroupShape<K, W>::THREADS;
  const GroupPos<K, W> gp(B);
  const int nworlds = gp.nworlds;
  const bool valid = gp.valid();
  const size_t wg = nworlds > 0 ? gp.g0 : 0, w = wg + (valid ? gp.slot : 0);
  R* scr0 = reinterpret_cast<R*>(nb2_smem) + (size_t)gp.gb * words * ST;
  R* scr = scr0 + gp.slot;
  const double* wi = winertia ? winertia + w : nullptr;
  double* gI = ginertia ? ginertia + w : nullptr;
  constexpr unsigned sync_mask = (K > 1) ? NB2_BWD_SYNC_MASK : NB2_BWD_SYNC_MASK_1LANE;
#pragma unroll 1
  for (int sg = 0; sg < NB2_BWD_STAGES; sg++) {
    if (sg == 0) { if (nworlds > 0) nb2::fd_bwd_load<R, ST>(M, scr0, state + wg * 2 * M.ndof, gqdd + wg * M.ndof, nworlds, gp.tid, NT); }
    else if (sg == NB2_BWD_STAGES - 1) {
      if (nworlds > 0) nb2::fd_bwd_store<R, ST>(M, scr0, gstate + wg * 2 * M.ndof, gtau + wg * M.ndof, nworlds, gp.tid, NT);
    } else if (valid) nb2::fd_backward_stage<R, ST>(M, scr, saved + w, (size_t)B, gp.lane, sg, nullptr, wi, (size_t)B, gI, (size_t)B);
    if ((sync_mask >> sg) & 1u) group_sync<K>();
  }
}

// The legacy entry's path for a model whose working set fits no schedule's shared memory (a long chain in fp64): one thread per world, the
// same stages with the world's scratch in global memory (stride 1), every lane of the schedule swept in turn by that thread.
__global__ void __launch_bounds__(64)
k_fd_fwd_global(const __grid_constant__ Nb2ModelDev<double> M, int B, int words, const double* __restrict__ q, int qs, const double* __restrict__ v,
                int vs, const double* __restrict__ tau, double* __restrict__ qdd, double* __restrict__ scratch) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= B) return;
  double* scr = scratch + (size_t)w * words;
  nb2::fd_load<double, 1>(M, scr, q + (size_t)w * qs, (size_t)qs, v + (size_t)w * vs, (size_t)vs, tau + (size_t)w * M.ndof, 1, 0, 1);
  for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++)
    for (int lane = 0; lane < M.lanes; lane++) nb2::world_forward_stage<double, 1, true>(M, scr, nullptr, 1, false, lane, sg);
  nb2::fd_store<double, 1>(M, scr, qdd + (size_t)w * M.ndof, 1, 0, 1);
}

template <class R, int K, int W> const void* kernel_of(int bwd) {
  return bwd ? reinterpret_cast<const void*>(k_fd_bwd<R, K, W>) : reinterpret_cast<const void*>(k_fd_fwd<R, K, W>);
}
template <class R, int K, int W>
void launch(int bwd, unsigned blocks, unsigned threads, size_t smem, cudaStream_t st, const Nb2ModelDev<R>& M, int B, const FdArgs& a, int words) {
  if (!bwd)
    k_fd_fwd<R, K, W><<<blocks, threads, smem, st>>>(M, B, (const R*)a.q, a.qs, (const R*)a.v, a.vs, (const R*)a.tau, (R*)a.qdd, (R*)a.saved, words, a.wi);
  else
    k_fd_bwd<R, K, W><<<blocks, threads, smem, st>>>(M, B, (const R*)a.state, (const R*)a.saved, (const R*)a.gqdd, (R*)a.gstate, (R*)a.gtau, a.gI, words,
                                                     a.wi);
}
template <class R, int K> const void* kernel_of_width(int W, int bwd) {
  if constexpr (K > 1) {
    if (W == NARROW_W<K>) return kernel_of<R, K, NARROW_W<K>>(bwd);
  }
  return kernel_of<R, K, 32>(bwd);
}
template <class R, int K>
void launch_width(int W, int bwd, unsigned blocks, unsigned threads, size_t smem, cudaStream_t st, const Nb2ModelDev<R>& M, int B, const FdArgs& a,
                  int words) {
  if constexpr (K > 1) {
    if (W == NARROW_W<K>) return launch<R, K, NARROW_W<K>>(bwd, blocks, threads, smem, st, M, B, a, words);
  }
  launch<R, K, 32>(bwd, blocks, threads, smem, st, M, B, a, words);
}

}  // namespace

template <class R> const void* nb2_fd_kernel(int K, int W, int bwd) {
  switch (K) {
    case 1: return kernel_of_width<R, 1>(W, bwd);
    case 2: return kernel_of_width<R, 2>(W, bwd);
    case 4: return kernel_of_width<R, 4>(W, bwd);
    default: return kernel_of_width<R, 8>(W, bwd);
  }
}
template <class R>
void nb2_fd_launch(int K, int W, int bwd, unsigned blocks, unsigned threads, size_t smem, cudaStream_t st, const Nb2ModelDev<R>& M, int B,
                   const FdArgs& a, int words) {
  switch (K) {
    case 1: launch_width<R, 1>(W, bwd, blocks, threads, smem, st, M, B, a, words); break;
    case 2: launch_width<R, 2>(W, bwd, blocks, threads, smem, st, M, B, a, words); break;
    case 4: launch_width<R, 4>(W, bwd, blocks, threads, smem, st, M, B, a, words); break;
    default: launch_width<R, 8>(W, bwd, blocks, threads, smem, st, M, B, a, words); break;
  }
}
cudaError_t nb2_fd_forward_global(const Nb2ModelDev<double>& M, int B, const FdArgs& a, cudaStream_t st) {
  const int words = nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree).total;
  double* scratch = nullptr;
  cudaError_t e = cudaMallocAsync((void**)&scratch, (size_t)B * words * sizeof(double), st);
  if (e != cudaSuccess) return e;
  k_fd_fwd_global<<<(B + 63) / 64, 64, 0, st>>>(M, B, words, (const double*)a.q, a.qs, (const double*)a.v, a.vs, (const double*)a.tau,
                                                (double*)a.qdd, scratch);
  e = cudaGetLastError();
  const cudaError_t f = cudaFreeAsync(scratch, st);
  return e != cudaSuccess ? e : f;
}
template const void* nb2_fd_kernel<float>(int, int, int);
template const void* nb2_fd_kernel<double>(int, int, int);
template void nb2_fd_launch<float>(int, int, int, unsigned, unsigned, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const FdArgs&, int);
template void nb2_fd_launch<double>(int, int, int, unsigned, unsigned, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const FdArgs&, int);
