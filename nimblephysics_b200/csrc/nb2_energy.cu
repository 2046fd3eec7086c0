// Energy-and-momentum kernels of libnb2.so (nb2_energy_momentum / _backward; DESIGN.md §6m), in a translation unit of their own (see
// nb2_energy.h).  The entries are in nb2_kernels.cu.
#include "nb2_energy.cuh"
#include "nb2_energy.h"

namespace {

// ONE WARP PER WORLD, NB2_EM_WPB worlds per block, the stages of nb2_energy.cuh with a __syncwarp between them
template <class R>
__global__ void __launch_bounds__(32 * NB2_EM_WPB)
k_em_fwd(const __grid_constant__ Nb2ModelDev<R> M, int B, int root, const R* __restrict__ state, const double* __restrict__ winertia,
         R* __restrict__ kin, R* __restrict__ pot, R* __restrict__ mom) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int lane = threadIdx.x & 31, n = M.ndof;
  const size_t w = (size_t)blockIdx.x * NB2_EM_WPB + (threadIdx.x >> 5);
  if (w >= (size_t)B) return;
  R* ws = reinterpret_cast<R*>(nb2_smem) + (threadIdx.x >> 5) * nb2::em_layout(M.nb, n, false).total;
  const R* q = state + w * 2 * n;
  const double* wi = winertia ? winertia + w : nullptr;
  nb2::jcdb_init<R>(M, q, root, ws, lane, 32);
  __syncwarp();
  nb2::jc_moments<R>(M, root, wi, (size_t)B, ws, lane, 32);
  __syncwarp();
  nb2::jcd_vel<R>(M, q + n, root, wi, (size_t)B, true, ws, lane);
  __syncwarp();
  nb2::em_bodies<R>(M, root, wi, (size_t)B, ws, lane, 32);
  __syncwarp();
  nb2::em_sums<R>(M, q, root, ws, lane, 32);
  __syncwarp();
  nb2::em_store<R>(M, root, ws, kin + w, pot + w, mom + w * 6, lane);
}
template <class R>
__global__ void __launch_bounds__(32 * NB2_EM_WPB)
k_em_bwd(const __grid_constant__ Nb2ModelDev<R> M, int B, int root, const R* __restrict__ state, const double* __restrict__ winertia,
         const R* __restrict__ gkin, const R* __restrict__ gpot, const R* __restrict__ gmom, R* __restrict__ gstate, double* __restrict__ ginertia) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int lane = threadIdx.x & 31, n = M.ndof;
  const nb2::EmLayout L = nb2::em_layout(M.nb, n, true);
  const size_t w = (size_t)blockIdx.x * NB2_EM_WPB + (threadIdx.x >> 5);
  if (w >= (size_t)B) return;
  R* ws = reinterpret_cast<R*>(nb2_smem) + (threadIdx.x >> 5) * L.total;
  const R* q = state + w * 2 * n;
  const double* wi = winertia ? winertia + w : nullptr;
  const R zero6[6] = {R(0), R(0), R(0), R(0), R(0), R(0)};
  const R gT = gkin ? gkin[w] : R(0), gU = gpot ? gpot[w] : R(0);
  const R* gh = gmom ? gmom + w * 6 : zero6;
  nb2::jcdb_init<R>(M, q, root, ws, lane, 32);
  __syncwarp();
  nb2::jc_moments<R>(M, root, wi, (size_t)B, ws, lane, 32);
  __syncwarp();
  nb2::jcd_vel<R>(M, q + n, root, wi, (size_t)B, true, ws, lane);
  __syncwarp();
  nb2::emb_bodies<R>(M, q, root, wi, (size_t)B, gT, gU, gh, ws, ginertia ? ginertia + w : nullptr, (size_t)B, lane, 32);
  __syncwarp();
  nb2::emb_reduce<R>(M, q, q + n, root, ws, lane);
  __syncwarp();
  nb2::jd_store_row<R>(n, ws + L.oGq, gstate + w * 2 * n, lane, 32);
}

template <auto Kern> cudaError_t allow_smem(size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) : cudaSuccess;
}

}  // namespace

size_t nb2_em_smem(int nb, int n, bool bwd, size_t word) { return (size_t)NB2_EM_WPB * nb2::em_layout(nb, n, bwd).total * word; }

template <class R>
cudaError_t nb2_em_launch(cudaStream_t s, size_t smem, const Nb2ModelDev<R>& M, int B, int root, const R* state, const double* wi, R* kin, R* pot,
                          R* mom, const R* gkin, const R* gpot, const R* gmom, R* gstate, double* gI) {
  const unsigned blocks = (unsigned)(((size_t)B + NB2_EM_WPB - 1) / NB2_EM_WPB);
  cudaError_t e;
  if (!gstate) {
    if ((e = allow_smem<k_em_fwd<R>>(smem)) != cudaSuccess) return e;
    k_em_fwd<R><<<blocks, 32 * NB2_EM_WPB, smem, s>>>(M, B, root, state, wi, kin, pot, mom);
  } else {
    if ((e = allow_smem<k_em_bwd<R>>(smem)) != cudaSuccess) return e;
    k_em_bwd<R><<<blocks, 32 * NB2_EM_WPB, smem, s>>>(M, B, root, state, wi, gkin, gpot, gmom, gstate, gI);
  }
  return cudaGetLastError();
}
template cudaError_t nb2_em_launch<float>(cudaStream_t, size_t, const Nb2ModelDev<float>&, int, int, const float*, const double*, float*, float*,
                                          float*, const float*, const float*, const float*, float*, double*);
template cudaError_t nb2_em_launch<double>(cudaStream_t, size_t, const Nb2ModelDev<double>&, int, int, const double*, const double*, double*,
                                           double*, double*, const double*, const double*, const double*, double*, double*);
