// Regressor kernels of libnb2.so (nb2_inverse_dynamics_regressor / nb2_energy_regressor; DESIGN.md §6n), in a translation unit of their
// own (see nb2_reg.h).  The entries are in nb2_kernels.cu.
#include "nb2_reg.cuh"
#include "nb2_reg.h"

namespace {

// ONE WARP PER WORLD, NB2_REG_WPB worlds per block, the stages of nb2_reg.cuh with a __syncwarp between them.  The ID kernel fills the
// buffer one row of Y at a time and the whole warp stores it, so the world's n * nb * 10 words leave in address order.
template <class R>
__global__ void __launch_bounds__(32 * NB2_REG_WPB)
k_reg_id(const __grid_constant__ Nb2ModelDev<R> M, int B, const R* __restrict__ state, const R* __restrict__ next_vel, R* __restrict__ Y,
         R* __restrict__ tau_passive) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int lane = threadIdx.x & 31, n = M.ndof, row = 10 * M.nb;
  const nb2::RegLayout L = nb2::reg_layout(M, false);
  const size_t w = (size_t)blockIdx.x * NB2_REG_WPB + (threadIdx.x >> 5);
  if (w >= (size_t)B) return;
  R* ws = reinterpret_cast<R*>(nb2_smem) + (threadIdx.x >> 5) * L.total;
  nb2::dj_load<R>(M, ws, state + w * 2 * n, next_vel + w * n, lane, 32);
  __syncwarp();
  nb2::reg_kinematics<R>(M, ws, lane, 1);
  __syncwarp();
  nb2::reg_kinematics<R>(M, ws, lane, 2);
  __syncwarp();
  nb2::reg_poses<R>(M, ws, lane);
  __syncwarp();
  nb2::reg_axes<R>(M, ws, tau_passive + w * n, lane, 32);
  __syncwarp();
  R* y = Y + w * n * row;
#pragma unroll 1
  for (int d = 0; d < n; d++) {
    nb2::reg_id_row<R>(M, ws, d, lane, 32);
    __syncwarp();
    nb2::reg_store<R>(ws + L.oY, y + (size_t)d * row, row, lane, 32);
    __syncwarp();
  }
}
template <class R>
__global__ void __launch_bounds__(32 * NB2_REG_WPB)
k_reg_energy(const __grid_constant__ Nb2ModelDev<R> M, int B, const R* __restrict__ state, R* __restrict__ YT, R* __restrict__ YU,
             R* __restrict__ spring) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int lane = threadIdx.x & 31, n = M.ndof, row = 10 * M.nb;
  const nb2::RegLayout L = nb2::reg_layout(M, true);
  const size_t w = (size_t)blockIdx.x * NB2_REG_WPB + (threadIdx.x >> 5);
  if (w >= (size_t)B) return;
  R* ws = reinterpret_cast<R*>(nb2_smem) + (threadIdx.x >> 5) * L.total;
  const R* s = state + w * 2 * n;
  nb2::dj_load<R>(M, ws, s, s + n, lane, 32);  // v' = qdot: the accelerations are not used
  __syncwarp();
  nb2::reg_kinematics<R>(M, ws, lane, 1);
  __syncwarp();
  nb2::reg_kinematics<R>(M, ws, lane, 2);
  __syncwarp();
  nb2::reg_poses<R>(M, ws, lane);
  __syncwarp();
  nb2::reg_energy_cols<R>(M, ws, lane, 32);
  __syncwarp();
  nb2::reg_store<R>(ws + L.oY, YT + w * row, row, lane, 32);
  nb2::reg_store<R>(ws + L.oY + row, YU + w * row, row, lane, 32);
  nb2::reg_spring_energy<R>(M, ws, spring + w, lane);
}

template <auto Kern> cudaError_t allow_smem(size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) : cudaSuccess;
}

}  // namespace

size_t nb2_reg_smem(int nb, int n, int nslots, int nfree, bool energy, size_t word) {
  return (size_t)NB2_REG_WPB * nb2::reg_layout(nb, n, nslots, nfree, energy).total * word;
}

template <class R>
cudaError_t nb2_reg_launch(cudaStream_t s, size_t smem, const Nb2ModelDev<R>& M, int B, const R* state, const R* next_vel, R* Y, R* tau_passive,
                           R* YT, R* YU, R* spring) {
  const unsigned blocks = (unsigned)(((size_t)B + NB2_REG_WPB - 1) / NB2_REG_WPB);
  cudaError_t e;
  if (Y) {
    if ((e = allow_smem<k_reg_id<R>>(smem)) != cudaSuccess) return e;
    k_reg_id<R><<<blocks, 32 * NB2_REG_WPB, smem, s>>>(M, B, state, next_vel, Y, tau_passive);
  } else {
    if ((e = allow_smem<k_reg_energy<R>>(smem)) != cudaSuccess) return e;
    k_reg_energy<R><<<blocks, 32 * NB2_REG_WPB, smem, s>>>(M, B, state, YT, YU, spring);
  }
  return cudaGetLastError();
}
template cudaError_t nb2_reg_launch<float>(cudaStream_t, size_t, const Nb2ModelDev<float>&, int, const float*, const float*, float*, float*, float*,
                                           float*, float*);
template cudaError_t nb2_reg_launch<double>(cudaStream_t, size_t, const Nb2ModelDev<double>&, int, const double*, const double*, double*, double*,
                                            double*, double*, double*);
