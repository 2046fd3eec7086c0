// Impulse-dynamics kernels of libnb2.so (nb2_impulse_dynamics / _backward; DESIGN.md §6q), in a translation unit of their own (see
// nb2_imp.h).  The entries are in nb2_kernels.cu.
#include "nb2_imp.cuh"
#include "nb2_imp.h"

namespace {

// ONE WARP PER WORLD, one world per block: the program of nb2_imp.cuh with a __syncwarp after every stage.  M: the passive-free model.
template <class R, int ST, bool BWD>
__global__ void __launch_bounds__(32)
k_imp(const __grid_constant__ Nb2ModelDev<R> M, const __grid_constant__ nb2::CfdNodes<R> N, int B, const R* __restrict__ state,
      const R* __restrict__ off, int off_pw, const double* __restrict__ winertia, R e, R rho, R* __restrict__ vel, R* __restrict__ imp,
      const R* __restrict__ gvel, const R* __restrict__ gimp, R* __restrict__ gstate, R* __restrict__ goff, double* __restrict__ gI) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int n = M.ndof, m = N.k * (N.point ? 3 : 6);
  const size_t w = blockIdx.x;
  nb2::ImpRows<R> io;
  io.state = state + w * 2 * n; io.off = off ? off + (off_pw ? w * N.k * 3 : 0) : nullptr;
  io.vel = BWD ? nullptr : vel + w * n; io.imp = BWD ? nullptr : imp + w * m;
  io.gvel = BWD ? gvel + w * n : nullptr; io.gimp = BWD ? gimp + w * m : nullptr;
  io.gstate = BWD ? gstate + w * 2 * n : nullptr;
  io.goff = BWD && goff ? goff + w * N.k * 3 : nullptr; io.gI = BWD && gI ? gI + w : nullptr;
  io.wi = winertia ? winertia + w : nullptr; io.wiB = (size_t)B;
  io.rho = rho; io.e = e;
  nb2::imp_world<R, ST, BWD>(M, N, io, ws, [&](auto&& f) {
    f((int)threadIdx.x, 32);
    __syncwarp();
  });
}

template <class R, int ST, bool BWD>
cudaError_t launch(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, const nb2::CfdNodes<R>& N, int B, const ImpArgs& a) {
  cudaError_t e = cudaFuncSetAttribute(k_imp<R, ST, BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_imp<R, ST, BWD><<<B, 32, smem, s>>>(M, N, B, (const R*)a.state, (const R*)a.off, a.off_pw, a.wi, (R)a.e, (R)a.rho, (R*)a.vel, (R*)a.imp,
                                         (const R*)a.gvel, (const R*)a.gimp, (R*)a.gstate, (R*)a.goff, a.gI);
  return cudaGetLastError();
}

}  // namespace

template <class R>
cudaError_t nb2_imp_launch(int bwd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const ImpArgs& a) {
  const Nb2ModelDev<R> P = nb2::imp_model(M);
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(a.k, a.point, a.body, a.T);
  if (slots == 8) return bwd ? launch<R, 8, true>(smem, s, P, N, B, a) : launch<R, 8, false>(smem, s, P, N, B, a);
  return bwd ? launch<R, 1, true>(smem, s, P, N, B, a) : launch<R, 1, false>(smem, s, P, N, B, a);
}
template cudaError_t nb2_imp_launch<float>(int, int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const ImpArgs&);
template cudaError_t nb2_imp_launch<double>(int, int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const ImpArgs&);
