// Dense-Jacobian kernel of impulse dynamics (nb2_impulse_dynamics_jacobians; DESIGN.md §6r), in a translation unit of its own: next to
// k_imp it would change the compiler's inlining of the functions they share, and so k_imp's code.  The entry is in nb2_kernels.cu.
#include "nb2_imp.cuh"
#include "nb2_imp.h"

namespace {

// the dense Jacobians: the same program's forward once, then rounds of ST seeds (nb2_imp.cuh impj_world).  M: the passive-free model.
template <class R, int ST>
__global__ void __launch_bounds__(32)
k_impj(const __grid_constant__ Nb2ModelDev<R> M, const __grid_constant__ nb2::CfdNodes<R> N, int B, const R* __restrict__ state,
       const R* __restrict__ off, int off_pw, const double* __restrict__ winertia, R e, R rho, R* __restrict__ vel, R* __restrict__ imp,
       R* __restrict__ Vq, R* __restrict__ Vqd, R* __restrict__ Iq, R* __restrict__ Iqd) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int n = M.ndof, m = N.k * (N.point ? 3 : 6);
  const size_t w = blockIdx.x, nn = (size_t)n * n, mn = (size_t)m * n;
  nb2::ImpRows<R> io{};
  io.state = state + w * 2 * n; io.off = off ? off + (off_pw ? w * N.k * 3 : 0) : nullptr;
  io.vel = vel + w * n; io.imp = imp + w * m;
  io.wi = winertia ? winertia + w : nullptr; io.wiB = (size_t)B;
  io.rho = rho; io.e = e;
  const nb2::ImpJacRows<R> out{Vq + w * nn, Vqd + w * nn, Iq + w * mn, Iqd + w * mn};
  nb2::impj_world<R, ST>(M, N, io, out, ws, [&](auto&& f) {
    f((int)threadIdx.x, 32);
    __syncwarp();
  });
}

template <class R, int ST>
cudaError_t launch_jac(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, const nb2::CfdNodes<R>& N, int B, const ImpArgs& a) {
  cudaError_t e = cudaFuncSetAttribute(k_impj<R, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_impj<R, ST><<<B, 32, smem, s>>>(M, N, B, (const R*)a.state, (const R*)a.off, a.off_pw, a.wi, (R)a.e, (R)a.rho, (R*)a.vel, (R*)a.imp,
                                     (R*)a.J[0], (R*)a.J[1], (R*)a.J[2], (R*)a.J[3]);
  return cudaGetLastError();
}

}  // namespace

template <class R>
cudaError_t nb2_impj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const ImpArgs& a) {
  const Nb2ModelDev<R> P = nb2::imp_model(M);
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(a.k, a.point, a.body, a.T);
  return slots == 8 ? launch_jac<R, 8>(smem, s, P, N, B, a) : launch_jac<R, 1>(smem, s, P, N, B, a);
}
template cudaError_t nb2_impj_launch<float>(int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const ImpArgs&);
template cudaError_t nb2_impj_launch<double>(int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const ImpArgs&);
