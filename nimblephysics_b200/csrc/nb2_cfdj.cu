// Dense-Jacobian kernel of constrained forward dynamics (nb2_constrained_forward_dynamics_jacobians; DESIGN.md §6p), in a translation unit
// of its own: next to k_cfd it would change the compiler's inlining of the functions they share, and so k_cfd's code.  The entry is in
// nb2_kernels.cu.
#include "nb2_cfd.cuh"
#include "nb2_cfd.h"

namespace {

// the dense Jacobians: the same program's forward once, then rounds of ST seeds (nb2_cfd.cuh cfdj_world)
template <class R, int ST>
__global__ void __launch_bounds__(32)
k_cfdj(const __grid_constant__ Nb2ModelDev<R> M, const __grid_constant__ nb2::CfdNodes<R> N, int B, const R* __restrict__ state,
       const R* __restrict__ tau, const R* __restrict__ off, int off_pw, const double* __restrict__ winertia, R rho, R* __restrict__ qdd,
       R* __restrict__ wrench, R* __restrict__ Jq, R* __restrict__ Jqd, R* __restrict__ Jt, R* __restrict__ Wq, R* __restrict__ Wqd,
       R* __restrict__ Wt) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int n = M.ndof, m = N.k * (N.point ? 3 : 6);
  const size_t w = blockIdx.x, nn = (size_t)n * n, mn = (size_t)m * n;
  nb2::CfdRows<R> io{};
  io.state = state + w * 2 * n; io.tau = tau + w * n; io.off = off ? off + (off_pw ? w * N.k * 3 : 0) : nullptr;
  io.qdd = qdd + w * n; io.wrench = wrench + w * m;
  io.wi = winertia ? winertia + w : nullptr; io.wiB = (size_t)B;
  io.rho = rho;
  const nb2::CfdJacRows<R> out{Jq + w * nn, Jqd + w * nn, Jt + w * nn, Wq + w * mn, Wqd + w * mn, Wt + w * mn};
  nb2::cfdj_world<R, ST>(M, N, io, out, ws, [&](auto&& f) {
    f((int)threadIdx.x, 32);
    __syncwarp();
  });
}

template <class R, int ST>
cudaError_t launch_jac(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, const nb2::CfdNodes<R>& N, int B, const CfdArgs& a) {
  cudaError_t e = cudaFuncSetAttribute(k_cfdj<R, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_cfdj<R, ST><<<B, 32, smem, s>>>(M, N, B, (const R*)a.state, (const R*)a.tau, (const R*)a.off, a.off_pw, a.wi, (R)a.rho, (R*)a.qdd,
                                     (R*)a.wrench, (R*)a.J[0], (R*)a.J[1], (R*)a.J[2], (R*)a.J[3], (R*)a.J[4], (R*)a.J[5]);
  return cudaGetLastError();
}

}  // namespace

template <class R>
cudaError_t nb2_cfdj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const CfdArgs& a) {
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(a.k, a.point, a.body, a.T);
  return slots == 8 ? launch_jac<R, 8>(smem, s, M, N, B, a) : launch_jac<R, 1>(smem, s, M, N, B, a);
}
template cudaError_t nb2_cfdj_launch<float>(int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const CfdArgs&);
template cudaError_t nb2_cfdj_launch<double>(int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const CfdArgs&);
