// Constrained forward-dynamics kernels of libnb2.so (nb2_constrained_forward_dynamics / _backward; DESIGN.md §6o), in a translation unit of
// their own (see nb2_cfd.h).  The entries are in nb2_kernels.cu.
#include "nb2_cfd.cuh"
#include "nb2_cfd.h"

namespace {

// ONE WARP PER WORLD, one world per block: the program of nb2_cfd.cuh with a __syncwarp after every stage.
template <class R, int ST, bool BWD>
__global__ void __launch_bounds__(32)
k_cfd(const __grid_constant__ Nb2ModelDev<R> M, const __grid_constant__ nb2::CfdNodes<R> N, int B, const R* __restrict__ state,
      const R* __restrict__ tau, const R* __restrict__ off, int off_pw, const double* __restrict__ winertia, R rho, R* __restrict__ qdd,
      R* __restrict__ wrench, const R* __restrict__ gqdd, const R* __restrict__ gw, R* __restrict__ gstate, R* __restrict__ gtau,
      R* __restrict__ goff, double* __restrict__ gI) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int n = M.ndof, m = N.k * (N.point ? 3 : 6);
  const size_t w = blockIdx.x;
  nb2::CfdRows<R> io;
  io.state = state + w * 2 * n; io.tau = tau + w * n; io.off = off ? off + (off_pw ? w * N.k * 3 : 0) : nullptr;
  io.qdd = BWD ? nullptr : qdd + w * n; io.wrench = BWD ? nullptr : wrench + w * m;
  io.gqdd = BWD ? gqdd + w * n : nullptr; io.gw = BWD ? gw + w * m : nullptr;
  io.gstate = BWD ? gstate + w * 2 * n : nullptr; io.gtau = BWD ? gtau + w * n : nullptr;
  io.goff = BWD && goff ? goff + w * N.k * 3 : nullptr; io.gI = BWD && gI ? gI + w : nullptr;
  io.wi = winertia ? winertia + w : nullptr; io.wiB = (size_t)B;
  io.rho = rho;
  nb2::cfd_world<R, ST, BWD>(M, N, io, ws, [&](auto&& f) {
    f((int)threadIdx.x, 32);
    __syncwarp();
  });
}

template <class R, int ST, bool BWD>
cudaError_t launch(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, const nb2::CfdNodes<R>& N, int B, const CfdArgs& a) {
  cudaError_t e = cudaFuncSetAttribute(k_cfd<R, ST, BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_cfd<R, ST, BWD><<<B, 32, smem, s>>>(M, N, B, (const R*)a.state, (const R*)a.tau, (const R*)a.off, a.off_pw, a.wi, (R)a.rho, (R*)a.qdd,
                                         (R*)a.wrench, (const R*)a.gqdd, (const R*)a.gw, (R*)a.gstate, (R*)a.gtau, (R*)a.goff, a.gI);
  return cudaGetLastError();
}

}  // namespace

int nb2_cfd_slots(int nb, int n, int nslots, int nfree, int m, int jac, size_t word, size_t max_smem, size_t* smem) {
  for (int st = 8; st >= 1; st = st == 8 ? 1 : 0) {
    const int words = jac ? nb2::cfdj_layout(nb, n, nslots, nfree, m, st).total : nb2::cfd_layout(nb, n, nslots, nfree, m, st).total;
    const size_t bytes = (size_t)words * word;
    if (bytes <= max_smem) { *smem = bytes; return st; }
  }
  return 0;
}
template <class R>
cudaError_t nb2_cfd_launch(int bwd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const CfdArgs& a) {
  const nb2::CfdNodes<R> N = nb2::cfd_nodes<R>(a.k, a.point, a.body, a.T);
  if (slots == 8) return bwd ? launch<R, 8, true>(smem, s, M, N, B, a) : launch<R, 8, false>(smem, s, M, N, B, a);
  return bwd ? launch<R, 1, true>(smem, s, M, N, B, a) : launch<R, 1, false>(smem, s, M, N, B, a);
}
template cudaError_t nb2_cfd_launch<float>(int, int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const CfdArgs&);
template cudaError_t nb2_cfd_launch<double>(int, int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const CfdArgs&);
