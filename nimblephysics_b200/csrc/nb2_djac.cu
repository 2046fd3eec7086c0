// Dense dynamics-Jacobian kernels of libnb2.so (nb2_inverse_dynamics_jacobians / nb2_forward_dynamics_jacobians; DESIGN.md §6l), in a
// translation unit of their own (see nb2_djac.h).  The entries are in nb2_kernels.cu.
#include "nb2_djac.cuh"
#include "nb2_djac.h"

namespace {

// ONE WARP PER WORLD, one world per block (nb2_djac.cuh): the forward on the model's lane schedule, the layer's output, then rounds of ST rows,
// each swept by one thread and written out by the whole warp.
template <class R, int ST, bool FD>
__global__ void __launch_bounds__(32)
k_dj(const __grid_constant__ Nb2ModelDev<R> M, int B, const R* __restrict__ state, const R* __restrict__ x, const double* __restrict__ winertia,
     R* __restrict__ out, R* __restrict__ J1, R* __restrict__ J2, R* __restrict__ J3) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  R* ws = reinterpret_cast<R*>(nb2_smem);
  const int lane = threadIdx.x, n = M.ndof;
  const size_t w = blockIdx.x, nn = (size_t)n * n;
  const R* s = state + w * 2 * n;
  const double* wi = winertia ? winertia + w : nullptr;
  nb2::dj_load<R>(M, ws, s, x + w * n, lane, 32);
  __syncwarp();
#pragma unroll 1
  for (int sg = 1; sg < nb2::dj_fwd_stages<FD>() - 1; sg++) {
    nb2::dj_forward_stage<R, FD>(M, ws, lane, sg, wi, (size_t)B);
    __syncwarp();
  }
  nb2::dj_store_out<R>(M, ws, out + w * n, lane, 32);
#pragma unroll 1
  for (int r0 = 0; r0 < n; r0 += ST) {
    const int nrows = min(ST, n - r0);
    if (lane < nrows) nb2::dj_row<R, ST, FD>(M, ws, s, r0 + lane, lane, wi, (size_t)B);
    __syncwarp();
    nb2::dj_rows_store<R, ST, FD>(M, ws, r0, nrows, J1 + w * nn, J2 + w * nn, J3 + w * nn, lane, 32);
    __syncwarp();
  }
}

template <class R, int ST, bool FD>
cudaError_t launch(size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const R* state, const R* x, const double* wi, R* out, R* J1, R* J2, R* J3) {
  cudaError_t e = cudaFuncSetAttribute(k_dj<R, ST, FD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_dj<R, ST, FD><<<B, 32, smem, s>>>(M, B, state, x, wi, out, J1, J2, J3);
  return cudaGetLastError();
}
template <class R, bool FD>
cudaError_t launch_slots(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const R* state, const R* x, const double* wi, R* out,
                         R* J1, R* J2, R* J3) {
  switch (slots) {
    case 32: return launch<R, 32, FD>(smem, s, M, B, state, x, wi, out, J1, J2, J3);
    case 16: return launch<R, 16, FD>(smem, s, M, B, state, x, wi, out, J1, J2, J3);
    case 8: return launch<R, 8, FD>(smem, s, M, B, state, x, wi, out, J1, J2, J3);
    default: return launch<R, 4, FD>(smem, s, M, B, state, x, wi, out, J1, J2, J3);
  }
}

}  // namespace

int nb2_dj_slots(int nb, int n, int nslots, int nfree, bool fd, size_t word, size_t max_smem, size_t* smem) {
  int want = 4;
  while (want < 32 && want < n) want *= 2;
  for (int st = want; st >= 4; st /= 2) {
    const size_t bytes = (size_t)nb2::dj_layout(nb, n, nslots, nfree, fd, st).total * word;
    if (bytes <= max_smem) { *smem = bytes; return st; }
  }
  return 0;
}
template <class R>
cudaError_t nb2_dj_launch(bool fd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const R* state, const R* x, const double* wi,
                          R* out, R* J1, R* J2, R* J3) {
  return fd ? launch_slots<R, true>(slots, smem, s, M, B, state, x, wi, out, J1, J2, J3)
            : launch_slots<R, false>(slots, smem, s, M, B, state, x, wi, out, J1, J2, J3);
}
template cudaError_t nb2_dj_launch<float>(bool, int, size_t, cudaStream_t, const Nb2ModelDev<float>&, int, const float*, const float*, const double*,
                                          float*, float*, float*, float*);
template cudaError_t nb2_dj_launch<double>(bool, int, size_t, cudaStream_t, const Nb2ModelDev<double>&, int, const double*, const double*,
                                           const double*, double*, double*, double*, double*);
