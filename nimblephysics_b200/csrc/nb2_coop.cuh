// The cooperative-lane shape of the contact-free kernels (step, inverse and forward dynamics), shared by nb2_kernels.cu and nb2_fd.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <type_traits>

#include "nb2_dyn.cuh"

namespace {

// K lanes cooperate on one world (K = M.lanes, compile-time here so that the scratch stride is a constant):
// a warp holds 32/K worlds, thread t of the warp is lane t % K of world slot t / K.  Scratch is [word][slot] with an
// odd stride (32/K + 1) so that the lanes of one world and the slots of one lane spread over the banks.
template <int K> struct CoopShape {
  static constexpr int WPW = 32 / K;                    // worlds per warp
  static constexpr int ST = (K == 1) ? 32 : WPW + 1;    // scratch stride in words
};

// With several lanes per world the per-body constants are staged once per block in shared memory (see nb2_dyn.cuh xtree):
// lanes of a warp sit on different bodies, which a constant-bank load would serialise.
template <int K> __host__ __device__ constexpr int body_table_words(int nb) { return (K > 1) ? ((nb * NB2_BT_WORDS + 3) & ~3) : 0; }
template <class R, int K>
__device__ __forceinline__ const R* stage_body_table(const Nb2ModelDev<R>& M, R* tab) {
  if constexpr (K == 1) return nullptr;
  else {
  // copied in 8-byte units: these loads have lane-varying addresses too, and the constant bank replays a load once per
  // distinct address, so fp32 tables take half the replays of a word-by-word copy.  The 8-byte loads need M itself 8-byte
  // aligned in the parameter space: every kernel that calls this takes M as its FIRST parameter (the parameter space starts
  // aligned), keep it there.  The member offsets are checked below; an alignas(8) on Nb2ModelDev would also guarantee it, but it
  // changes the code generated for most kernels that read the model (inverse dynamics, mass matrix, the one-lane step kernels).
  using U = std::conditional_t<sizeof(R) == 4, float2, double>;
  constexpr int XU = 12 * sizeof(R) / sizeof(U), IU = 10 * sizeof(R) / sizeof(U), BU = XU + IU;  // units per Xtree / inertia row
  static_assert(offsetof(Nb2ModelDev<R>, Xtree) % sizeof(U) == 0 && offsetof(Nb2ModelDev<R>, inertia) % sizeof(U) == 0, "unaligned body tables");
  const U* xs = reinterpret_cast<const U*>(&M.Xtree[0][0]);
  const U* is = reinterpret_cast<const U*>(&M.inertia[0][0]);
  U* t = reinterpret_cast<U*>(tab);
  for (int k = threadIdx.x; k < M.nb * BU; k += blockDim.x) {
    const int i = k / BU, j = k - i * BU;
    t[k] = (j < XU) ? xs[i * XU + j] : is[i * IU + j - XU];
  }
  __syncthreads();
  return tab;
  }
}

}  // namespace
