// Host interface of the forward-dynamics kernels (nb2_fd.cu).  They are a translation unit of their own: they instantiate the step's
// device functions a second time (the B1 / B2 / B3 sweeps, the passes), and compiled next to the step kernels they would change the
// compiler's inlining of those functions, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nb2_model.h"

// arguments of one launch: the forward reads q, qdot (rows qs / vs words apart) and tau and writes qdd and, when not NULL, the saved
// stream; the backward reads state, saved and gqdd and writes gstate, gtau and, when not NULL, gI
struct FdArgs {
  const void* q; int qs; const void* v; int vs; const void* tau; void* qdd; void* saved;
  const void* state; const void* gqdd; void* gstate; void* gtau; double* gI;
  const double* wi;
};
// the kernel of lane count K (1, 2, 4 or 8) and group width W (32, or NARROW_W<K> = 32/K with K > 1; nb2_coop.cuh), forward (bwd = 0) or
// backward: for cudaFuncSetAttribute and the occupancy query
template <class R> const void* nb2_fd_kernel(int K, int W, int bwd);
template <class R>
void nb2_fd_launch(int K, int W, int bwd, unsigned blocks, unsigned threads, size_t smem, cudaStream_t st, const Nb2ModelDev<R>& M, int B, const FdArgs& a,
                   int words);
// fp64 forward, one thread per world with its scratch in global memory (allocated stream-ordered for the call): the path of
// nb2_forward_dynamics for a model that no schedule's shared-memory working set fits
cudaError_t nb2_fd_forward_global(const Nb2ModelDev<double>& M, int B, const FdArgs& a, cudaStream_t st);
