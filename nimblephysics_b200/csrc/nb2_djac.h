// Host interface of the dense dynamics-Jacobian kernels (nb2_djac.cu, DESIGN.md §6l).  They are a translation unit of their own: they
// instantiate the inverse-dynamics and step passes and sweeps once more (with other strides), and compiled next to the step or
// forward-dynamics kernels they would change the compiler's inlining of those functions, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nb2_model.h"

// Row slots per round: the largest of 32, 16, 8, 4 that is not above the next power of two of n and whose working set fits `max_smem`
// bytes; 0 if none fits.  *smem: the working set's bytes at that slot count.  fd: the forward-dynamics Jacobian, else inverse dynamics.
int nb2_dj_slots(int nb, int n, int nslots, int nfree, bool fd, size_t word, size_t max_smem, size_t* smem);
// one launch, B blocks of one warp: out [B, n] (tau or qdd), J1 / J2 / J3 [B, n, n] (d/dq, d/dqdot, d/dv' or d/dtau); M is the model (FD:
// with an identity action map).  Raises the kernel's shared-memory limit to `smem` first.
template <class R>
cudaError_t nb2_dj_launch(bool fd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const R* state, const R* x, const double* wi,
                          R* out, R* J1, R* J2, R* J3);
