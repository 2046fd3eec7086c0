// Host interface of the regressor kernels (nb2_reg.cu, DESIGN.md §6n).  They are a translation unit of their own: they instantiate the
// inverse-dynamics forward passes once more (with stride 1), and compiled next to the step or ID kernels they would change the compiler's
// inlining of those functions, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nb2_model.h"

// warps (= worlds) per block of both kernels
#define NB2_REG_WPB 4
// bytes of shared memory per block: the working set of the ID regressor, or of the energy regressor
size_t nb2_reg_smem(int nb, int n, int nslots, int nfree, bool energy, size_t word);
// one launch.  ID (Y != NULL): Y [B][n][nb][10] and tau_passive [B][n] at state [B][2n] and next_vel [B][n].  Energy (Y == NULL):
// YT, YU [B][nb][10] and spring [B] at state.  Raises the kernel's shared-memory limit to `smem` first when it is above the default.
template <class R>
cudaError_t nb2_reg_launch(cudaStream_t s, size_t smem, const Nb2ModelDev<R>& M, int B, const R* state, const R* next_vel, R* Y, R* tau_passive,
                           R* YT, R* YU, R* spring);
