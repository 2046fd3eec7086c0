// Host interface of the energy-and-momentum kernels (nb2_energy.cu, DESIGN.md §6m).  They are a translation unit of their own: they
// instantiate the COM-Jacobian stages of nb2_jac.cuh once more, and compiled next to the Jacobian kernels they would change the compiler's
// inlining of those functions, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "nb2_model.h"

// warps (= worlds) per block of both kernels
#define NB2_EM_WPB 4
// bytes of shared memory per block: the forward's working set, or the backward's
size_t nb2_em_smem(int nb, int n, bool bwd, size_t word);
// one launch of the tree rooted at `root`.  Forward (gstate == NULL): kin [B], pot [B], mom [B][6].  Backward: the adjoints gkin [B],
// gpot [B], gmom [B][6] (any may be NULL: zero) into gstate [B][2n] and, when not NULL, gI (fp64 [10 nb][B]).  Raises the kernel's
// shared-memory limit to `smem` first when it is above the default.
template <class R>
cudaError_t nb2_em_launch(cudaStream_t s, size_t smem, const Nb2ModelDev<R>& M, int B, int root, const R* state, const double* wi, R* kin, R* pot,
                          R* mom, const R* gkin, const R* gpot, const R* gmom, R* gstate, double* gI);
