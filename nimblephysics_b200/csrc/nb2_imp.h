// Host interface of the impulse-dynamics kernels (nb2_imp.cu, DESIGN.md §6q).  They are a translation unit of their own for the reason
// nb2_cfd.h gives: compiled next to other kernels they would change the compiler's inlining of the shared stages, and so the code of the
// existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nb2_model.h"

// arguments of one launch (checked by the caller).  Contacts as CfdArgs (nb2_cfd.h).  Rows in the arithmetic type: state [B][2n],
// offsets ([k][3], [B][k][3] with off_pw, or NULL); forward: vel [B][n] (qdot+), imp [B][k][6 or 3]; backward: the seeds gvel, gimp, and
// gstate [B][2n], goff [B][k][3] (or NULL), gI ([10 nb][B] fp64, or NULL).  wi: per-world inertia ([10 nb][B] fp64) or NULL.  e: the
// restitution, rho: the damping.  Dense Jacobians (J[0] != NULL): vel and imp as the forward, and J = {dvel/dq, dvel/dqdot- [B][n][n],
// dimp/dq, dimp/dqdot- [B][m][n]}.
struct ImpArgs {
  int k, point; const int32_t* body; const double* T;
  const void* state; const void* off; int off_pw; const double* wi; double e, rho;
  void* vel; void* imp;
  const void* gvel; const void* gimp; void* gstate; void* goff; double* gI;
  void* J[4];
};
// one launch, forward (bwd = 0) or backward, one world per 32-thread block, on the passive-free copy of the FD model M (nb2_imp.cuh
// imp_model); `slots` and `smem` from nb2_cfd_slots (the working set is constrained forward dynamics's).  Raises the kernel's
// shared-memory limit to `smem` first.
template <class R>
cudaError_t nb2_imp_launch(int bwd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const ImpArgs& a);
// the dense Jacobians (a.J set; nb2_impj.cu), launched as nb2_imp_launch on the passive-free copy of M; `slots` and `smem` from
// nb2_cfd_slots with jac = 1 (the working set is nb2_cfd.cuh cfdj_layout)
template <class R>
cudaError_t nb2_impj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const ImpArgs& a);
