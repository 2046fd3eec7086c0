// Host interface of the constrained forward-dynamics kernels (nb2_cfd.cu, DESIGN.md §6o).  They are a translation unit of their own: they
// instantiate the FD passes and sweeps and the point-Jacobian stages once more, and compiled next to the step or Jacobian kernels they would
// change the compiler's inlining of those functions, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nb2_model.h"

// arguments of one launch (checked by the caller).  Contacts: k canonical bodies, their body <- node transforms [k][12] and whether they
// are point contacts.  Rows in the arithmetic type: state [B][2n], tau [B][n], offsets ([k][3], [B][k][3] with off_pw, or NULL);
// forward: qdd [B][n], wrench [B][k][6 or 3]; backward: the seeds gqdd, gw, and gstate [B][2n], gtau [B][n], goff [B][k][3] (or NULL),
// gI ([10 nb][B] fp64, or NULL).  wi: per-world inertia ([10 nb][B] fp64) or NULL.  Dense Jacobians (J[0] != NULL): qdd and wrench as the
// forward, and J = {dqdd/dq, dqdd/dqdot, dqdd/dtau [B][n][n], dwrench/dq, dwrench/dqdot, dwrench/dtau [B][m][n]}.
struct CfdArgs {
  int k, point; const int32_t* body; const double* T;
  const void* state; const void* tau; const void* off; int off_pw; const double* wi; double rho;
  void* qdd; void* wrench;
  const void* gqdd; const void* gw; void* gstate; void* gtau; void* goff; double* gI;
  void* J[6];
};
// the row slots of the launch whose working set fits `max_smem` bytes (8, else 1; 0: none fits), and its bytes; jac: the Jacobian kernel's
// working set (nb2_cfd.cuh cfdj_layout), which adds the backward words of every slot's seed
int nb2_cfd_slots(int nb, int n, int nslots, int nfree, int m, int jac, size_t word, size_t max_smem, size_t* smem);
// one launch, forward (bwd = 0) or backward, one world per 32-thread block; raises the kernel's shared-memory limit to `smem` first
template <class R>
cudaError_t nb2_cfd_launch(int bwd, int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const CfdArgs& a);
// the dense Jacobians (a.J set; nb2_cfdj.cu), launched as nb2_cfd_launch
template <class R>
cudaError_t nb2_cfdj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const CfdArgs& a);
