// Host interface of the dense contact-inverse-dynamics Jacobian kernel (nb2_mcidj.cu, DESIGN.md §6s).  It is a translation unit of its own
// for the reason nb2_djac.h gives: compiled next to the inverse-dynamics or contact kernels it would change the compiler's inlining of the
// functions they share, and so the code of the existing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "nb2_model.h"

// arguments of one launch (checked by the caller).  Contacts: k canonical bodies and each body's own origin in its canonical frame
// [k][3] (as nb2_multiple_contact_inverse_dynamics).  Rows in the arithmetic type: state [B][2n], next_vel [B][n], guess [B][k][6] or NULL;
// tau [B][n], wrench [B][k][6]; J = {T_q, T_qdot, T_next_vel [B][n][n], T_guess [B][n][6k], W_q, W_qdot, W_next_vel [B][6k][n],
// W_guess [B][6k][6k]}, the two guess blocks may be NULL.  wi: per-world inertia ([10 nb][B] fp64) or NULL.
struct McidjArgs {
  int k; const int32_t* body; const double* point;
  const void* state; const void* next_vel; const void* guess; const double* wi;
  void* tau; void* wrench;
  void* J[8];
};
// Row slots per round: the largest of 32, 16, 8, 4 that is not above the next power of two of the n + 6k rows and whose working set
// (nb2_mcidj.cuh mcidj_layout) fits `max_smem` bytes; 0 if none fits.  *smem: the working set's bytes at that slot count.
int nb2_mcidj_slots(int nb, int n, int nslots, int nfree, int k, size_t word, size_t max_smem, size_t* smem);
// one launch, B blocks of one warp, on the inverse-dynamics model M; raises the kernel's shared-memory limit to `smem` first
template <class R>
cudaError_t nb2_mcidj_launch(int slots, size_t smem, cudaStream_t s, const Nb2ModelDev<R>& M, int B, const McidjArgs& a);
