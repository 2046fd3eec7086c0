// Contact / boxed-LCP stage, WARP-COOPERATIVE: one warp owns one world, the whole problem (LCP matrix, factors, rows,
// contact list) lives in that warp's shared-memory workspace, and every dense loop is spread over the 32 lanes.
//
// Programming model (SPMD inside a warp).  Code in this file is written once and runs
//   * on the device with 32 lanes:  CW_FOR(i, n) hands index i to lane i % 32; everything outside a CW_FOR is UNIFORM code
//     that all lanes execute redundantly on identical values (reads of one shared-memory word are broadcasts, data-dependent
//     branches never diverge because a warp holds ONE world); reductions are shuffle butterflies that leave the same bits in
//     every lane; CW_SYNC() orders shared-memory traffic between phases;
//   * on the host (tests/host_emul, no GPU in the build container) with ONE lane: CW_FOR is a plain loop — optionally run
//     backwards (cw_host_reverse) so that an iteration reading what another iteration of the SAME loop wrote shows up.
// Rules that keep both builds equivalent: a CW_FOR body touches only its own outputs; uniform code never read-modify-writes
// shared memory (CW_ONE { } does that on one lane); a CW_SYNC() separates writers from later readers.
//
// What is restated (reference file:line) is unchanged from the first version of this stage:
//   contact filtering / rows / bounds     dart/constraint/ConstraintSolver.cpp:576-601, ContactConstraint.cpp:66-230, 361-514, 734-795
//   A by impulse tests                    dart/constraint/BoxedLcpConstraintSolver.cpp:190-349
//   solve chain                           BoxedLcpConstraintSolver.cpp:352-789; LCPUtils.cpp:12-201, 346-444; PgsBoxedLcpSolver.cpp:79-278
//   Dantzig                               dart/external/odelcpsolver/lcp.cpp:362-1114
//   classification / standardisation      dart/neural/ConstrainedGroupGradientMatrices.cpp:482-872, 218-339
//   impulses, velocity update             ContactConstraint.cpp:630-684, Skeleton.cpp:13571-13595
// Where a pivot or a label is DECIDED the summation order of the serial algorithms is kept (column-oriented triangular
// solves and factor updates give each entry the same sequence of subtractions as the row-oriented serial loops; ratio
// tests resolve ties by position like the serial strict-'<' scans).  Plain inner products are tree-summed.
#pragma once
#include <math.h>
#include <stdint.h>

#include "nb2_dyn.cuh"
#include "nb2_geom.cuh"

#include "../../include/nb2.h"  // NB2_MAX_CONTACTS, NB2_MAX_ROWS

#define NB2_MAX_SHAPES 24
#define NB2_MAX_LIMITS 32   // joints whose position limits are enforced (JointLimitConstraint rows)
#define NB2_MAX_CB 64       // collision bodies: moving bodies that carry a shape, plus child and parent of every limit joint
#define NB2_CT_LIMIT_LOWER 100  // "contact" types of the pseudo contacts that carry joint-limit rows
#define NB2_CT_LIMIT_UPPER 101
#define NB2_MAX_PAIRS 64

// status bits (per world)
#define NB2_ST_SHORTCIRCUIT 1
#define NB2_ST_DANTZIG 2
#define NB2_ST_DANTZIG_FAILED 4
#define NB2_ST_PGS 8
#define NB2_ST_FRICTION_DROPPED 16
#define NB2_ST_NAN 32
#define NB2_ST_NOT_STANDARDIZED 64
#define NB2_ST_UNSUPPORTED_GEOMETRY 128
#define NB2_ST_CONTACT_OVERFLOW 256
#define NB2_ST_MERGED 512    // LCPUtils::reduce merged near-identical columns before a solver ran
#define NB2_ST_BOUNCE 1024   // a restitution (bounce) term raised some b_i: the backward runs a second reverse sweep for such a world
#define NB2_ST_PENCORR 4096  // a penetration-correction velocity raised some b_i (informational: the backward handles it)
#define NB2_ST_BWD_ERROR 2048  // set by the BACKWARD kernel: the step could not be back-propagated (gradients are NaN)

// ConstraintMapping (dart/neural/ConstrainedGroupGradientMatrices.hpp:33-39)
#define NB2_MAP_NOT_CLAMPING (-1)
#define NB2_MAP_CLAMPING (-2)
#define NB2_MAP_ILLEGAL (-3)

struct Nb2ContactDev {
  int nshapes, npairs, pen_correction, ncb;  // ncb: number of COLLISION BODIES (moving bodies that carry a shape)
  double clip_depth, fallback_cfm;
  int16_t shape_body[NB2_MAX_SHAPES];       // canonical body index, -1 = static (world-fixed)
  int16_t shape_type[NB2_MAX_SHAPES];       // 0 box, 1 sphere, 2 capsule
  int16_t shape_orig_body[NB2_MAX_SHAPES];  // reference BodyNode index (reported with the contacts)
  int16_t pair_a[NB2_MAX_PAIRS], pair_b[NB2_MAX_PAIRS];  // collision pairs in the reference's enumeration order
  int16_t cb_body[NB2_MAX_CB];              // collision body k -> canonical body
  int nlim, pad2_;                          // joints with enforced position limits (1-dof joints)
  int16_t lim_body[NB2_MAX_LIMITS];         // canonical body whose parent joint it is
  int16_t cb_of_body[NB2_MAX_BODIES];       // canonical body -> collision body index or -1
  int16_t cdof0[NB2_MAX_BODIES];            // number of dofs of the PROPER ancestors of a body (offset of its own dofs on its chain)
  int max_chain_dofs, pad_;                 // most dofs on the chain root .. collision body, over the collision bodies
  unsigned long long anc_mask[NB2_MAX_BODIES];  // bit j: body j is an ancestor of (or is) this body; bodies are numbered in DFS pre-order
  double shape_dims[NB2_MAX_SHAPES][3];
  double shape_T[NB2_MAX_SHAPES][12];       // shape frame -> canonical body frame (or world)
  double shape_mu[NB2_MAX_SHAPES], shape_rest[NB2_MAX_SHAPES];
};

// the big routines of the solver chain; inlined by default (NB2_CW_NOINLINE: real calls)
#if defined(__CUDACC__) && defined(NB2_CW_NOINLINE)
#define NB2_HDN __host__ __device__ __noinline__   // experiment: -23 % static code, but slower (calls cost ~60 cycles each, see scripts/dev/ubench)
#elif defined(__CUDACC__)
#define NB2_HDN __host__ __device__ __forceinline__
#else
#define NB2_HDN inline
#endif

namespace nb2 {
namespace cw {

// ------------------------------------------------------------------------------------------------ SPMD layer
#ifdef __CUDA_ARCH__
#define CW_DEV 1
#define CW_LANE ((int)(threadIdx.x & 31))
#define CW_SYNC() __syncwarp()
// NB2_CW_FOR_UNIFORM: the loop over passes gets a warp-uniform trip count and only the body is predicated.  In isolation a divergent loop
// exit costs more than this form (scripts/dev/ubench/br.cu measures both); inside the real kernels the compiler turns the guarded bodies
// into divergent branches anyway, so the plain per-lane loop is the default.
#ifndef NB2_CW_FOR_UNIFORM
#define CW_FOR(i, n) for (int i = (int)(threadIdx.x & 31); i < (n); i += 32)
#else
#define CW_FOR(i, n)                                                         \
  for (int i##_b = 0, i##_n = (n); i##_b < i##_n; i##_b += 32)               \
    for (int i = i##_b + (int)(threadIdx.x & 31), i##_1 = 1; i##_1; i##_1 = 0) \
      if (i < i##_n)
#endif
#define CW_ONE if ((threadIdx.x & 31) == 0)
#define CW_FULL 0xFFFFFFFFu
#else
#define CW_DEV 0
#define CW_LANE 0
#define CW_SYNC() ((void)0)
inline int& cw_host_reverse() { static int r = 0; return r; }
inline int cw_host_idx(int it, int n) { return cw_host_reverse() ? n - 1 - it : it; }
#define CW_FOR(i, n) for (int i##_it = 0, i##_n = (n), i = cw_host_idx(0, i##_n); i##_it < i##_n; i##_it++, i = cw_host_idx(i##_it, i##_n))
#define CW_ONE
#endif

// 2-D index space nr x nc spread over the lanes in row-major order WITHOUT an integer division per element (a runtime divisor costs
// ~25 instructions): every lane walks (r, c) by the lane count.
struct It2 { int row, col, e, dr, dc, tot, nc; };
NB2_HD It2 it2_begin(int nr, int nc, int lane, int stride) {
  It2 t; t.nc = nc; t.tot = (nc > 0) ? nr * nc : 0; t.e = lane;
  t.row = (nc > 0) ? lane / nc : 0; t.col = lane - t.row * nc;
  t.dr = (nc > 0) ? stride / nc : 0; t.dc = stride - t.dr * nc;
  return t;
}
NB2_HD void it2_next(It2& t, int stride) { t.e += stride; t.row += t.dr; t.col += t.dc; if (t.col >= t.nc) { t.col -= t.nc; t.row++; } }
#if CW_DEV
#define CW_FOR2(R_, C_, nr, nc)                                                                                                   \
  for (nb2::cw::It2 R_##_t = nb2::cw::it2_begin((nr), (nc), (int)(threadIdx.x & 31), 32); R_##_t.e - (int)(threadIdx.x & 31) < R_##_t.tot; nb2::cw::it2_next(R_##_t, 32)) \
    for (int R_ = R_##_t.row, C_ = R_##_t.col, R_##_1 = 1; R_##_1; R_##_1 = 0)                                                    \
      if (R_##_t.e < R_##_t.tot)
#else
#define CW_FOR2(R_, C_, nr, nc)                                                                           \
  for (nb2::cw::It2 R_##_t = nb2::cw::it2_begin((nr), (nc), 0, 1); R_##_t.e < R_##_t.tot; nb2::cw::it2_next(R_##_t, 1)) \
    for (int R_ = R_##_t.row, C_ = R_##_t.col, R_##_1 = 1; R_##_1; R_##_1 = 0)
#endif

// ---- optional per-phase cycle counters (-DNB2_CW_PROFILE; dev builds only): lane 0 adds clock64() deltas to a global table
#if defined(NB2_CW_PROFILE) && defined(__CUDACC__)
__device__ unsigned long long nb2_cw_prof[64];
#endif
#if defined(NB2_CW_PROFILE) && CW_DEV
#define CW_PROF_DECL long long cw_t0_ = clock64()
#define CW_PROF(k) do { const long long cw_t1_ = clock64(); if (CW_LANE == 0) atomicAdd(&nb2_cw_prof[k], (unsigned long long)(cw_t1_ - cw_t0_)); cw_t0_ = clock64(); } while (0)
#else
#define CW_PROF_DECL
#define CW_PROF(k)
#endif

// Block-level phase barrier (solve kernel with several worlds per block, NB2_CW_LOCKSTEP): the warps of a block enter every phase of
// the chain together, so that they fetch the same code at the same time (the kernels are instruction-fetch bound: each warp wandering
// through its own part of a few hundred KB of code thrashes the instruction caches).  A warp that skips a phase just waits.
#if CW_DEV
#define CW_PHASE() __syncthreads()
#else
#define CW_PHASE() ((void)0)
#endif
#define NB2_CHAIN_PHASES 6

// per-lane partial -> the same total in every lane (host: the loop before it already produced the total)
NB2_HD double cw_sum(double a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(CW_FULL, a, off);
#endif
  return a;
}
NB2_HD double cw_max(double a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { const double o = __shfl_xor_sync(CW_FULL, a, off); a = o > a ? o : a; }
#endif
  return a;
}
NB2_HD int cw_isum(int a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(CW_FULL, a, off);
#endif
  return a;
}
NB2_HD int cw_imin(int a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { const int o = __shfl_xor_sync(CW_FULL, a, off); a = o < a ? o : a; }
#endif
  return a;
}
NB2_HD bool cw_any(bool p) {
#if CW_DEV
  return __any_sync(CW_FULL, p);
#else
  return p;
#endif
}
// value + position; "better" = larger (Max) / smaller (Min) value, ties -> LOWER position (what a serial scan with a strict
// comparison keeps).  pos < 0 = no candidate yet (v then holds the threshold a candidate has to beat strictly).
struct VI { double v; int i; };
NB2_HD void vi_max(VI& b, double d, int i) { if (b.i < 0 ? d > b.v : (d > b.v || (d == b.v && i < b.i))) { b.v = d; b.i = i; } }
NB2_HD void vi_min(VI& b, double d, int i) { if (b.i < 0 ? d < b.v : (d < b.v || (d == b.v && i < b.i))) { b.v = d; b.i = i; } }
NB2_HD VI cw_vi_max(VI a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    VI o; o.v = __shfl_xor_sync(CW_FULL, a.v, off); o.i = __shfl_xor_sync(CW_FULL, a.i, off);
    if (o.i >= 0 && (a.i < 0 || o.v > a.v || (o.v == a.v && o.i < a.i))) a = o;
  }
#endif
  return a;
}
NB2_HD VI cw_vi_min(VI a) {
#if CW_DEV
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    VI o; o.v = __shfl_xor_sync(CW_FULL, a.v, off); o.i = __shfl_xor_sync(CW_FULL, a.i, off);
    if (o.i >= 0 && (a.i < 0 || o.v < a.v || (o.v == a.v && o.i < a.i))) a = o;
  }
#endif
  return a;
}
// ranks: for every i < n with pred(i), write(i, number of j < i with pred(j)); returns the count.  Uniform call.
template <class P, class Wr> NB2_HD int cw_enumerate(int n, const P& pred, const Wr& write) {
  int cnt = 0;
#if CW_DEV
  const int lane = CW_LANE;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const bool f = (i < n) && pred(i);
    const unsigned bal = __ballot_sync(CW_FULL, f);
    if (f) write(i, cnt + __popc(bal & ((1u << lane) - 1u)));
    cnt += __popc(bal);
  }
#else
  for (int i = 0; i < n; i++) if (pred(i)) { write(i, cnt); cnt++; }
#endif
  return cnt;
}

// ---- triangular solves with the unknowns in registers (device) / plain loops (host).  L(r, k) = Lp[rm(r) * ld + k] for k < r,
// rm = identity when rowmap == nullptr; UNIT: unit diagonal, else the diagonal sits in the matrix.  n <= 64.
// Each y_r receives its subtractions in the order k = 0 .. r-1 (lower) / k = n-1 .. r+1 (upper): the serial order.
template <bool UNIT> NB2_HDN void trsv_lower(int n, const double* Lp, int ld, const int* rowmap, double* y) {
#if CW_DEV
  const int lane = CW_LANE, r0 = lane, r1 = lane + 32;
  const double* row0 = Lp + (size_t)((r0 < n) ? (rowmap ? rowmap[r0] : r0) : 0) * ld;
  const double* row1 = Lp + (size_t)((r1 < n) ? (rowmap ? rowmap[r1] : r1) : 0) * ld;
  double s0 = (r0 < n) ? y[r0] : 0.0, s1 = (r1 < n) ? y[r1] : 0.0;
  double id0 = 1.0, id1 = 1.0;
  if (!UNIT) { if (r0 < n) id0 = nb2_rcp(row0[r0]); if (r1 < n) id1 = nb2_rcp(row1[r1]); }
  const int n0 = n < 32 ? n : 32;
#pragma unroll 4
  for (int k = 0; k < n0; k++) {
    if (!UNIT && lane == k) s0 *= id0;
    const double yk = __shfl_sync(CW_FULL, s0, k);
    if (r0 > k && r0 < n) s0 -= row0[k] * yk;
    if (r1 < n) s1 -= row1[k] * yk;
  }
  for (int k = 32; k < n; k++) {
    if (!UNIT && lane == k - 32) s1 *= id1;
    const double yk = __shfl_sync(CW_FULL, s1, k - 32);
    if (r1 > k && r1 < n) s1 -= row1[k] * yk;
  }
  if (r0 < n) y[r0] = s0;
  if (r1 < n) y[r1] = s1;
  __syncwarp();
#else
  for (int r = 0; r < n; r++) {
    const double* row = Lp + (size_t)(rowmap ? rowmap[r] : r) * ld;
    double s = y[r];
    for (int k = 0; k < r; k++) s -= row[k] * y[k];
    y[r] = UNIT ? s : s * nb2_rcp(row[r]);
  }
#endif
}
// L^T y = rhs (in place)
template <bool UNIT> NB2_HDN void trsv_lower_T(int n, const double* Lp, int ld, const int* rowmap, double* y) {
#if CW_DEV
  const int lane = CW_LANE, j0 = lane, j1 = lane + 32;
  double s0 = (j0 < n) ? y[j0] : 0.0, s1 = (j1 < n) ? y[j1] : 0.0;
  double id0 = 1.0, id1 = 1.0;
  if (!UNIT) {
    if (j0 < n) id0 = nb2_rcp(Lp[(size_t)(rowmap ? rowmap[j0] : j0) * ld + j0]);
    if (j1 < n) id1 = nb2_rcp(Lp[(size_t)(rowmap ? rowmap[j1] : j1) * ld + j1]);
  }
  for (int k = n - 1; k >= 32; k--) {
    if (!UNIT && lane == k - 32) s1 *= id1;
    const double yk = __shfl_sync(CW_FULL, s1, k - 32);
    const double* rowk = Lp + (size_t)(rowmap ? rowmap[k] : k) * ld;
    if (j1 < k) s1 -= rowk[j1] * yk;
    if (j0 < n) s0 -= rowk[j0] * yk;
  }
  const int n0 = n < 32 ? n : 32;
#pragma unroll 4
  for (int k = n0 - 1; k >= 0; k--) {
    if (!UNIT && lane == k) s0 *= id0;
    const double yk = __shfl_sync(CW_FULL, s0, k);
    const double* rowk = Lp + (size_t)(rowmap ? rowmap[k] : k) * ld;
    if (j0 < k) s0 -= rowk[j0] * yk;
  }
  if (j0 < n) y[j0] = s0;
  if (j1 < n) y[j1] = s1;
  __syncwarp();
#else
  for (int j = n - 1; j >= 0; j--) {
    double s = y[j];
    for (int k = n - 1; k > j; k--) s -= Lp[(size_t)(rowmap ? rowmap[k] : k) * ld + j] * y[k];
    y[j] = UNIT ? s : s * nb2_rcp(Lp[(size_t)(rowmap ? rowmap[j] : j) * ld + j]);
  }
#endif
}

// ------------------------------------------------------------------------------------------------ workspace
// Capacities of one world's workspace: MC contacts, MR LCP rows, LD = MR | 1 (odd leading dimension: row AND column walks of a
// matrix are bank-conflict free).  Problems are stored with their own leading dimension ld = m | 1 <= LD.
struct Dims { int nb, n, MC, MR, LD, ncb, cdofs, nfree, bwd, mode; size_t mats; };
// bytes of one pair slot of the collision phase: count, status, 8 contacts x (point, normal, depth, type)
#define NB2_CW_PAIR_SLOT 66
NB2_HD Dims make_dims(int nb, int n, int nfree, int MC, int MR, int ncb, int cdofs, int bwd = 0, int mode = 0) {
  Dims d; d.nb = nb; d.n = n; d.nfree = nfree; d.MC = MC; d.MR = MR; d.LD = MR | 1; d.ncb = ncb; d.cdofs = cdofs; d.bwd = bwd; d.mode = mode;
  // the two work matrices double as: private chain buffers of the impulse tests (one per row / collision body), spatial velocity
  // changes of all bodies (impulse application), pair slots of the collision phase (at least 4)
  size_t mats = 0;
  const size_t priv = (size_t)MR * cdofs, dv = (size_t)ncb * cdofs + (bwd ? (size_t)nb * 30 + 3 * (size_t)n + 32 : (size_t)nb * 6), slots = 4 * (size_t)NB2_CW_PAIR_SLOT;
  if (mode != 2) mats = 2 * (size_t)MR * d.LD;       // FULL / SOLVE: the two work matrices
  if (mode == 0 && mats < priv) mats = priv;          // FULL: private chain buffers of the impulse tests
  if (mode != 1 && mats < dv) mats = dv;              // FULL / APPLY: impulse application buffers
  if (mode == 0 && mats < slots) mats = slots;        // FULL: pair slots of the collision phase
  d.mats = mats;
  return d;
}
struct Ws {
  double *Wcb, *Vcb, *Fcb;      // [ncb][12], [ncb][6], [ncb][6]: world transform / spatial velocity (at v*) / net impulse of the collision bodies
  double *uI, *dqd;             // [n]
  double *Iinv;                 // [nfree][21] inverse articulated inertia of the FREE bodies (forward: written by the ABA pass)
  double *aeff, *vplus, *JcTmu, *inj;  // backward only: [n] [n] [n] [ncb][24]
  double *cpoint, *cnormal, *cdepth, *cmu, *crest;   // contacts
  int *cbodyA, *cbodyB, *ctype, *cshapeA, *cshapeB, *crow;  // crow: first LCP row of a contact
  double *JA, *JB;              // [MR][6] body-frame wrenches of a row on body A / B
  double *b, *lo, *hi, *x, *x0, *colnorm;
  int *findex, *mapping, *clampIdx, *ubIdx, *rowc;
  double *A, *M1, *M2;          // MR x LD each (M1|M2 contiguous: also the private buffers of the impulse tests)
  double *v1, *v2, *v3, *v4, *v5, *v6, *v7, *v8, *v9, *v10, *v11;
  int *i1, *i2, *i3, *i4;
  int *tbl;                     // [ncb] distinct bodies touched by this world's contacts
  int *meta;                    // [8]
};
// Which arrays a kernel needs.  The forward step is split into three kernels so that the expensive, register-light solver phase runs
// at a higher occupancy than the register-hungry tree sweeps and collision code allow: BUILD (everything; contacts, rows, A), SOLVE
// (the LCP and its work matrices only), APPLY (row wrenches, impulses, tree buffers).  Dims.mode selects the subset; absent arrays are
// nullptr.  The layout is a pure function of Dims, computed by one routine (count == true: size only).
#define NB2_WS_FULL 0
#define NB2_WS_SOLVE 1
#define NB2_WS_APPLY 2
NB2_HD size_t ws_layout(double* base, const Dims& d, Ws* out) {
  Ws w;
  size_t off = 0;
  const size_t MC = d.MC, MR = d.MR;
  const bool full = d.mode == NB2_WS_FULL, solve = d.mode != NB2_WS_APPLY, apply = d.mode != NB2_WS_SOLVE;
  auto D = [&](bool need, size_t cnt) -> double* { if (!need) return nullptr; double* r = base ? base + off : nullptr; off += cnt; return r; };
  auto I = [&](bool need, size_t cnt) -> int* { if (!need) return nullptr; int* r = base ? (int*)(base + off) : nullptr; off += (cnt + 1) / 2; return r; };
  w.Wcb = D(full, (size_t)d.ncb * 12); w.Vcb = D(full, (size_t)d.ncb * 6); w.Fcb = D(apply, (size_t)d.ncb * 6);
  w.uI = D(apply, d.n); w.dqd = D(apply, d.n); w.Iinv = D(full, (size_t)d.nfree * 21);
  const bool bw = full && d.bwd;
  w.aeff = D(bw, d.n); w.vplus = D(bw, d.n); w.JcTmu = D(bw, d.n); w.inj = D(bw, (size_t)d.ncb * 24);
  w.cpoint = D(full, MC * 3); w.cnormal = D(full, MC * 3); w.cdepth = D(full, MC); w.cmu = D(full, MC); w.crest = D(full, MC);
  w.cbodyA = I(apply, MC); w.cbodyB = I(apply, MC); w.ctype = I(full, MC); w.cshapeA = I(full, MC); w.cshapeB = I(full, MC); w.crow = I(full, MC);
  w.JA = D(apply, MR * 6); w.JB = D(apply, MR * 6);
  w.b = D(solve, MR); w.lo = D(solve, MR); w.hi = D(solve, MR); w.x = D(true, MR); w.x0 = D(solve, MR); w.colnorm = D(solve, MR);
  w.findex = I(solve, MR); w.mapping = I(solve, MR); w.clampIdx = I(solve, MR); w.ubIdx = I(solve, MR); w.rowc = I(apply, MR);
  w.A = D(solve, MR * d.LD);
  w.M1 = D(true, d.mats); w.M2 = solve ? w.M1 + MR * d.LD : nullptr;
  w.v1 = D(solve, MR); w.v2 = D(solve, MR); w.v3 = D(solve, MR); w.v4 = D(solve, MR); w.v5 = D(solve, MR); w.v6 = D(solve, MR); w.v7 = D(solve, MR);
  w.v8 = D(solve, MR); w.v9 = D(solve, MR); w.v10 = D(solve, MR); w.v11 = D(solve, MR);
  w.i1 = I(solve, MR); w.i2 = I(solve, MR); w.i3 = I(solve, MR); w.i4 = I(solve, MR);
  w.tbl = I(full, d.ncb);
  w.meta = I(true, 8);
  if (out) *out = w;
  return off;
}
NB2_HD size_t ws_doubles(const Dims& d) { return ws_layout(nullptr, d, nullptr); }
NB2_HD Ws carve(double* base, const Dims& d) { Ws w; ws_layout(base, d, &w); return w; }

// ------------------------------------------------------------------------------------------------ LCP validity
// LCPUtils::isLCPSolutionValid (LCPUtils.cpp:12-80), tol 1e-5; one row per lane.  Uniform call, uniform result.
NB2_HDN bool lcp_valid(int m, const double* A, int ld, const double* x, const double* b, const double* hi, const double* lo, const int* fi,
                      bool ignoreFriction) {
  bool bad = false;
  CW_FOR(i, m) {
    const double* row = A + (size_t)i * ld;
    double v = 0;
    for (int j = 0; j < m; j++) v += row[j] * x[j];
    v -= b[i];
    double up = hi[i], low = lo[i];
    bool skip = false;
    if (fi[i] != -1) { if (ignoreFriction) { if (x[i] != 0) bad = true; skip = true; } else { up *= x[fi[i]]; low *= x[fi[i]]; } }
    if (!skip) {
      const double tol = 1e-5;
      if (fabs(low) < tol && fabs(up) < tol && fabs(x[i]) < tol) {}
      else if (fabs(x[i] - low) < tol) { if (v < -tol) bad = true; }
      else if (fabs(x[i] - up) < tol) { if (v > tol) bad = true; }
      else if (x[i] > low && x[i] < up) { if (fabs(v) > tol) bad = true; }
      else bad = true;
    }
  }
  return !cw_any(bad);
}

// ------------------------------------------------------------------------------------------------ min-norm least squares
// x = Q^+ rhs for a symmetric PSD n x n matrix G (leading dimension ld), DESTROYED.  Rank-revealing pivoted Cholesky
// G = P L L^T P^T (L: n x r) and Q^+ = L (L^T L)^-2 L^T (replaces Eigen's completeOrthogonalDecomposition().solve,
// third party).  Lf: n x ld work matrix; t1, t2, t3: n doubles; perm: n ints.  x may alias nothing else.
NB2_HDN void pinv_psd(int n, double* G, int ld, const double* rhs, double* x, double* Lf, double* t1, double* t2, double* dg, int* perm) {
  double dmax0 = 0;
  CW_FOR(i, n) { perm[i] = i; const double d = G[(size_t)i * ld + i]; dg[i] = d; dmax0 = d > dmax0 ? d : dmax0; x[i] = 0; }
  dmax0 = cw_max(dmax0);
  CW_SYNC();
  const double tol = dmax0 * 1e-12;
  int r = 0;
  for (int k = 0; k < n; k++) {
    VI best; best.v = tol; best.i = -1;
    CW_FOR(i, n) if (i >= k) vi_max(best, dg[perm[i]], i);
    best = cw_vi_max(best);
    if (best.i < 0) break;
    const int pk = perm[best.i], pold = perm[k];
    CW_SYNC();  // everyone has read perm[] before it changes
    CW_ONE { perm[best.i] = pold; perm[k] = pk; }
    CW_SYNC();
    const double rlkk = nb2_rsqrt(best.v), lkk = best.v * rlkk;
    const double* Lk = Lf + (size_t)pk * ld;
    CW_FOR(i, n) {
      if (i == k) Lf[(size_t)pk * ld + k] = lkk;
      else if (i > k) {
        const int pi = perm[i];
        double* Li = Lf + (size_t)pi * ld;
        double s = G[(size_t)pi * ld + pk];
        for (int j = 0; j < k; j++) s -= Li[j] * Lk[j];
        const double l = s * rlkk;
        Li[k] = l;
        dg[pi] -= l * l;
      }
    }
    CW_SYNC();
    r++;
  }
  if (r == 0) { CW_SYNC(); return; }
  if (r == n) {  // full rank: Q^-1 = P L^-T L^-1 P^T
    CW_FOR(i, n) t1[i] = rhs[perm[i]];
    CW_SYNC();
    trsv_lower<false>(n, Lf, ld, perm, t1);
    trsv_lower_T<false>(n, Lf, ld, perm, t1);
    CW_FOR(i, n) x[perm[i]] = t1[i];
    CW_SYNC();
    return;
  }
  // rows of the pivoted indices carry garbage above their own column: zero it (L is n x r, "lower trapezoidal" in pivot order)
  CW_FOR(k, r) for (int j = k + 1; j < r; j++) Lf[(size_t)perm[k] * ld + j] = 0;
  CW_SYNC();
  // Mm = L^T L (r x r) into G ; y = L^T rhs
  CW_FOR2(a, c, r, r) {
    if (c >= a) {
      double s = 0;
      for (int i = 0; i < n; i++) s += Lf[(size_t)i * ld + a] * Lf[(size_t)i * ld + c];
      G[(size_t)a * ld + c] = s; G[(size_t)c * ld + a] = s;
    }
  }
  CW_FOR(a, r) { double ya = 0; for (int i = 0; i < n; i++) ya += Lf[(size_t)i * ld + a] * rhs[i]; t1[a] = ya; }
  CW_SYNC();
  // Cholesky of Mm in place (lower), column by column: every entry gets its subtractions in the serial order
  for (int j = 0; j < r; j++) {
    double d = G[(size_t)j * ld + j];
    for (int k = 0; k < j; k++) d -= G[(size_t)j * ld + k] * G[(size_t)j * ld + k];
    const double rd = nb2_rsqrt(d);
    d = d * rd;
    CW_SYNC();
    CW_FOR(i, r) {
      if (i == j) G[(size_t)j * ld + j] = d;
      else if (i > j) {
        double s = G[(size_t)i * ld + j];
        for (int k = 0; k < j; k++) s -= G[(size_t)i * ld + k] * G[(size_t)j * ld + k];
        G[(size_t)i * ld + j] = s * rd;
      }
    }
    CW_SYNC();
  }
  // z = Mm^-2 y : two Cholesky solves
  for (int rep = 0; rep < 2; rep++) {
    trsv_lower<false>(r, G, ld, nullptr, t1);
    trsv_lower_T<false>(r, G, ld, nullptr, t1);
  }
  CW_FOR(i, n) { double s = 0; for (int a = 0; a < r; a++) s += Lf[(size_t)i * ld + a] * t1[a]; x[i] = s; }
  CW_SYNC();
  (void)t2;
}

// ------------------------------------------------------------------------------------------------ classification
// ConstrainedGroupGradientMatrices::constructMatrices (labels) + opportunisticallyStandardizeResults (f_c = Q^+ b_c).
// Labels: normal rows (findex = -1) depend on their own data only; a friction row looks at the label of its normal row —
// two parallel phases.  x is updated in place when the standardised solution is valid.  Returns true when standardised.
NB2_HD bool classify_once(int m, const double* A, int ld, double* x, const double* b, const double* lo, const double* hi, const int* fi,
                          const double* colnorm, bool ignoreFriction, const Ws& ws, bool* again) {
  *again = false;
  int* mapping = ws.mapping; int* clampIdx = ws.clampIdx; int* ubIdx = ws.ubIdx;
  for (int phase = 0; phase < 2; phase++) {
    CW_FOR(j, m) {
      const int fp = fi[j];
      if ((phase == 0) != (fp == -1)) continue;
      int lab;
      if (colnorm[j] < 1e-9) lab = NB2_MAP_NOT_CLAMPING;
      else {
        double up = hi[j], low = lo[j];
        if (fp != -1) { up *= x[fp]; low *= x[fp]; }
        if (fabs(x[j]) < 1e-6) {
          if (fp != -1) lab = (fabs(x[fp]) < 1e-6 || ignoreFriction) ? NB2_MAP_NOT_CLAMPING : NB2_MAP_CLAMPING;
          else lab = NB2_MAP_NOT_CLAMPING;
        } else {
          const double tie = 1e-5;
          if ((x[j] > low + tie && x[j] < up - tie) || (low - x[j] > 1e-2 || x[j] - up > 1e-2)) lab = NB2_MAP_CLAMPING;
          else if (fp != -1 && fabs(x[fp]) > 1e-9 && colnorm[fp] > 1e-9 && ((fp > j) || mapping[fp] == NB2_MAP_CLAMPING)) lab = fp;
          else lab = NB2_MAP_NOT_CLAMPING;
        }
      }
      mapping[j] = lab;
    }
    CW_SYNC();
  }
  // NB: a friction row whose normal row comes LATER (fp > j) never looks at mapping[fp]; normal rows precede their friction
  // rows in every problem this stage builds, and the general case is covered by the phase order above.
  int* cl = ws.i1; int* ub = ws.i2;
  const int nCl = cw_enumerate(m, [&](int j) { return mapping[j] == NB2_MAP_CLAMPING; }, [&](int j, int r) { cl[r] = j; });
  const int nUb = cw_enumerate(m, [&](int j) { return mapping[j] >= 0; }, [&](int j, int r) { ub[r] = j; });
  CW_FOR(j, m) { clampIdx[j] = -1; ubIdx[j] = -1; }
  CW_SYNC();
  CW_FOR(r, nCl) clampIdx[cl[r]] = r;
  CW_FOR(u, nUb) ubIdx[ub[u]] = u;
  CW_SYNC();
  // ---- opportunisticallyStandardizeResults
  if (nCl == 0) {
    CW_FOR(i, m) ws.v1[i] = 0;
    CW_SYNC();
    const bool ok = lcp_valid(m, A, ld, ws.v1, b, hi, lo, fi, ignoreFriction);
    if (ok) { CW_FOR(i, m) x[i] = 0; CW_SYNC(); }
    return ok;
  }
  const int lq = nCl | 1;
  double* Q = ws.M1; double* bc = ws.v2; double* orig = ws.v3; double* fc = ws.v4;
  CW_FOR2(r, c, nCl, nCl) Q[(size_t)r * lq + c] = A[(size_t)cl[r] * ld + cl[c]];
  CW_FOR(r, nCl) { bc[r] = b[cl[r]]; orig[r] = x[cl[r]]; }
  CW_SYNC();
  if (nUb > 0) {
    // E(u, clampIdx[fp]) = hi or lo of the row; Q = A[cl,cl] + A[cl,ub] E  (each upper-bound row adds to ONE column: rows in parallel,
    // upper-bound rows in their serial order)
    CW_FOR(r, nCl) {
      for (int u = 0; u < nUb; u++) {
        const int j = ub[u], fp = mapping[j];
        const double up = x[fp] * hi[j], low = x[fp] * lo[j];
        const double e = (fabs(x[j] - up) < fabs(x[j] - low)) ? hi[j] : lo[j];
        Q[(size_t)r * lq + clampIdx[fp]] += A[(size_t)cl[r] * ld + j] * e;
      }
    }
    CW_SYNC();
    // general Q: f = (Q^T Q)^+ Q^T b
    double* QtQ = ws.M2; double* Qtb = ws.v7;
    CW_FOR2(a, c, nCl, nCl) {
      double t = 0; for (int r = 0; r < nCl; r++) t += Q[(size_t)r * lq + a] * Q[(size_t)r * lq + c];
      QtQ[(size_t)a * lq + c] = t;
    }
    CW_FOR(a, nCl) { double s = 0; for (int r = 0; r < nCl; r++) s += Q[(size_t)r * lq + a] * bc[r]; Qtb[a] = s; }
    CW_SYNC();
    pinv_psd(nCl, QtQ, lq, Qtb, fc, Q /* Lf */, ws.v5, ws.v6, ws.v9, ws.i3);
  } else {
    pinv_psd(nCl, Q, lq, bc, fc, ws.M2, ws.v5, ws.v6, ws.v9, ws.i3);
  }
  bool anyNew = false;
  double* nx = ws.v8;
  CW_FOR(i, m) {
    double v = 0;
    if (clampIdx[i] != -1) {
      v = fc[clampIdx[i]];
      if (fabs(v) < 1e-6 && fabs(x[i]) > 1e-6 && fi[i] == -1) anyNew = true;
    }
    if (ubIdx[i] != -1) {
      const int fp = fi[i];
      const double origMult = nb2_div(orig[clampIdx[fp]], x[i]);
      const double clean = (fabs(origMult - hi[i]) < fabs(origMult - lo[i])) ? hi[i] : lo[i];
      v = fc[clampIdx[fp]] * clean;
    }
    nx[i] = v;
  }
  anyNew = cw_any(anyNew);
  CW_SYNC();
  if (lcp_valid(m, A, ld, nx, b, hi, lo, fi, ignoreFriction)) {
    CW_FOR(i, m) x[i] = nx[i];
    CW_SYNC();
    *again = anyNew;  // a previously clamping normal row dropped to ~0: re-classify (:283-331)
    return true;
  }
  return false;
}
NB2_HDN bool classify_and_standardize(int m, const double* A, int ld, double* x, const double* b, const double* lo, const double* hi,
                                      const int* fi, const double* colnorm, bool ignoreFriction, const Ws& ws_) {
  const Ws ws = ws_;  // array pointers into registers (the descriptor itself lives in shared memory / the caller's frame)
  bool ok = false, again = false;
  for (int it = 0; it < 6; it++) {
    ok = classify_once(m, A, ld, x, b, lo, hi, fi, colnorm, ignoreFriction, ws, &again);
    if (!ok || !again) break;
  }
  return ok;
}

// ------------------------------------------------------------------------------------------------ PGS
// PgsBoxedLcpSolver::solve with Option(30, 1e-6, 1e-3, 1e-9, false) (PgsBoxedLcpSolver.cpp:79-278); A (m x m, ld) and b are
// clobbered.  Gauss-Seidel is sequential in the rows; what is spread over the lanes is the row residual: lane j keeps
// r_j = sum_k A_jk x_k up to date (one FMA per accepted change of some x_i), so a row update costs O(1) on its dependent chain
// instead of an m-term inner product.  r is recomputed from scratch at the start of every sweep (no drift).
NB2_HDN bool pgs_solve(int m, double* A, int ld, double* x, double* b, const double* lo, const double* hi, const int* fi, double* r, int* skip) {
  const double dxTol = 1e-6, relTol = 1e-3, epsDiv = 1e-9;
#if CW_DEV && !defined(NB2_CW_PGS_SMEM)
  if (m <= 32) {
    // register form: lane j owns row j (x_j, its row residual r_j = sum_k A_jk x_k, b_j, bounds).  Per row step every lane evaluates the
    // update of ITS row (branch-free; only the owner's result is kept), the owner's change is broadcast and every lane folds it into its
    // residual with one multiply-add on the column entry A_ji.  Rows are rescaled in place after the first sweep like the reference
    // (PgsBoxedLcpSolver.cpp:163-180).  Same arithmetic, in the same order, as the shared-memory form below.
    const int lane = CW_LANE;
    const bool act = lane < m;
    double* rowj = A + (size_t)(act ? lane : 0) * ld;
    double xj = act ? x[lane] : 0.0, bj = act ? b[lane] : 0.0;
    const double hij = act ? hi[lane] : 0.0, loj = act ? lo[lane] : 0.0;
    double ajj = act ? rowj[lane] : 1.0;
    const int fj = act ? fi[lane] : -1;
    const int fsrc = fj >= 0 ? fj : 0;
    bool skipj = false;
    auto residual = [&]() {
      double rr = 0;
      for (int k = 0; k < m; k++) { const double xk = __shfl_sync(CW_FULL, xj, k); if (act) rr += rowj[k] * xk; }
      return rr;
    };
    double rj = residual();
    bool changed = false;
    // first sweep: unscaled rows, division by the diagonal, absolute change test
    // xf: x of this lane's own normal row, kept in a register and refreshed from the broadcast of row fsrc's new value (the two broadcasts of a
    // step are independent of each other, so they overlap; reading x[fsrc] by a shuffle at the start of every step put two dependent
    // shuffles on the critical path of each row.  Measured: no change in the step time — the sweep is bound elsewhere)
    double xf = __shfl_sync(CW_FULL, xj, fsrc);
#pragma unroll 2
    for (int i = 0; i < m; i++) {
      const bool own = lane == i;
      const bool sk = ajj < epsDiv;
      const double nx = nb2_div(bj - (rj - ajj * xj), sk ? 1.0 : ajj);
      const double hi_t = fj >= 0 ? hij * xf : hij, lo_t = fj >= 0 ? -hi_t : loj;
      double xi = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
      xi = sk ? 0.0 : xi;
      const double dl = own ? xi - xj : 0.0;
      changed = changed || (own && !sk && fabs(dl) > dxTol);
      skipj = skipj || (own && sk);
      xj = own ? xi : xj;
      const double delta = __shfl_sync(CW_FULL, dl, i);
      const double xnew = __shfl_sync(CW_FULL, xj, i);
      if (fsrc == i) xf = xnew;
      if (act) rj = fma(A[(size_t)lane * ld + i], delta, rj);
    }
    bool term = !__any_sync(CW_FULL, changed);
    if (!term) {
      if (act && !skipj) { const double dm = nb2_rcp(ajj); bj *= dm; for (int k = 0; k < m; k++) rowj[k] *= dm; ajj = rowj[lane]; }
      __syncwarp();
      for (int iter = 1; iter < 30; iter++) {
        rj = residual();
        changed = false;
#pragma unroll 4
        for (int i = 0; i < m; i++) {
          const bool own = (lane == i) && !skipj;
          const double nx = bj - (rj - ajj * xj);
          const double hi_t = fj >= 0 ? hij * xf : hij, lo_t = fj >= 0 ? -hi_t : loj;
          const double xi = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
          const double dl = own ? xi - xj : 0.0;
          changed = changed || (own && fabs(xi) > epsDiv && fabs(dl) > relTol * fabs(xi));
          xj = own ? xi : xj;
          const double delta = __shfl_sync(CW_FULL, dl, i);
          const double xnew = __shfl_sync(CW_FULL, xj, i);
          if (fsrc == i) xf = xnew;
          if (act) rj = fma(A[(size_t)lane * ld + i], delta, rj);
        }
        term = !__any_sync(CW_FULL, changed);
        if (term) break;
      }
    }
    if (act) x[lane] = xj;
    __syncwarp();
    return term;
  }
#endif
  auto residuals = [&]() {
    CW_FOR(j, m) { const double* row = A + (size_t)j * ld; double s = 0; for (int k = 0; k < m; k++) s += row[k] * x[k]; r[j] = s; }
    CW_SYNC();
  };
  residuals();
  bool term = true;
  for (int i = 0; i < m; i++) {  // first sweep: unscaled rows (:120-160)
    const double aii = A[(size_t)i * ld + i], old_x = x[i];
    double xi;
    int sk = 0;
    if (aii < epsDiv) { xi = 0.0; sk = 1; }
    else {
      const double nx = nb2_div(b[i] - (r[i] - aii * old_x), aii);
      double hi_t = hi[i], lo_t = lo[i];
      const int f = fi[i];
      if (f >= 0) { hi_t = hi[i] * x[f]; lo_t = -hi_t; }
      xi = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
      if (term && fabs(xi - old_x) > dxTol) term = false;
    }
    const double delta = xi - old_x;
    CW_SYNC();  // every lane has read x[i], r[i] before they change
    CW_FOR(j, m) r[j] += A[(size_t)j * ld + i] * delta;  // column i (a reduced problem has doubled columns: not symmetric)
    CW_ONE { x[i] = xi; skip[i] = sk; }
    CW_SYNC();
  }
  if (term) return true;
  CW_FOR(i, m) if (!skip[i]) {
    double* row = A + (size_t)i * ld;
    const double dm = nb2_rcp(row[i]);
    b[i] *= dm;
    for (int j = 0; j < m; j++) row[j] *= dm;
  }
  CW_SYNC();
  for (int iter = 1; iter < 30; iter++) {
    residuals();
    term = true;
    for (int i = 0; i < m; i++) {
      if (skip[i]) continue;
      const double old_x = x[i];
      const double nx = b[i] - (r[i] - A[(size_t)i * ld + i] * old_x);
      double hi_t = hi[i], lo_t = lo[i];
      const int f = fi[i];
      if (f >= 0) { hi_t = hi[i] * x[f]; lo_t = -hi_t; }
      const double xi = nx > hi_t ? hi_t : (nx < lo_t ? lo_t : nx);
      if (term && fabs(xi) > epsDiv) { if (fabs(xi - old_x) > relTol * fabs(xi)) term = false; }
      const double delta = xi - old_x;
      CW_SYNC();
      CW_FOR(j, m) r[j] += A[(size_t)j * ld + i] * delta;  // rows were rescaled: column i
      CW_ONE x[i] = xi;
      CW_SYNC();
    }
    if (term) break;
  }
  return term;
}

// ------------------------------------------------------------------------------------------------ reduce
// LCPUtils::reduce (LCPUtils.cpp:144-201) + mergeLCPColumns (:346-444): near-identical columns (same bounds, findex,
// |b_a - b_b| < 1e-4, ||A_a - A_b||^2 < 1e-4 over the CURRENT problem) are merged one pair at a time — column a doubled,
// row/column b dropped — until none is left.  Instead of compacting after every merge the state is kept on the ORIGINAL
// indices: alive[i], mult[i] (2^merges of a kept column), target[i] (the kept column an index was merged into; the un-merge
// map x = mapOut * x_r has exactly one 1 per row) and fcur[i] (findex with merged normals redirected).  The reduced problem is
// gathered once at the end: Ar (ldr = mr | 1), xr, br, lor, hir, fir.  Returns mr; keep[] lists the kept indices.
NB2_HDN int lcp_reduce(int m, const double* A, int ld, const double* x, const double* b, const double* lo, const double* hi, const int* fi,
                      double* Ar, double* xr, double* br, double* lor, double* hir, int* fir,
                      double* mult, int* alive, int* target, int* fcur, int* keep) {
  CW_FOR(i, m) { mult[i] = 1.0; alive[i] = 1; target[i] = i; fcur[i] = fi[i]; }
  CW_SYNC();
  for (;;) {
    int first = 0x7fffffff;
    CW_FOR2(a, c, m, m) {
      const int p = a * m + c;
      if (c <= a || !alive[a] || !alive[c] || p > first) continue;
      if (fcur[a] != fcur[c] || hi[a] != hi[c] || lo[a] != lo[c] || !(fabs(b[a] - b[c]) < 1e-4)) continue;
      const double ma = mult[a], mc = mult[c];
      double d2 = 0;
      for (int r = 0; r < m; r++) if (alive[r]) { const double d = A[(size_t)r * ld + a] * ma - A[(size_t)r * ld + c] * mc; d2 += d * d; }
      if (d2 < 1e-4 && p < first) first = p;
    }
    first = cw_imin(first);
    if (first == 0x7fffffff) break;
    const int ca = first / m, cb = first - ca * m;
    CW_SYNC();
    CW_FOR(i, m) {
      if (target[i] == cb) target[i] = ca;
      if (fcur[i] == cb) fcur[i] = ca;
      if (i == cb) alive[i] = 0;
      if (i == ca) mult[i] *= 2.0;
    }
    CW_SYNC();
  }
  const int mr = cw_enumerate(m, [&](int i) { return alive[i] != 0; }, [&](int i, int r) { keep[r] = i; });
  CW_SYNC();
  // rank of an original (kept) index in the reduced problem: alive[] is reused as rank + 1 for kept indices (0 = dropped)
  CW_FOR(r, mr) alive[keep[r]] = r + 1;
  CW_SYNC();
  const int ldr = mr | 1;
  CW_FOR2(ri, ci, mr, mr) { Ar[(size_t)ri * ldr + ci] = A[(size_t)keep[ri] * ld + keep[ci]] * mult[keep[ci]]; }
  CW_FOR(ri, mr) {
    const int i = keep[ri];
    xr[ri] = x[i]; br[ri] = b[i]; lor[ri] = lo[i]; hir[ri] = hi[i];
    fir[ri] = (fcur[i] < 0) ? -1 : alive[fcur[i]] - 1;
  }
  CW_SYNC();
  return mr;
}
// x[i] = x_r[rank(target[i])]
NB2_HD void lcp_unreduce(int m, const double* xr, const int* alive /* rank + 1 */, const int* target, double* x) {
  CW_FOR(i, m) x[i] = xr[alive[target[i]] - 1];
  CW_SYNC();
}

// ------------------------------------------------------------------------------------------------ Dantzig
// dSolveLCP / dLCP (dart/external/odelcpsolver/lcp.cpp:362-1114) for problems without unbounded rows (contact problems:
// nub = 0).  Same physical permutation of the problem, same loop orders and strict comparisons as the reference, so the same
// index sets are reached; the dense linear algebra is spread over the lanes:
//   * A is a full symmetric n x n matrix (ld odd), swapped in place (rows then columns, one element per lane);
//   * L D L^T of A[C,C]: rows appended from the latest solve1 (lcp.cpp:503-535); rebuilt column by column when an index leaves C
//     (the reference downdates with dLDLTRemove: identical in exact arithmetic);
//   * solve1's two triangular solves run with the unknowns in registers (trsv_lower / trsv_lower_T);
//   * delta_w(N) = A(N,C) delta_x(C): one row per lane; the ratio test is a (value, position) arg-min whose positions follow the
//     order of the serial scans (driving row, its bound, N rows, C rows lo-then-hi).
struct DzWork {
  double *A; int ld;
  double *x, *b, *w, *lo, *hi, *L, *d, *delta_x, *delta_w, *Dell, *ell, *tmp;
  int *findex, *p, *C, *state;
};
NB2_HD void dz_swap(const DzWork& W, int n, int i1, int i2) {
  if (i1 == i2) return;
  CW_FOR(k, n) { double* r1 = W.A + (size_t)i1 * W.ld; double* r2 = W.A + (size_t)i2 * W.ld; const double t = r1[k]; r1[k] = r2[k]; r2[k] = t; }
  CW_SYNC();
  CW_FOR(k, n) { double* r = W.A + (size_t)k * W.ld; const double t = r[i1]; r[i1] = r[i2]; r[i2] = t; }
  CW_ONE {
#define NB2_SW(arr, T) { T t = W.arr[i1]; W.arr[i1] = W.arr[i2]; W.arr[i2] = t; }
    NB2_SW(x, double) NB2_SW(b, double) NB2_SW(w, double) NB2_SW(lo, double) NB2_SW(hi, double)
    NB2_SW(p, int) NB2_SW(state, int) NB2_SW(findex, int)
#undef NB2_SW
  }
  CW_SYNC();
}
// L D L^T of A[C,C] (C in factor order); d holds the reciprocals like ODE's m_d.  Column by column.
NB2_HD void dz_factor(const DzWork& W, int nC) {
  const int ld = W.ld;
  for (int j = 0; j < nC; j++) {
    const int cj = W.C[j];
    const double* Lj = W.L + (size_t)j * ld;
    // row j scaled back by the pivots once (L_jk / d_k with d the RECIPROCAL pivots), instead of one division per lane and term
    CW_FOR(k, j) W.Dell[k] = nb2_div(Lj[k], W.d[k]);
    CW_SYNC();
    CW_FOR(i, nC) if (i >= j) {
      const double* Li = W.L + (size_t)i * ld;
      double s = W.A[(size_t)W.C[i] * ld + cj];
      for (int k = 0; k < j; k++) s -= Li[k] * W.Dell[k];
      W.tmp[i] = s;
    }
    CW_SYNC();
    const double dj = nb2_rcp(W.tmp[j]);
    CW_FOR(i, nC) { if (i > j) W.L[(size_t)i * ld + j] = W.tmp[i] * dj; else if (i == j) W.d[j] = dj; }
    CW_SYNC();
  }
}
// solve1 (lcp.cpp:703-753): Dell = L \ A[C,i] ; ell = Dell .* d ; a[C] = -dir * L^T \ ell
NB2_HD void dz_solve1(const DzWork& W, int nC, double* a, int i, int dir, bool only_transfer) {
  if (nC <= 0) return;
  const double* Ai = W.A + (size_t)i * W.ld;
  CW_FOR(j, nC) W.Dell[j] = Ai[W.C[j]];
  CW_SYNC();
  trsv_lower<true>(nC, W.L, W.ld, nullptr, W.Dell);
  CW_FOR(j, nC) { const double e = W.Dell[j] * W.d[j]; W.ell[j] = e; W.tmp[j] = e; }
  CW_SYNC();
  if (only_transfer) return;
  trsv_lower_T<true>(nC, W.L, W.ld, nullptr, W.tmp);
  if (dir > 0) { CW_FOR(j, nC) a[W.C[j]] = -W.tmp[j]; } else { CW_FOR(j, nC) a[W.C[j]] = W.tmp[j]; }
  CW_SYNC();
}
// append index (physical slot i, about to be swapped into slot nC) using the ell / Dell of the latest solve1
NB2_HD void dz_append(const DzWork& W, int nC, int i) {
  double s = 0;
  CW_FOR(j, nC) { W.L[(size_t)nC * W.ld + j] = W.ell[j]; s += W.ell[j] * W.Dell[j]; }
  s = cw_sum(s);
  const double dd = nb2_rcp(W.A[(size_t)i * W.ld + i] - s);
  CW_ONE W.d[nC] = dd;
  CW_SYNC();
}
// returns 1 on success, 0 on early termination (s <= 0), -1 when the iteration cap is hit
NB2_HDN int dantzig_solve(const DzWork& W_, int n, bool early_termination) {
  const DzWork W = W_;  // pointers into registers: the caller's copy sits in local memory
  const double INF = HUGE_VAL;
  const int ld = W.ld;
  int nC = 0, nN = 0;
  CW_FOR(k, n) { W.x[k] = 0.0; W.w[k] = 0.0; W.p[k] = k; W.state[k] = 0; }
  CW_SYNC();
  // unbounded rows first (lcp.cpp:835-850; contact problems have none): factor A[0:nub, 0:nub] and solve for x there
  int nub = 0;
  for (int k = 0; k < n; k++) {
    if (W.findex[k] >= 0) continue;
    if (W.lo[k] == -INF && W.hi[k] == INF) { dz_swap(W, n, nub, k); nub++; }
  }
  if (nub > 0) {
    CW_FOR(k, nub) { W.C[k] = k; W.tmp[k] = W.b[k]; }
    CW_SYNC();
    dz_factor(W, nub);
    CW_FOR(k, nub) W.Dell[k] = W.b[k];
    CW_SYNC();
    trsv_lower<true>(nub, W.L, ld, nullptr, W.Dell);
    CW_FOR(k, nub) W.Dell[k] *= W.d[k];
    CW_SYNC();
    trsv_lower_T<true>(nub, W.L, ld, nullptr, W.Dell);
    CW_FOR(k, nub) W.x[k] = W.Dell[k];
    CW_SYNC();
    nC = nub;
  }
  // move friction rows to the end (lcp.cpp:491-501)
  {
    int num_at_end = 0;
    for (int k = n - 1; k >= nub; k--) {
      if (W.findex[k] >= 0) { dz_swap(W, n, k, n - 1 - num_at_end); num_at_end++; }
    }
  }
  bool hit_first_friction_index = false;
  long iter_cap = 200L * n + 1000;
  for (int i = nub; i < n; i++) {
    if (!hit_first_friction_index && W.findex[i] >= 0) {
      CW_FOR(j, n) W.delta_w[W.p[j]] = W.x[j];
      CW_SYNC();
      CW_FOR(k, n) if (k >= i) {
        const double wfk = W.delta_w[W.findex[k]];
        if (wfk == 0) { W.hi[k] = 0; W.lo[k] = 0; }
        else { const double h = fabs(W.hi[k] * wfk); W.hi[k] = h; W.lo[k] = -h; }
      }
      CW_SYNC();
      hit_first_friction_index = true;
    }
    {
      const double* Ai = W.A + (size_t)i * ld;
      double s = 0.0;
      CW_FOR(k, nC + nN) s += Ai[k] * W.x[k];
      s = cw_sum(s);
      const double wi = s - W.b[i];
      CW_SYNC();
      CW_ONE W.w[i] = wi;
      CW_SYNC();
    }
    const double wi0 = W.w[i];
    if (W.lo[i] == 0 && wi0 >= 0) { nN++; CW_ONE W.state[i] = 0; CW_SYNC(); }
    else if (W.hi[i] == 0 && wi0 <= 0) { nN++; CW_ONE W.state[i] = 1; CW_SYNC(); }
    else if (wi0 == 0) {
      dz_solve1(W, nC, W.delta_x, i, 0, true);
      dz_append(W, nC, i);
      dz_swap(W, n, nC, i);
      CW_ONE W.C[nC] = nC;
      CW_SYNC();
      nC++;
    } else {
      for (;;) {
        if (--iter_cap < 0) return -1;
        int dir; double dirf;
        if (W.w[i] <= 0) { dir = 1; dirf = 1.0; } else { dir = -1; dirf = -1.0; }
        dz_solve1(W, nC, W.delta_x, i, dir, false);
        // delta_w(N) = A(N,C) delta_x(C) + dir * A(N,i) ; delta_w(i) = A(i,C) delta_x(C) + A(i,i) dirf   (one row per lane)
        {
          const double* Ai = W.A + (size_t)i * ld;
          CW_FOR(k, nN + 1) {
            const int row = (k < nN) ? nC + k : i;
            const double* Ak = W.A + (size_t)row * ld;
            double s = 0.0;
            for (int j = 0; j < nC; j++) s += Ak[j] * W.delta_x[j];
            if (k < nN) W.delta_w[row] = (dir > 0) ? s + Ai[row] : s - Ai[row];
            else W.delta_w[i] = s + Ai[i] * dirf;
          }
          CW_SYNC();
        }
        // ratio test.  positions: 0 driving row to w = 0 (cmd 1) | 1 driving row to its bound (cmd 2/3) | 2 + k: N row k (cmd 4) |
        // 2 + nN + 2k, +1: C row k to lo (cmd 5) / hi (cmd 6).  The serial code initialises with position 0 and replaces on strict '<'.
        const double s_first = nb2_div(-W.w[i], W.delta_w[i]);
        VI best; best.v = s_first; best.i = 0;
        {
          VI loc; loc.v = INF; loc.i = -1;
          const int ncand = 1 + nN + 2 * nC;
          CW_FOR(q, ncand) {
            if (q == 0) {
              if (dir > 0) { if (W.hi[i] < INF) vi_min(loc, (W.hi[i] - W.x[i]) * dirf, 1); }
              else { if (W.lo[i] > -INF) vi_min(loc, (W.lo[i] - W.x[i]) * dirf, 1); }
            } else if (q <= nN) {
              const int ik = nC + q - 1;
              const double dw = W.delta_w[ik];
              if (!W.state[ik] ? dw < 0 : dw > 0) {
                if (!(W.lo[ik] == 0 && W.hi[ik] == 0)) vi_min(loc, nb2_div(-W.w[ik], dw), 1 + q);
              }
            } else {
              const int e = q - 1 - nN, k = e >> 1;
              const double dx = W.delta_x[k];
              if (k < nub) {}
              else if (!(e & 1)) { if (dx < 0 && W.lo[k] > -INF) vi_min(loc, nb2_div(W.lo[k] - W.x[k], dx), 2 + nN + e); }
              else { if (dx > 0 && W.hi[k] < INF) vi_min(loc, nb2_div(W.hi[k] - W.x[k], dx), 2 + nN + e); }
            }
          }
          loc = cw_vi_min(loc);
          if (loc.i >= 0 && loc.v < best.v) best = loc;  // strict: position 0 wins ties, as in the serial scan
        }
        const double s = best.v;
        int cmd = 1, si = 0;
        if (best.i == 1) cmd = (dir > 0) ? 3 : 2;
        else if (best.i >= 2 && best.i < 2 + nN) { cmd = 4; si = nC + best.i - 2; }
        else if (best.i >= 2 + nN) { const int e = best.i - 2 - nN; si = e >> 1; cmd = (e & 1) ? 6 : 5; }
        if (s <= 0.0) {
          if (early_termination) return 0;
          CW_SYNC();
          CW_FOR(k, n) if (k >= i) { W.x[k] = 0; W.w[k] = 0; }
          CW_SYNC();
          goto unpermute;  // the reference reports success in this case (lcp.cpp:1044-1050, 1113)
        }
        CW_SYNC();
        CW_FOR(k, nC + nN + 1) {
          if (k < nC) W.x[k] += s * W.delta_x[k];
          else if (k < nC + nN) W.w[k] += s * W.delta_w[k];
          else { W.x[i] += s * dirf; W.w[i] += s * W.delta_w[i]; }
        }
        CW_SYNC();
        switch (cmd) {
          case 1: CW_ONE W.w[i] = 0; CW_SYNC(); dz_append(W, nC, i); dz_swap(W, n, nC, i); CW_ONE W.C[nC] = nC; CW_SYNC(); nC++; break;
          case 2: CW_ONE { W.x[i] = W.lo[i]; W.state[i] = 0; } CW_SYNC(); nN++; break;
          case 3: CW_ONE { W.x[i] = W.hi[i]; W.state[i] = 1; } CW_SYNC(); nN++; break;
          case 4:  // transfer_i_from_N_to_C (lcp.cpp:538-590): its own forward solve, then append
            CW_ONE W.w[si] = 0;
            CW_SYNC();
            dz_solve1(W, nC, W.delta_x, si, 0, true);
            dz_append(W, nC, si);
            dz_swap(W, n, nC, si);
            CW_ONE W.C[nC] = nC;
            CW_SYNC();
            nN--; nC++;
            break;
          case 5:
          case 6: {
            CW_ONE {
              if (cmd == 5) { W.x[si] = W.lo[si]; W.state[si] = 0; } else { W.x[si] = W.hi[si]; W.state[si] = 1; }
              // transfer_i_from_C_to_N (lcp.cpp:602-646): drop si from the factor order, rename the slot nC-1 -> si
              int j = 0, last_idx = -1;
              for (; j < nC; j++) {
                if (W.C[j] == nC - 1) last_idx = j;
                if (W.C[j] == si) {
                  int k;
                  if (last_idx == -1) { for (k = j + 1; k < nC; k++) if (W.C[k] == nC - 1) break; }
                  else k = last_idx;
                  W.C[k] = W.C[j];
                  for (int mm = j; mm < nC - 1; mm++) W.C[mm] = W.C[mm + 1];
                  break;
                }
              }
            }
            CW_SYNC();
            dz_swap(W, n, si, nC - 1);
            nN++; nC--;
            dz_factor(W, nC);
            break;
          }
        }
        if (cmd <= 3) break;
      }
    }
  }
unpermute:
  CW_SYNC();
  CW_FOR(j, n) { W.tmp[j] = W.x[j]; W.delta_w[j] = W.w[j]; }
  CW_SYNC();
  CW_FOR(j, n) { W.x[W.p[j]] = W.tmp[j]; W.w[W.p[j]] = W.delta_w[j]; }
  CW_SYNC();
  return 1;
}

// ------------------------------------------------------------------------------------------------ solve chain
// BoxedLcpConstraintSolver::solveLcp (:352-789) on the problem held in the workspace (A with leading dimension ld = m | 1, b, lo, hi,
// findex): warm start -> short-circuit classification -> [reduce] Dantzig -> cfm + [reduce] PGS -> friction drop ->
// classification / standardisation.  x_cached: last step's solution when it has the same size, else nullptr
// (LCPUtils::guessSolution).  Leaves x in ws.x and the labels in ws.mapping; returns the status bits.
// ws: the caller's (register) copy of the workspace descriptor; ws_mem: the same descriptor at a stable address (shared memory on the
// device), handed to the non-inlined classification so that the register copy never has to be spilled for a call
#define NB2_HEAD_PHASES 2
#ifdef NB2_TAIL_FREE
#define NB2_TAIL_PHASES 2   /* experiment: Dantzig -> PGS -> friction drop without block-wide barriers in between */
#else
#define NB2_TAIL_PHASES 4
#endif
NB2_HD void lcp_colnorms(int m, const Ws& ws) {
  const int ld = m | 1;
  CW_FOR(c, m) { double sn = 0; for (int r = 0; r < m; r++) { const double a = ws.A[(size_t)r * ld + c]; sn += a * a; } ws.colnorm[c] = sn; }
  CW_SYNC();
}
// head of the chain: warm start + the short-circuit classification.  true: x / mapping hold the answer (status NB2_ST_SHORTCIRCUIT);
// false: x == x0 (the warm start) and the tail has to run.
NB2_HD bool lcp_chain_head(int m, const Ws& ws, const Ws& ws_mem, const double* x_cached) {
  CW_PROF_DECL;
  const int ld = m | 1;
  double* A = ws.A;
  double* b = ws.b; double* lo = ws.lo; double* hi = ws.hi; int* fi = ws.findex; double* x = ws.x; double* x0 = ws.x0;
  lcp_colnorms(m, ws);
  // ---- warm start: cached solution if it has the same size, else LCPUtils::guessSolution (LCPUtils.cpp:86-140)
  CW_PHASE();  // 1
  if (x_cached) { CW_FOR(i, m) x0[i] = x_cached[i]; CW_SYNC(); }
  else {
    CW_FOR(i, m) x0[i] = 0;
    int* gi = ws.i1;
    const int ng = cw_enumerate(m, [&](int i) { return fi[i] != -1 || b[i] > 0; }, [&](int i, int r) { gi[r] = i; });
    CW_SYNC();
    if (ng > 0) {
      const int lg = ng | 1;
      CW_FOR2(r, c, ng, ng) { ws.M1[(size_t)r * lg + c] = A[(size_t)gi[r] * ld + gi[c]]; }
      CW_FOR(r, ng) ws.v1[r] = b[gi[r]];
      CW_SYNC();
      pinv_psd(ng, ws.M1, lg, ws.v1, ws.v2, ws.M2, ws.v5, ws.v6, ws.v9, ws.i3);
      CW_FOR(r, ng) x0[gi[r]] = ws.v2[r];
      CW_SYNC();
    }
  }
  CW_FOR(i, m) x[i] = x0[i];
  CW_SYNC();
  CW_PROF(10);
  CW_PHASE();  // 2
  // ---- solve chain
  bool success = classify_and_standardize(m, A, ld, x, b, lo, hi, fi, ws.colnorm, false, ws_mem);
  CW_PROF(11);
  return success;
}
// tail of the chain (the short-circuit failed): [reduce] Dantzig -> cfm + [reduce] PGS -> friction drop -> classification.
// Entry: x == x0, colnorm valid.  Returns the status bits.
NB2_HD int lcp_chain_tail(int m, const Ws& ws, const Ws& ws_mem, double fallback_cfm) {
  int status = 0;
  CW_PROF_DECL;
  const int ld = m | 1;
  double* A = ws.A;
  double* b = ws.b; double* lo = ws.lo; double* hi = ws.hi; int* fi = ws.findex; double* x = ws.x; double* x0 = ws.x0;
  bool success = false;
  const bool shortCircuit = false;
  bool ignoredFriction = false;
  // reduced problem: matrix in M1, vectors v1 (b) v2 (lo) v3 (hi) v4 (x), findex i1; bookkeeping v9 (mult), i2 (alive -> rank + 1),
  // i3 (target), i4 (fcur), mapping (keep list: free until the final classification)
  double *Ar = ws.M1, *br = ws.v1, *lor = ws.v2, *hir = ws.v3, *xr = ws.v4;
  int* fir = ws.i1;
  CW_PHASE();  // 3
  if (success) status |= NB2_ST_SHORTCIRCUIT;
  else {
    status |= NB2_ST_DANTZIG;
    const int mr = lcp_reduce(m, A, ld, x, b, lo, hi, fi, Ar, xr, br, lor, hir, fir, ws.v9, ws.i2, ws.i3, ws.i4, ws.mapping);  // :596 reduce before Dantzig
    if (mr < m) status |= NB2_ST_MERGED;
    DzWork W;
    W.A = Ar; W.ld = mr | 1; W.x = xr; W.b = br; W.w = ws.v5; W.lo = lor; W.hi = hir; W.L = ws.M2; W.d = ws.v6; W.delta_x = ws.v7; W.delta_w = ws.v8;
    W.Dell = ws.v9; W.ell = ws.v10; W.tmp = ws.v11;  // v9 (mult) is dead once the reduced problem is gathered
    W.findex = fir; W.p = ws.clampIdx; W.C = ws.ubIdx; W.state = ws.i4;
    CW_PROF(12);
    const int rc = dantzig_solve(W, mr, true);
    CW_PROF(13);
    success = (rc == 1);
    if (success) {
      lcp_unreduce(m, xr, ws.i2, ws.i3, x);  // x = mapOut * x_reduced
      if (!lcp_valid(m, A, ld, x, b, hi, lo, fi, false)) success = false;
    }
    if (!success) status |= NB2_ST_DANTZIG_FAILED;
  }
  {
    bool nan = false;
    CW_FOR(i, m) if (x[i] != x[i]) nan = true;
    if (cw_any(nan)) { success = false; CW_SYNC(); CW_FOR(i, m) x[i] = 0; CW_SYNC(); status |= NB2_ST_NAN; }
  }
#ifndef NB2_TAIL_FREE
  CW_PHASE();  // 4
#endif
  if (!success) {
    CW_FOR(i, m) A[(size_t)i * ld + i] += fallback_cfm;  // :539-547 (both backups get the cfm; colnorms were taken before)
    CW_SYNC();
    status |= NB2_ST_PGS;
    const int mr = lcp_reduce(m, A, ld, x0, b, lo, hi, fi, Ar, xr, br, lor, hir, fir, ws.v9, ws.i2, ws.i3, ws.i4, ws.mapping);  // :551-557
    if (mr < m) status |= NB2_ST_MERGED;
    CW_PROF(14);
    success = pgs_solve(mr, Ar, mr | 1, xr, br, lor, hir, fir, ws.v5, ws.clampIdx);
    CW_PROF(15);
    if (success) {
      lcp_unreduce(m, xr, ws.i2, ws.i3, x);
      if (!lcp_valid(m, A, ld, x, b, hi, lo, fi, false)) success = false;
    }
  }
#ifndef NB2_TAIL_FREE
  CW_PHASE();  // 5
#endif
  if (!success) {
    ignoredFriction = true;
    status |= NB2_ST_FRICTION_DROPPED;
    int* nl = ws.i2;
    const int k = cw_enumerate(m, [&](int i) { return fi[i] == -1; }, [&](int i, int r) { nl[r] = i; });
    CW_SYNC();
    const int lk = k | 1;
    CW_FOR2(r, c, k, k) { Ar[(size_t)r * lk + c] = A[(size_t)nl[r] * ld + nl[c]]; }
    CW_FOR(r, k) { br[r] = b[nl[r]]; lor[r] = lo[nl[r]]; hir[r] = hi[nl[r]]; xr[r] = 0; ws.i4[r] = -1; }
    CW_SYNC();
    pgs_solve(k, Ar, lk, xr, br, lor, hir, ws.i4, ws.v5, ws.clampIdx);
    CW_FOR(i, m) x[i] = 0;
    CW_SYNC();
    CW_FOR(r, k) x[nl[r]] = xr[r];
    CW_SYNC();
  }
  {
    bool nan = false;
    CW_FOR(i, m) if (x[i] != x[i]) nan = true;
    if (cw_any(nan)) { CW_SYNC(); CW_FOR(i, m) x[i] = 0; CW_SYNC(); status |= NB2_ST_NAN; }
  }
  CW_PROF(16);
  CW_PHASE();  // 6
  if (!shortCircuit) {
    // classify works on x in place and only keeps the standardised x when valid
    if (!classify_and_standardize(m, A, ld, x, b, lo, hi, fi, ws.colnorm, ignoredFriction, ws_mem)) status |= NB2_ST_NOT_STANDARDIZED;
  }
  CW_PROF(17);
  return status;
}
// the whole chain (fused kernels, host emulation): same phase barriers as the split form
NB2_HD int lcp_chain(int m, const Ws& ws, const Ws& ws_mem, double fallback_cfm, const double* x_cached) {
  if (lcp_chain_head(m, ws, ws_mem, x_cached)) {
    for (int k = 0; k < NB2_TAIL_PHASES; k++) CW_PHASE();
    return NB2_ST_SHORTCIRCUIT;
  }
  return lcp_chain_tail(m, ws, ws_mem, fallback_cfm);
}

// ------------------------------------------------------------------------------------------------ tree data
// Where the per-body results of the ABA pass are read from: the forward kernel keeps them in the world's ABA scratch (FwdLayout,
// stride 1) + ws.Iinv; the backward kernel reads the saved stream of the world (world-major: word k at sv[k]).
struct TreeSrc {
  const double* scr; FwdLayout L; const double* Iinv;  // forward (scr != nullptr)
  const double* sv;                                      // backward
  const float* st;                                       // input state row (fp32): prismatic joint positions
  int nb, nfree;
};
NB2_HD Xf<double> ts_xf(const Nb2ModelDev<double>& M, const TreeSrc& S, int i) {
  const int jt = M.jtype[i];
  if (jt == NB2_JT_PRIS) return xf_pris(M, i, (double)S.st[M.dof_off[i]]);
  if (S.scr) {
    if (jt == NB2_JT_REV) { const double* b = S.scr + S.L.oBody + NB2_FWD_BODY_WORDS * i + 6; return xf_rev(M, i, b[0], b[1]); }
    return ldXf<double, 1>(S.scr + S.L.oFree + 18 * M.free_idx[i]);
  }
  if (jt == NB2_JT_REV) { const double* b = S.sv + i * 21 + 19; return xf_rev(M, i, b[0], b[1]); }
  return ldXf<double, 1>(S.sv + S.nb * 21 + M.free_idx[i] * 33 + 21);
}
NB2_HD V6<double> ts_U(const TreeSrc& S, int i) { return ld6<double, 1>(S.scr ? S.scr + S.L.oBody + NB2_FWD_BODY_WORDS * i + 8 : S.sv + i * 21 + 12); }
NB2_HD double ts_psi(const TreeSrc& S, int i) { return S.scr ? S.scr[S.L.oBody + NB2_FWD_BODY_WORDS * i + 14] : S.sv[i * 21 + 18]; }
NB2_HD SI<double> ts_Iinv(const Nb2ModelDev<double>& M, const TreeSrc& S, int i) {
  return ldSI<double, 1>(S.scr ? S.Iinv + 21 * M.free_idx[i] : S.sv + S.nb * 21 + M.free_idx[i] * 33);
}
NB2_HD int lowest_bit(unsigned long long m) {
#if CW_DEV
  return __ffsll((long long)m) - 1;
#else
  return __builtin_ctzll(m);
#endif
}
NB2_HD Xf<double> xf_mul(const Xf<double>& A, const Xf<double>& B) { Xf<double> C; C.R_ = mul(A.R_, B.R_); C.p = mul(A.R_, B.p) + A.p; return C; }
NB2_HD V3<double> xf_apply_inv(const Xf<double>& A, const V3<double>& x) { return mulT(A.R_, x - A.p); }
NB2_HD V6<double> ldv6(const double* p) { return ld6<double, 1>(p); }
NB2_HD void stv6(double* p, const V6<double>& v) { st6<double, 1>(p, v); }

// world transform (and spatial velocity for the joint velocities `vj`, may be nullptr) of every collision body: one body per lane,
// walking its ancestor chain root -> body (bodies are numbered in DFS pre-order: ancestors in ascending order)
NB2_HD void fk_collision_bodies(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const TreeSrc& S, const double* vj, const Ws& ws) {
  CW_FOR(k, C.ncb) {
    unsigned long long mask = C.anc_mask[C.cb_body[k]];
    Xf<double> W; V6<double> V = zero6<double>();
    bool first = true;
    while (mask) {
      const int j = lowest_bit(mask); mask &= mask - 1;
      const Xf<double> T = ts_xf(M, S, j);
      W = first ? T : xf_mul(W, T);
      if (vj) {
        V = first ? zero6<double>() : AdInvT(T, V);
        const int o = M.dof_off[j];
        if (M.jtype[j] == NB2_JT_REV) V.a.z += vj[o]; else if (M.jtype[j] == NB2_JT_PRIS) V.l.z += vj[o]; else V = V + ldv6(vj + o);
      }
      first = false;
    }
    stXf<double, 1>(ws.Wcb + 12 * k, W);
    stv6(ws.Vcb + 6 * k, V);
  }
  CW_SYNC();
}

// contacts of one collision pair (shape sa in frame Ta, shape sb in frame Tb), scalar-generic (plain doubles or dual numbers).
// Capsule vs box: libccd's MPR (third party) decides in the reference which part of the capsule touches; here the deeper end sphere
// is taken (identical on box faces), equal depths — a capsule lying flat — are flagged.
template <class S>
NB2_HD int pair_contacts(const Nb2ContactDev& C, int sa, int sb, const Xf<S>& Ta, const Xf<S>& Tb, ContactOutT<S>* co, int* status) {
  const int ta = C.shape_type[sa], tb = C.shape_type[sb];
  const V3<S> da = mk3<S>(S(C.shape_dims[sa][0]), S(C.shape_dims[sa][1]), S(C.shape_dims[sa][2]));
  const V3<S> db = mk3<S>(S(C.shape_dims[sb][0]), S(C.shape_dims[sb][1]), S(C.shape_dims[sb][2]));
  if (ta == 0 && tb == 0) return collide_box_box(da, Ta, db, Tb, C.clip_depth, co);
  if (ta == 0 && tb == 1) return collide_box_sphere(da, Ta, db.x, Tb, C.clip_depth, 0, false, co);
  if (ta == 1 && tb == 0) return collide_box_sphere(db, Tb, da.x, Ta, C.clip_depth, 0, true, co);
  if (ta == 1 && tb == 1) return round_contact(Ta.p, da.x, Tb.p, db.x, C.clip_depth, false, true, 6, co);
  if (ta == 2 && tb == 2) return collide_capsule_capsule(C.shape_dims[sa][1], da.x, Ta, C.shape_dims[sb][1], db.x, Tb, C.clip_depth, co);
  if (ta == 1 && tb == 2) return collide_sphere_capsule(da.x, Ta, C.shape_dims[sb][1], db.x, Tb, C.clip_depth, true, co);
  if (ta == 2 && tb == 1) return collide_sphere_capsule(db.x, Tb, C.shape_dims[sa][1], da.x, Ta, C.clip_depth, false, co);
  if ((ta == 0 && tb == 2) || (ta == 2 && tb == 0)) {
    const bool boxFirst = (ta == 0);
    const Xf<S>& Tc = boxFirst ? Tb : Ta; const Xf<S>& Tbx = boxFirst ? Ta : Tb;
    const V3<S> bdim = boxFirst ? da : db;
    const S r = boxFirst ? db.x : da.x; const double h = boxFirst ? C.shape_dims[sb][1] : C.shape_dims[sa][1];
    double dep[2]; Xf<S> Tend[2];
    for (int e = 0; e < 2; e++) {
      Tend[e] = Tc; Tend[e].p = gxf_apply(Tc, mk3<S>(S(0.0), S(0.0), S(e == 0 ? h / 2 : -h / 2)));
      const V3<S> pld = gxf_apply_inv(Tbx, Tend[e].p);
      const double pl[3] = {gval(pld.x), gval(pld.y), gval(pld.z)};
      double q[3] = {pl[0], pl[1], pl[2]};
      bool inside = true;
      for (int kk = 0; kk < 3; kk++) { const double hk = 0.5 * gval(gget3(bdim, kk)); if (q[kk] < -hk) { q[kk] = -hk; inside = false; } if (q[kk] > hk) { q[kk] = hk; inside = false; } }
      if (inside) { double mn = 1e300; for (int kk = 0; kk < 3; kk++) { const double v = 0.5 * gval(gget3(bdim, kk)) - fabs(pl[kk]); mn = v < mn ? v : mn; } dep[e] = mn + gval(r); }
      else { const double dx = pl[0] - q[0], dy = pl[1] - q[1], dz = pl[2] - q[2]; dep[e] = gval(r) - sqrt(dx * dx + dy * dy + dz * dz); }
    }
    if ((dep[0] > dep[1] ? dep[0] : dep[1]) >= 0) {
      if (fabs(dep[0] - dep[1]) < 1e-9) { *status |= NB2_ST_UNSUPPORTED_GEOMETRY; return 0; }
      const int e = dep[0] > dep[1] ? 0 : 1;
      return collide_box_sphere(bdim, Tbx, r, Tend[e], C.clip_depth, e == 0 ? 1 : 2, !boxFirst, co);
    }
    return 0;
  }
  *status |= NB2_ST_UNSUPPORTED_GEOMETRY;
  return 0;
}
NB2_HD Xf<double> shape_pose(const Nb2ContactDev& C, const Ws& ws, int sh) {
  const Xf<double> Ts = ldXf<double, 1>(C.shape_T[sh]);
  const int bdy = C.shape_body[sh];
  return (bdy >= 0) ? xf_mul(ldXf<double, 1>(ws.Wcb + 12 * C.cb_of_body[bdy]), Ts) : Ts;
}

// collision pass + contact filtering (ConstraintSolver.cpp:576-601) + row bookkeeping.  Pairs are spread over the lanes in chunks
// (one slot of NB2_CW_PAIR_SLOT doubles per pair in the matrix region); one lane then appends the surviving contacts in pair order —
// the reference's enumeration order, which fixes the LCP row order.  meta: [0] m, [1] nc, [2] status, [3] capacity overflow,
// [4] number of distinct contact bodies.  max_contacts / max_rows: the ABSOLUTE limits (beyond them contacts are dropped and
// flagged); d.MC / d.MR: the capacity of THIS workspace (beyond it meta[3] is set and the caller retries with the large one).
// Afterwards the active joint limits (JointLimitConstraint::update, constraint/JointLimitConstraint.cpp:150-240) are appended as pseudo contacts
// with one frictionless row each, in joint order (ConstraintSolver.cpp:642-695 adds them after the contacts): M / st give the positions.
NB2_HD void collide_and_filter(const Nb2ContactDev& C, const Ws& ws, const Dims& d, const Nb2ModelDev<double>* Mp = nullptr, const float* st = nullptr) {
  const int slots = (int)(d.mats / NB2_CW_PAIR_SLOT);
  CW_ONE { ws.meta[0] = 0; ws.meta[1] = 0; ws.meta[2] = 0; ws.meta[3] = 0; ws.meta[4] = 0; }
  CW_SYNC();
  for (int p0 = 0; p0 < C.npairs; p0 += slots) {
    const int cnt = (C.npairs - p0 < slots) ? C.npairs - p0 : slots;
    CW_FOR(q, cnt) {
      const int pi = p0 + q, sa = C.pair_a[pi], sb = C.pair_b[pi];
      ContactOutT<double> co[8];
      int st = 0;
      const int k = pair_contacts<double>(C, sa, sb, shape_pose(C, ws, sa), shape_pose(C, ws, sb), co, &st);
      double* sl = ws.M1 + (size_t)q * NB2_CW_PAIR_SLOT;
      sl[0] = (double)k; sl[1] = (double)st;
      for (int c = 0; c < k; c++) {
        double* o = sl + 2 + 8 * c;
        o[0] = co[c].point.x; o[1] = co[c].point.y; o[2] = co[c].point.z; o[3] = co[c].normal.x; o[4] = co[c].normal.y; o[5] = co[c].normal.z;
        o[6] = co[c].depth; o[7] = (double)co[c].type;
      }
    }
    CW_SYNC();
    CW_ONE {
      int m = ws.meta[0], nc = ws.meta[1], status = ws.meta[2], ovf = ws.meta[3], ntb = ws.meta[4];
      for (int q = 0; q < cnt && !ovf; q++) {
        const double* sl = ws.M1 + (size_t)q * NB2_CW_PAIR_SLOT;
        const int pi = p0 + q, sa = C.pair_a[pi], sb = C.pair_b[pi], ba = C.shape_body[sa], bb = C.shape_body[sb];
        status |= (int)sl[1];
        const int k = (int)sl[0];
        for (int c = 0; c < k; c++) {
          const double* o = sl + 2 + 8 * c;
          if (o[3] * o[3] + o[4] * o[4] + o[5] * o[5] < 1e-12) continue;
          if (o[6] < 0.0 || o[6] > C.clip_depth) continue;
          if (ba < 0 && bb < 0) continue;
          const double mu = C.shape_mu[sa] < C.shape_mu[sb] ? C.shape_mu[sa] : C.shape_mu[sb];
          const int dim = (mu > 1e-3) ? 3 : 1;
          if (nc >= NB2_MAX_CONTACTS || m + dim > NB2_MAX_ROWS) { status |= NB2_ST_CONTACT_OVERFLOW; continue; }
          if (nc >= d.MC || m + dim > d.MR) { ovf = 1; break; }
          for (int e = 0; e < 3; e++) { ws.cpoint[3 * nc + e] = o[e]; ws.cnormal[3 * nc + e] = o[3 + e]; }
          ws.cdepth[nc] = o[6]; ws.ctype[nc] = (int)o[7]; ws.cbodyA[nc] = ba; ws.cbodyB[nc] = bb; ws.cshapeA[nc] = sa; ws.cshapeB[nc] = sb;
          ws.cmu[nc] = mu; ws.crest[nc] = C.shape_rest[sa] * C.shape_rest[sb];
          ws.crow[nc] = m;
          for (int e = 0; e < dim; e++) ws.rowc[m + e] = nc;
          for (int side = 0; side < 2; side++) {
            const int bdy = side ? bb : ba;
            if (bdy < 0) continue;
            bool seen = false;
            for (int e = 0; e < ntb; e++) if (ws.tbl[e] == bdy) seen = true;
            if (!seen) ws.tbl[ntb++] = bdy;
          }
          m += dim; nc++;
        }
      }
      ws.meta[0] = m; ws.meta[1] = nc; ws.meta[2] = status; ws.meta[3] = ovf; ws.meta[4] = ntb;
    }
    CW_SYNC();
    if (ws.meta[3]) return;
  }
  if (C.nlim > 0 && Mp && st) {
    const Nb2ModelDev<double>& M = *Mp;
    CW_ONE {
      int m = ws.meta[0], nc = ws.meta[1], status = ws.meta[2], ovf = ws.meta[3], ntb = ws.meta[4];
      for (int l = 0; l < C.nlim && !ovf; l++) {
        const int i = C.lim_body[l], dd = M.dof_off[i];
        const double q = (double)st[dd];
        int type = 0;
        if (q - (double)M.pos_lo[dd] <= 0.0) type = NB2_CT_LIMIT_LOWER;
        else if (q - (double)M.pos_hi[dd] >= 0.0) type = NB2_CT_LIMIT_UPPER;
        if (!type) continue;
        if (nc >= NB2_MAX_CONTACTS || m + 1 > NB2_MAX_ROWS) { status |= NB2_ST_CONTACT_OVERFLOW; continue; }
        if (nc >= d.MC || m + 1 > d.MR) { ovf = 1; break; }
        for (int e = 0; e < 3; e++) { ws.cpoint[3 * nc + e] = 0.0; ws.cnormal[3 * nc + e] = 0.0; }
        ws.cdepth[nc] = 0.0; ws.ctype[nc] = type; ws.cbodyA[nc] = i; ws.cbodyB[nc] = M.parent[i]; ws.cshapeA[nc] = -1; ws.cshapeB[nc] = -1;
        ws.cmu[nc] = 0.0; ws.crest[nc] = 0.0;
        ws.crow[nc] = m; ws.rowc[m] = nc;
        for (int side = 0; side < 2; side++) {
          const int bdy = side ? M.parent[i] : i;
          if (bdy < 0) continue;
          bool seen = false;
          for (int e = 0; e < ntb; e++) if (ws.tbl[e] == bdy) seen = true;
          if (!seen) ws.tbl[ntb++] = bdy;
        }
        m += 1; nc++;
      }
      ws.meta[0] = m; ws.meta[1] = nc; ws.meta[2] = status; ws.meta[3] = ovf; ws.meta[4] = ntb;
    }
    CW_SYNC();
  }
}

// rows of the LCP: wrenches, b = -J v*, bounds, findex (ContactConstraint.cpp:66-230, 361-514, 687-695, 734-795); one row per lane.
// Returns the status bits raised here (bounce).  want_b = false (backward pass): wrenches only.
// eeff (optional, [m]): per row the restitution coefficient the forward APPLIED — e when b = (1 + e)(-J v*), -1 when the bounce velocity hit its
// cap (a constant was added), 0 otherwise; needs Vcb at v* like want_b.
NB2_HD int build_rows(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const Ws& ws, int m, bool want_b, double* eeff = nullptr) {
  bool bounced = false, pencorr = false;
  CW_FOR(r, m) {
    const int c = ws.rowc[r], k = r - ws.crow[c];
    const double mu = ws.cmu[c], e = ws.crest[c];
    const V3<double> nrm = mk3<double>(ws.cnormal[3 * c], ws.cnormal[3 * c + 1], ws.cnormal[3 * c + 2]);
    const V3<double> pt = mk3<double>(ws.cpoint[3 * c], ws.cpoint[3 * c + 1], ws.cpoint[3 * c + 2]);
    V3<double> dir = nrm;
    if (k > 0) { V3<double> t1, t2; tangent_basis<double>(nrm, &t1, &t2); dir = (k == 1) ? t1 : t2; }
    const int ba = ws.cbodyA[c], bb = ws.cbodyB[c];
    double rel = 0;
    V6<double> JA = zero6<double>(), JB = zero6<double>();
    if (ws.ctype[c] >= NB2_CT_LIMIT_LOWER) {
      // joint-limit row: a unit impulse on the joint (JointLimitConstraint::applyUnitImpulse, :258-283) is S on the child and its reaction
      // on the parent; b = -(JA.V_A + JB.V_B) = -qdot* (getInformation :243-256: the "bouncing velocity" is +-allowance * erp / dt, allowance 0)
      JA = S_times<double>(M.jtype[ba], 1.0);
      const Xf<double> Wc = ldXf<double, 1>(ws.Wcb + 12 * C.cb_of_body[ba]);
      rel -= dot(JA, ldv6(ws.Vcb + 6 * C.cb_of_body[ba]));
      if (bb >= 0) {
        const Xf<double> Wp = ldXf<double, 1>(ws.Wcb + 12 * C.cb_of_body[bb]);
        Xf<double> X; X.R_ = mul(transpose(Wp.R_), Wc.R_); X.p = mulT(Wp.R_, Wc.p - Wp.p);   // parent <- child
        JB = zero6<double>() - dAdInvT(X, JA);
        rel -= dot(JB, ldv6(ws.Vcb + 6 * C.cb_of_body[bb]));
      }
      stv6(ws.JA + 6 * r, JA); stv6(ws.JB + 6 * r, JB);
      if (eeff) eeff[r] = 0;
      if (want_b) {
        if (ws.ctype[c] == NB2_CT_LIMIT_LOWER) { ws.lo[r] = 0.0; ws.hi[r] = HUGE_VAL; } else { ws.lo[r] = -HUGE_VAL; ws.hi[r] = 0.0; }
        ws.findex[r] = -1; ws.b[r] = rel;
      }
      continue;
    }
    if (ba >= 0) {
      const int kb = C.cb_of_body[ba];
      const Xf<double> W = ldXf<double, 1>(ws.Wcb + 12 * kb);
      const V3<double> pA = xf_apply_inv(W, pt), dA = mulT(W.R_, dir);
      JA.a = cross(pA, dA); JA.l = dA;
      rel -= dot(JA, ldv6(ws.Vcb + 6 * kb));
    }
    if (bb >= 0) {
      const int kb = C.cb_of_body[bb];
      const Xf<double> W = ldXf<double, 1>(ws.Wcb + 12 * kb);
      const V3<double> pB = xf_apply_inv(W, pt), dB = mulT(W.R_, -dir);
      JB.a = cross(pB, dB); JB.l = dB;
      rel -= dot(JB, ldv6(ws.Vcb + 6 * kb));
    }
    stv6(ws.JA + 6 * r, JA); stv6(ws.JB + 6 * r, JB);
    if (eeff) {  // the same decisions as below, on the same numbers
      double ee = 0;
      if (k == 0) {
        double bv = ws.cdepth[c];
        if (bv < 0) bv = 0; else { bv *= 0.01 * (1.0 / M.dt); if (bv > 1e-3) bv = 1e-3; }
        if (!C.pen_correction) bv = 0;
        if (e > 1e-3) { const double rv = rel * e; if (rv > 1e-1 && rv > bv) ee = (rv > 1e2) ? -1.0 : e; }
      }
      eeff[r] = ee;
    }
    if (want_b) {
      if (k == 0) {
        ws.lo[r] = 0.0; ws.hi[r] = HUGE_VAL; ws.findex[r] = -1;
        // bounce / penetration-correction velocity (ContactConstraint.cpp:395-442)
        double bv = ws.cdepth[c];
        if (bv < 0) bv = 0; else { bv *= 0.01 * (1.0 / M.dt); if (bv > 1e-3) bv = 1e-3; }
        if (!C.pen_correction) bv = 0;
        else if (bv > 0) pencorr = true;
        if (e > 1e-3) { const double rv = rel * e; if (rv > 1e-1) { if (rv > bv) { bv = rv; if (bv > 1e2) bv = 1e2; bounced = true; } } }
        rel += bv;
      } else { ws.lo[r] = -mu; ws.hi[r] = mu; ws.findex[r] = ws.crow[c]; }
      ws.b[r] = rel;
    }
  }
  bounced = cw_any(bounced); pencorr = cw_any(pencorr);
  CW_SYNC();
  return (bounced ? NB2_ST_BOUNCE : 0) | (pencorr ? NB2_ST_PENCORR : 0);
}

// ---- impulse response along one chain (impulse-ABA with the forward's U, psi; BodyNode.cpp:2117-2138, 2188-2215,
// GenericJoint.hpp:2482-2498, 2607-2613, 2713-2725).  An impulse on body sb only loads the bodies on the chain sb -> root:
// chain_up walks it once with the bias impulse in registers and leaves the joint-space impulses in priv[] (indexed by the dof's
// offset on its chain, C.cdof0); chain_down then gives the spatial velocity change of ANY body t by walking root -> t, where
// only the common ancestors of sb and t carry a joint-space impulse.
NB2_HD void chain_up(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const TreeSrc& S, int sb, V6<double> pI, double* priv) {
  for (int i = sb; i >= 0; i = M.parent[i]) {
    const int jt = M.jtype[i], p = M.parent[i], c0 = C.cdof0[i];
    if (jt != NB2_JT_FREE) {
      const double u = -S_dot(jt, pI);
      priv[c0] = u;
      if (p >= 0) { const V6<double> beta = pI + ts_U(S, i) * (ts_psi(S, i) * u); pI = dAdInvT(ts_xf(M, S, i), beta); }
    } else {
      stv6(priv + c0, zero6<double>() - pI);
      pI = zero6<double>();  // pI + I (I^-1 u) = 0: a 6-dof joint absorbs the whole impulse
    }
  }
}
NB2_HD V6<double> chain_down(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const TreeSrc& S, unsigned long long src_mask, int t,
                             const double* priv) {
  V6<double> dV = zero6<double>();
  unsigned long long mask = C.anc_mask[t];
  while (mask) {
    const int j = lowest_bit(mask); mask &= mask - 1;
    const bool common = (src_mask >> j) & 1ull;
    const int jt = M.jtype[j], c0 = C.cdof0[j];
    const V6<double> Vp = (M.parent[j] >= 0) ? AdInvT(ts_xf(M, S, j), dV) : zero6<double>();
    if (jt != NB2_JT_FREE) {
      const double u = common ? priv[c0] : 0.0;
      const double dq = ts_psi(S, j) * (u - dot(ts_U(S, j), Vp));
      dV = Vp;
      if (jt == NB2_JT_REV) dV.a.z += dq; else dV.l.z += dq;
    } else {
      dV = common ? mul(ts_Iinv(M, S, j), ldv6(priv + c0)) : zero6<double>();
    }
  }
  return dV;
}

// A = J M^-1 J^T by impulse tests (BoxedLcpConstraintSolver.cpp:190-349): one row per lane.  As in the reference the upper blocks
// (contact of the column >= contact of the row) are the measured ones, the lower blocks mirror them.  rows == nullptr: all m rows;
// else only the listed nrows rows are measured (backward pass: clamping and upper-bound rows) and nothing is mirrored.
NB2_HD void assemble_A(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const TreeSrc& S, const Ws& ws, int m, int ld, const int* rows, int nrows) {
  const int cd = C.max_chain_dofs, ntb = ws.meta[4];
  CW_FOR(q, rows ? nrows : m) {
    const int r = rows ? rows[q] : q;
    double* Arow = ws.A + (size_t)r * ld;
    for (int s = 0; s < m; s++) Arow[s] = 0;
    double* priv = ws.M1 + (size_t)q * cd;
    const int c = ws.rowc[r];
    for (int side = 0; side < 2; side++) {
      const int sb = side ? ws.cbodyB[c] : ws.cbodyA[c];
      if (sb < 0) continue;
      chain_up(M, C, S, sb, zero6<double>() - ldv6((side ? ws.JB : ws.JA) + 6 * r), priv);
      const unsigned long long smask = C.anc_mask[sb];
      for (int e = 0; e < ntb; e++) {
        const int t = ws.tbl[e];
        const V6<double> dV = chain_down(M, C, S, smask, t, priv);
        for (int s = 0; s < m; s++) {
          const int cs = ws.rowc[s];
          if (ws.cbodyA[cs] == t) Arow[s] += dot(ldv6(ws.JA + 6 * s), dV);
          if (ws.cbodyB[cs] == t) Arow[s] += dot(ldv6(ws.JB + 6 * s), dV);
        }
      }
    }
  }
  CW_SYNC();
  if (!rows) {
    CW_FOR2(r, s2, m, m) { if (ws.rowc[s2] < ws.rowc[r]) ws.A[(size_t)r * ld + s2] = ws.A[(size_t)s2 * ld + r]; }
    CW_SYNC();
  }
}

// velocity change of every joint for body-frame impulses F_t on the collision bodies (ContactConstraint.cpp:630-684,
// Skeleton.cpp:13571-13595): per collision body one chain_up (parallel), joint-space impulses summed in a fixed order, then one
// root -> leaf sweep over ALL bodies along the model's trunk / limb schedule.  Fcb: [ncb][6] impulses (consumed as -F).
// Results: ws.dqd [n]; spatial velocity changes of all bodies in dVb [nb][6] (= ws.M1).
NB2_HD void impulse_response_all(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const TreeSrc& S, const Ws& ws, const double* Fcb, double* dVb) {
  const int cd = C.max_chain_dofs, n = M.ndof;
  double* privb = ws.M1;
  CW_FOR(k, C.ncb) chain_up(M, C, S, C.cb_body[k], zero6<double>() - ldv6(Fcb + 6 * k), privb + (size_t)k * cd);
  CW_FOR(dd, n) ws.uI[dd] = 0;
  CW_SYNC();
  CW_ONE {
    for (int k = 0; k < C.ncb; k++)
      for (int i = C.cb_body[k]; i >= 0; i = M.parent[i]) {
        const int o = M.dof_off[i], c0 = C.cdof0[i], nd = (M.jtype[i] == NB2_JT_FREE) ? 6 : 1;
        for (int e = 0; e < nd; e++) ws.uI[o + e] += privb[(size_t)k * cd + c0 + e];
      }
  }
  CW_SYNC();
  auto sweep = [&](int lo, int hi) {
    for (int i = lo; i < hi; i++) {
      const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i];
      V6<double> dV = (p >= 0) ? AdInvT(ts_xf(M, S, i), ldv6(dVb + 6 * p)) : zero6<double>();
      if (jt != NB2_JT_FREE) {
        const double dq = ts_psi(S, i) * (ws.uI[o] - dot(ts_U(S, i), dV));
        ws.dqd[o] = dq;
        if (jt == NB2_JT_REV) dV.a.z += dq; else dV.l.z += dq;
      } else {
        const V6<double> dq = mul(ts_Iinv(M, S, i), ldv6(ws.uI + o)) - dV;
        stv6(ws.dqd + o, dq);
        dV = dV + dq;
      }
      stv6(dVb + 6 * i, dV);
    }
  };
  CW_FOR(l, 1) for (int r = 0; r < M.trunk_n; r++) sweep(M.trunk_lo[r], M.trunk_hi[r]);
  CW_SYNC();
  CW_FOR(l, M.lanes) for (int r = 0; r < M.limb_n[l]; r++) sweep(M.limb_lo[l][r], M.limb_hi[l][r]);
  CW_SYNC();
}
// net body-frame impulse on every collision body: F_t = sum_r coef_r * wrench of row r on t
NB2_HD void net_wrenches(const Nb2ContactDev& C, const Ws& ws, int m, const double* coef, double* Fcb) {
  CW_FOR(k, C.ncb) {
    const int t = C.cb_body[k];
    V6<double> F = zero6<double>();
    for (int r = 0; r < m; r++) {
      const int c = ws.rowc[r];
      if (coef[r] == 0.0) continue;
      if (ws.cbodyA[c] == t) F = F + ldv6(ws.JA + 6 * r) * coef[r];
      if (ws.cbodyB[c] == t) F = F + ldv6(ws.JB + 6 * r) * coef[r];
    }
    stv6(Fcb + 6 * k, F);
  }
  CW_SYNC();
}

// record of a step for the backward pass, per world: [0] m, [1] status, then mapping[NB2_MAX_ROWS], x[NB2_MAX_ROWS], dqd[n]
NB2_HD size_t record_doubles(int ndof) { return 2 + 2 * (size_t)NB2_MAX_ROWS + ndof; }

// pool of LARGE workspaces in global memory for the rare world whose contacts exceed the shared-memory capacity: slots are handed
// out with an atomic counter (reset by the host before every launch); a world that finds the pool empty keeps the contacts that fit
// and is flagged NB2_ST_CONTACT_OVERFLOW.
struct BigPool { int* counter; double* base; size_t stride; int nslots; };
NB2_HD double* pool_acquire(const BigPool& P) {
  if (!P.base || P.nslots <= 0) return nullptr;
#if CW_DEV
  int slot = 0;
  if (CW_LANE == 0) slot = atomicAdd(P.counter, 1);
  slot = __shfl_sync(CW_FULL, slot, 0);
#else
  const int slot = (*P.counter)++;
#endif
  return (slot < P.nslots) ? P.base + (size_t)slot * P.stride : nullptr;
}

struct FwdIO {
  double* x_io;     // [NB2_MAX_ROWS] cached LCP solution in / this step's solution out
  int* m_io;        // its size (-1: none) in / LCP dimension out
  int* labels;      // [NB2_MAX_ROWS]
  int* status;      // out
  int* nc;          // out
  float* cinfo;     // [NB2_MAX_CONTACTS][10] optional
  double* rec;      // optional record for the backward pass
};

// =====================================================================================================
// the contact stage of one world.  `scr` is the world's ABA scratch after the three sweeps: q+ in oQ, v* = v + dt qdd in oV (fp64);
// on exit oV holds v+.  ws_s / d_s: the shared-memory workspace; big: a global-memory block of ws_doubles(d_b) doubles for the rare
// world whose contact count exceeds the shared capacity (may be nullptr: such worlds then drop contacts and are flagged).
// =====================================================================================================
// wsm: storage of the workspace descriptor, ALREADY carved for the small workspace by the caller (shared memory on the device: the
// non-inlined routines read the array pointers from there instead of dragging ~60 pointers through registers / local memory).
NB2_HD void contact_forward(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, double* scr, const float* st, Ws* wsm, const Dims& d_s,
                            const BigPool& pool, const Dims& d_b, const double* Iinv_fwd, const FwdIO& io) {
  const FwdLayout L = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof;
  Ws ws = *wsm;  // register copy for the inlined code
  Dims d = d_s;
  TreeSrc S; S.scr = scr; S.L = L; S.Iinv = ws.Iinv; S.sv = nullptr; S.st = st; S.nb = M.nb; S.nfree = M.nfree;
  (void)Iinv_fwd;
  CW_PROF_DECL;
  fk_collision_bodies(M, C, S, scr + L.oV, ws);
  CW_PROF(1);
  collide_and_filter(C, ws, d, &M, st);
  CW_PROF(2);
  double* ws_big = ws.meta[3] ? pool_acquire(pool) : nullptr;
  if (ws_big) {  // more contacts than the shared workspace holds: redo the stage in a large global workspace
    const Ws wb = carve(ws_big, d_b);
    CW_FOR(e, C.ncb * 12) wb.Wcb[e] = ws.Wcb[e];
    CW_FOR(e, C.ncb * 6) wb.Vcb[e] = ws.Vcb[e];
    CW_FOR(e, M.nfree * 21) wb.Iinv[e] = ws.Iinv[e];
    CW_SYNC();
    CW_ONE *wsm = wb;
    CW_SYNC();
    ws = wb; d = d_b;
    collide_and_filter(C, ws, d, &M, st);
  }
  const int m = ws.meta[0], nc = ws.meta[1];
  int status = ws.meta[2];
  if (ws.meta[3]) status |= NB2_ST_CONTACT_OVERFLOW;
  CW_ONE {
    *io.nc = nc;
    if (io.cinfo) for (int c = 0; c < nc; c++) {
      float* o = io.cinfo + 10 * c;
      for (int e = 0; e < 3; e++) { o[e] = (float)ws.cpoint[3 * c + e]; o[3 + e] = (float)ws.cnormal[3 * c + e]; }
      o[6] = (float)ws.cdepth[c]; o[7] = (float)(ws.cshapeA[c] >= 0 ? C.shape_orig_body[ws.cshapeA[c]] : -1); o[8] = (float)(ws.cshapeB[c] >= 0 ? C.shape_orig_body[ws.cshapeB[c]] : -1);  // (joint-limit rows have no shapes)
      o[9] = (float)ws.ctype[c];
    }
  }
  if (m == 0) {
    CW_ONE { *io.m_io = 0; *io.status = status; if (io.rec) { io.rec[0] = 0; io.rec[1] = (double)status; } }
    CW_SYNC();
    return;  // scr already holds v*
  }
  status |= build_rows(M, C, ws, m, true);
  CW_PROF(3);
  const int ld = m | 1;
  assemble_A(M, C, S, ws, m, ld, nullptr, 0);
  CW_PROF(4);
  status |= lcp_chain(m, ws, *wsm, C.fallback_cfm, (*io.m_io == m) ? io.x_io : nullptr);
  CW_SYNC();
  CW_PROF(5);
  // ---- apply the impulses and update the velocities
  net_wrenches(C, ws, m, ws.x, ws.Fcb);
  impulse_response_all(M, C, S, ws, ws.Fcb, ws.M1 + (size_t)C.ncb * C.max_chain_dofs);
  CW_FOR(dd, n) scr[L.oV + dd] += ws.dqd[dd];
  CW_FOR(i, m) { io.x_io[i] = ws.x[i]; io.labels[i] = ws.mapping[i]; }
  if (io.rec) {
    CW_FOR(i, m) { io.rec[2 + i] = (double)ws.mapping[i]; io.rec[2 + NB2_MAX_ROWS + i] = ws.x[i]; }
    CW_FOR(dd, n) io.rec[2 + 2 * NB2_MAX_ROWS + dd] = ws.dqd[dd];
  }
  CW_ONE { *io.m_io = m; *io.status = status; if (io.rec) { io.rec[0] = (double)m; io.rec[1] = (double)status; } }
  CW_SYNC();
  CW_PROF(6);
}

// =====================================================================================================
// The forward contact stage as THREE kernels (build | solve | apply) that hand a world over through an exchange record in global
// memory.  Why: the solver chain is ~3/4 of the stage, needs few registers and only the LCP in shared memory, while the tree
// sweeps and the collision code need 255 registers — in one kernel every phase runs at the occupancy of the hungriest.
// Exchange record of a world (doubles; capacities NB2_MAX_ROWS / NB2_MAX_CONTACTS, only the used part is touched):
//   [0] m  [1] nc  [2] status so far  [3] -   then b, lo, hi, findex, rowc (MRX each), cbodyA, cbodyB (MCX each), JA, JB (6 MRX each),
//   x0 (MRX: the warm start, written by the first solve kernel for the worlds it hands on), v* (n), A (m x (m | 1), packed with the
//   problem's own leading dimension)
// =====================================================================================================
struct XLayout { int oB, oLo, oHi, oFi, oRowc, oCA, oCB, oJA, oJB, oX0, oV, oA; size_t total; };
NB2_HD XLayout xlayout(int n) {
  const int MRX = NB2_MAX_ROWS, MCX = NB2_MAX_CONTACTS;
  XLayout x; x.oB = 4; x.oLo = x.oB + MRX; x.oHi = x.oLo + MRX; x.oFi = x.oHi + MRX; x.oRowc = x.oFi + MRX; x.oCA = x.oRowc + MRX; x.oCB = x.oCA + MCX;
  x.oJA = x.oCB + MCX; x.oJB = x.oJA + 6 * MRX; x.oX0 = x.oJB + 6 * MRX; x.oV = x.oX0 + MRX; x.oA = x.oV + n;
  x.total = ((size_t)x.oA + (size_t)MRX * (MRX | 1) + 1) & ~(size_t)1;
  return x;
}

// ---- build: collision, rows, A; leaves the record.  `scr`: the world's ABA scratch (q+ in oQ, v* in oV).  X == nullptr: a warp
// without a world (tail of the last block) — it only takes part in the phase barriers.
#define NB2_BUILD_PHASES 4
NB2_HD void contact_build(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, double* scr, const float* st, Ws* wsm, const Dims& d_s,
                          const BigPool& pool, const Dims& d_b, const FwdIO& io, double* X) {
  int ph = 0;
  if (!X) { while (ph < NB2_BUILD_PHASES) { CW_PHASE(); ph++; } return; }
  const FwdLayout L = fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const XLayout xl = xlayout(M.ndof);
  Ws ws = *wsm;
  Dims d = d_s;
  TreeSrc S; S.scr = scr; S.L = L; S.Iinv = ws.Iinv; S.sv = nullptr; S.st = st; S.nb = M.nb; S.nfree = M.nfree;
  CW_PROF_DECL;
  fk_collision_bodies(M, C, S, scr + L.oV, ws);
  CW_PROF(1);
  CW_PHASE(); ph++;  // 1
  collide_and_filter(C, ws, d, &M, st);
  double* ws_big = ws.meta[3] ? pool_acquire(pool) : nullptr;
  if (ws_big) {
    const Ws wb = carve(ws_big, d_b);
    CW_FOR(e, C.ncb * 12) wb.Wcb[e] = ws.Wcb[e];
    CW_FOR(e, C.ncb * 6) wb.Vcb[e] = ws.Vcb[e];
    CW_FOR(e, M.nfree * 21) wb.Iinv[e] = ws.Iinv[e];
    CW_SYNC();
    CW_ONE *wsm = wb;
    CW_SYNC();
    ws = wb; d = d_b;
    collide_and_filter(C, ws, d, &M, st);
  }
  CW_PROF(2);
  const int m = ws.meta[0], nc = ws.meta[1];
  int status = ws.meta[2];
  if (ws.meta[3]) status |= NB2_ST_CONTACT_OVERFLOW;
  CW_ONE {
    *io.nc = nc;
    if (io.cinfo) for (int c = 0; c < nc; c++) {
      float* o = io.cinfo + 10 * c;
      for (int e = 0; e < 3; e++) { o[e] = (float)ws.cpoint[3 * c + e]; o[3 + e] = (float)ws.cnormal[3 * c + e]; }
      o[6] = (float)ws.cdepth[c]; o[7] = (float)(ws.cshapeA[c] >= 0 ? C.shape_orig_body[ws.cshapeA[c]] : -1); o[8] = (float)(ws.cshapeB[c] >= 0 ? C.shape_orig_body[ws.cshapeB[c]] : -1);  // (joint-limit rows have no shapes)
      o[9] = (float)ws.ctype[c];
    }
  }
  if (m == 0) {
    CW_ONE { X[0] = 0; X[1] = (double)nc; X[2] = (double)status; *io.m_io = 0; *io.status = status; if (io.rec) { io.rec[0] = 0; io.rec[1] = (double)status; } }
    CW_SYNC();
    while (ph < NB2_BUILD_PHASES) { CW_PHASE(); ph++; }
    return;
  }
  CW_PHASE(); ph++;  // 2
  status |= build_rows(M, C, ws, m, true);
  CW_PROF(3);
  CW_PHASE(); ph++;  // 3
  const int ld = m | 1;
  assemble_A(M, C, S, ws, m, ld, nullptr, 0);
  CW_PROF(4);
  CW_PHASE(); ph++;  // 4
  CW_FOR(i, m) {
    X[xl.oB + i] = ws.b[i]; X[xl.oLo + i] = ws.lo[i]; X[xl.oHi + i] = ws.hi[i]; X[xl.oFi + i] = (double)ws.findex[i]; X[xl.oRowc + i] = (double)ws.rowc[i];
  }
  CW_FOR(c, nc) { X[xl.oCA + c] = (double)ws.cbodyA[c]; X[xl.oCB + c] = (double)ws.cbodyB[c]; }
  CW_FOR(e, m * 6) { X[xl.oJA + e] = ws.JA[e]; X[xl.oJB + e] = ws.JB[e]; }
  CW_FOR(dd, M.ndof) X[xl.oV + dd] = scr[L.oV + dd];
  if (ld > m) { CW_FOR(i, m) ws.A[(size_t)i * ld + m] = 0.0; CW_SYNC(); }  // the padding column travels with the matrix: keep it defined
  CW_FOR(e, m * ld) X[xl.oA + e] = ws.A[e];
  CW_ONE { X[0] = (double)m; X[1] = (double)nc; X[2] = (double)status; }
  CW_SYNC();
  CW_PROF(6);
}

// ---- solve, in two kernels so that the worlds of a block do the same amount of work (they run in lockstep):
//   A  warm start + short-circuit classification for every world; the worlds it does not settle are appended to `todo`
//   B  Dantzig / PGS / friction drop / classification for the worlds of `todo`
// wsm: descriptor carved in NB2_WS_SOLVE mode (small; large from the pool when m > d_s.MR).  X == nullptr: warp without a world.
NB2_HD bool solve_workspace(Ws* wsm, Ws& ws, int m, const Dims& d_s, const BigPool& pool, const Dims& d_b) {
  if (m <= d_s.MR) return true;
  double* big = pool_acquire(pool);
  if (!big) return false;
  const Ws wb = carve(big, d_b);
  CW_SYNC();
  CW_ONE *wsm = wb;
  CW_SYNC();
  ws = wb;
  return true;
}
NB2_HD void solve_load(const Ws& ws, int m, const double* X, const XLayout& xl) {
  const int ld = m | 1;
  CW_FOR(i, m) { ws.b[i] = X[xl.oB + i]; ws.lo[i] = X[xl.oLo + i]; ws.hi[i] = X[xl.oHi + i]; ws.findex[i] = (int)X[xl.oFi + i]; }
  CW_FOR(e, m * ld) ws.A[e] = X[xl.oA + e];
  CW_SYNC();
}
NB2_HD void contact_solve_a(const Nb2ContactDev& C, int ndof, Ws* wsm, const Dims& d_s, const BigPool& pool, const Dims& d_b, const FwdIO& io, double* X,
                            int* status_accum, int world, int* todo, int* todo_count) {
  const int m = X ? (int)X[0] : 0;
  if (m <= 0) {
    CW_ONE { if (X && status_accum) *status_accum |= (int)X[2]; }
    for (int k = 0; k < NB2_HEAD_PHASES; k++) CW_PHASE();
    return;
  }
  const XLayout xl = xlayout(ndof);
  Ws ws = *wsm;
  if (!solve_workspace(wsm, ws, m, d_s, pool, d_b)) {  // pool exhausted: this world cannot be solved here — flag it and leave v*
    CW_ONE {
      const int st = (int)X[2] | NB2_ST_CONTACT_OVERFLOW;
      *io.m_io = 0; *io.status = st; if (status_accum) *status_accum |= st; X[0] = 0; if (io.rec) { io.rec[0] = 0; io.rec[1] = (double)st; }
    }
    CW_SYNC();
    for (int k = 0; k < NB2_HEAD_PHASES; k++) CW_PHASE();
    return;
  }
  solve_load(ws, m, X, xl);
  const bool done = lcp_chain_head(m, ws, *wsm, (*io.m_io == m) ? io.x_io : nullptr);
  CW_SYNC();
  if (done) {
    const int status = (int)X[2] | NB2_ST_SHORTCIRCUIT;
    CW_FOR(i, m) { io.x_io[i] = ws.x[i]; io.labels[i] = ws.mapping[i]; }
    CW_ONE { *io.m_io = m; *io.status = status; if (status_accum) *status_accum |= status; X[2] = (double)status; }
  } else {
    CW_FOR(i, m) X[xl.oX0 + i] = ws.x0[i];
    CW_ONE {
#if CW_DEV
      const int slot = atomicAdd(todo_count, 1);
#else
      const int slot = (*todo_count)++;
#endif
      todo[slot] = world;
    }
  }
  CW_SYNC();
}
NB2_HD void contact_solve_b(const Nb2ContactDev& C, int ndof, Ws* wsm, const Dims& d_s, const BigPool& pool, const Dims& d_b, const FwdIO& io, double* X,
                            int* status_accum) {
  const int m = X ? (int)X[0] : 0;
  if (m <= 0) { for (int k = 0; k < NB2_TAIL_PHASES; k++) CW_PHASE(); return; }
  const XLayout xl = xlayout(ndof);
  Ws ws = *wsm;
  if (!solve_workspace(wsm, ws, m, d_s, pool, d_b)) {  // (cannot happen when kernel A got its slot: same pool, same demand)
    for (int k = 0; k < NB2_TAIL_PHASES; k++) CW_PHASE();
    return;
  }
  solve_load(ws, m, X, xl);
  CW_FOR(i, m) { ws.x0[i] = X[xl.oX0 + i]; ws.x[i] = X[xl.oX0 + i]; }
  CW_SYNC();
  lcp_colnorms(m, ws);
  const int status = (int)X[2] | lcp_chain_tail(m, ws, *wsm, C.fallback_cfm);
  CW_SYNC();
  CW_FOR(i, m) { io.x_io[i] = ws.x[i]; io.labels[i] = ws.mapping[i]; }
  CW_ONE { *io.m_io = m; *io.status = status; if (status_accum) *status_accum |= status; X[2] = (double)status; }
  CW_SYNC();
}

// ---- apply: impulses -> joint velocity changes -> v+ (fp32 row `vnext`), and the record of the step for the backward pass.
// wsm: descriptor carved in NB2_WS_APPLY mode.  sv: the world's saved stream (world-major).
NB2_HD void contact_apply(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const float* st, const double* sv, Ws* wsm, const Dims& d_s,
                          const BigPool& pool, const Dims& d_b, const FwdIO& io, const double* X, float* vnext) {
  const int m = X ? (int)X[0] : 0, nc = X ? (int)X[1] : 0;
  if (m <= 0) { CW_PHASE(); CW_PHASE(); return; }
  const XLayout xl = xlayout(M.ndof);
  const int n = M.ndof;
  Ws ws = *wsm;
  if (m > d_s.MR || nc > d_s.MC) {
    double* big = pool_acquire(pool);
    if (!big) { CW_PHASE(); CW_PHASE(); return; }  // (contact_solve already flagged the world when the pool ran dry: same pool size, same demand)
    const Ws wb = carve(big, d_b);
    CW_SYNC();
    CW_ONE *wsm = wb;
    CW_SYNC();
    ws = wb;
  }
  CW_FOR(i, m) { ws.rowc[i] = (int)X[xl.oRowc + i]; ws.x[i] = io.x_io[i]; }
  CW_FOR(c, nc) { ws.cbodyA[c] = (int)X[xl.oCA + c]; ws.cbodyB[c] = (int)X[xl.oCB + c]; }
  CW_FOR(e, m * 6) { ws.JA[e] = X[xl.oJA + e]; ws.JB[e] = X[xl.oJB + e]; }
  CW_SYNC();
  CW_PHASE();
  TreeSrc S; S.scr = nullptr; S.Iinv = nullptr; S.sv = sv; S.st = st; S.nb = M.nb; S.nfree = M.nfree;
  S.L = fwd_layout(M.nb, n, M.nslots, M.nfree);
  net_wrenches(C, ws, m, ws.x, ws.Fcb);
  impulse_response_all(M, C, S, ws, ws.Fcb, ws.M1 + (size_t)C.ncb * C.max_chain_dofs);
  CW_PHASE();
  CW_FOR(dd, n) vnext[dd] = (float)(X[xl.oV + dd] + ws.dqd[dd]);
  if (io.rec) {
    CW_FOR(i, m) { io.rec[2 + i] = (double)io.labels[i]; io.rec[2 + NB2_MAX_ROWS + i] = ws.x[i]; }
    CW_FOR(dd, n) io.rec[2 + 2 * NB2_MAX_ROWS + dd] = ws.dqd[dd];
    CW_ONE { io.rec[0] = (double)m; io.rec[1] = X[2]; }
  }
  CW_SYNC();
}

// =====================================================================================================
// backward through the contact stage (classification frozen at the forward solution), adjoint form.
// With  P = A_c + A_ub E,  f = Q^+ b_c,  v+ = v* + M^-1 P f  (BackpropSnapshot.cpp:980-1107 materialises the Jacobians of
// this map); for an incoming g = dL/dv+ :
//     lambda = M^-1 g ;  fbar = P^T lambda ;  mu = Q^-T fbar ;  nu = M^-1 A_c mu ;  w = lambda - nu
//     dL/dv* = g - A_c mu  (so the ABA part is back-propagated with w in place of lambda and the REALISED acceleration
//     (v+ - v)/dt in place of the unconstrained one) ;  dL/dtau = dt w
//     contact-Jacobian part:  d/dq of  Phi(q) = sum_r  f_r J_r(q) w  -  mu_r J_r(q) v+   at fixed w, v+  (upper-bound rows: f_r := x_r, mu_r := 0),
//     split into (i) the motion of the contact frame with the pose of the moving body — the contact generator re-run on
//     dual numbers, one pose direction per lane, any contact type — and (ii) the kinematic chain (reverse velocity recursion).
// Runs between the lambda sweeps (B1/B2) and the reverse RNEA sweep (B3) of the backward kernel, all 32 lanes:
//     scr: lambda -> w, W_i -> W_i(w);   returned views: per-body injections, realised accelerations, v+ fields.
// Q is re-measured by impulse tests on the clamping / upper-bound rows (cheap here) instead of being stored by the forward.
// =====================================================================================================
typedef DualT<1> D1;
// world transform W of a body perturbed by the body twist direction kx:  W (I + [xi_w]x , xi_v), derivative part only for kx
// (member by member: no address of a field is taken, so the transform can live in registers)
NB2_HD Xf<D1> lift1(const Xf<double>& X) {
  Xf<D1> o;
  o.R_.m00 = D1(X.R_.m00); o.R_.m01 = D1(X.R_.m01); o.R_.m02 = D1(X.R_.m02);
  o.R_.m10 = D1(X.R_.m10); o.R_.m11 = D1(X.R_.m11); o.R_.m12 = D1(X.R_.m12);
  o.R_.m20 = D1(X.R_.m20); o.R_.m21 = D1(X.R_.m21); o.R_.m22 = D1(X.R_.m22);
  o.p.x = D1(X.p.x); o.p.y = D1(X.p.y); o.p.z = D1(X.p.z);
  return o;
}
NB2_HD Xf<D1> dual_pose1(const Xf<double>& Wd, int kx) {
  Xf<D1> WD = lift1(Wd);
  const V3<double> c0 = mk3<double>(Wd.R_.m00, Wd.R_.m10, Wd.R_.m20), c1 = mk3<double>(Wd.R_.m01, Wd.R_.m11, Wd.R_.m21), c2 = mk3<double>(Wd.R_.m02, Wd.R_.m12, Wd.R_.m22);
  // d(R [e_k]x)/d.: column j of R [e_k]x is R (e_k x e_j)
  if (kx == 0) { WD.R_.m01.d[0] = c2.x; WD.R_.m11.d[0] = c2.y; WD.R_.m21.d[0] = c2.z; WD.R_.m02.d[0] = -c1.x; WD.R_.m12.d[0] = -c1.y; WD.R_.m22.d[0] = -c1.z; }
  else if (kx == 1) { WD.R_.m00.d[0] = -c2.x; WD.R_.m10.d[0] = -c2.y; WD.R_.m20.d[0] = -c2.z; WD.R_.m02.d[0] = c0.x; WD.R_.m12.d[0] = c0.y; WD.R_.m22.d[0] = c0.z; }
  else if (kx == 2) { WD.R_.m00.d[0] = c1.x; WD.R_.m10.d[0] = c1.y; WD.R_.m20.d[0] = c1.z; WD.R_.m01.d[0] = -c0.x; WD.R_.m11.d[0] = -c0.y; WD.R_.m21.d[0] = -c0.z; }
  else { const V3<double> c = (kx == 3) ? c0 : (kx == 4 ? c1 : c2); WD.p.x.d[0] = c.x; WD.p.y.d[0] = c.y; WD.p.z.d[0] = c.z; }
  return WD;
}

// The dual-number instance of the contact generator.  Measured: as an out-of-line call (NB2_DUAL_NOINLINE) the kernel's spill count drops
// 3.7 -> 3.2 KB but the step gets 2 % slower (arguments travel through local memory); inlined is the default.
#if CW_DEV && defined(NB2_DUAL_NOINLINE)
__device__ __noinline__
#elif CW_DEV
__device__ __forceinline__
#else
inline
#endif
int pair_contacts_dual(const Nb2ContactDev& C, int sa, int sb, const Xf<D1>& Ta, const Xf<D1>& Tb, ContactOutT<D1>* co, int* status) {
  return pair_contacts<D1>(C, sa, sb, Ta, Tb, co, status);
}

// BOUNCE = false compiles the restitution branch out (models whose bodies all have restitution 0 — the usual case — keep the leaner kernel)
template <bool BOUNCE>
NB2_HD BwdContactData<1> contact_backward(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const float* st, const double* sv, Ws* wsm,
                                          const Dims& d_s, const BigPool& pool, const Dims& d_b, const double* rec, double* scr, int oLam, int oBody) {
  const int nb = M.nb, n = M.ndof;
  BwdContactData<1> cd;
  cd.Aacc.p = cd.Uplus.p = cd.aeff.p = cd.vplus.p = cd.inj.p = cd.JcTmu.p = nullptr;
  cd.inj_of_body = C.cb_of_body; cd.active = 0; cd.error = 0;
  int ph = 0;
#define NB2_BWD_PHASES 7
#define NB2_BWD_DRAIN() do { while (ph < NB2_BWD_PHASES) { CW_PHASE(); ph++; } } while (0)
  const int m = rec ? (int)rec[0] : 0;
  if (m <= 0) { NB2_BWD_DRAIN(); return cd; }
  cd.active = 1;
  const int fstatus = (int)rec[1];
  // restitution: b_r = (1 + e_r)(-J_r v*) on the rows that bounced.  With B = diag(1 + e):  dL/dv* = g - A_c B mu (the tree part is driven by
  // w_B = w - nu_e, nu_e = M^-1 A_c E mu) while the impulse part keeps w = lambda - M^-1 A_c mu, and the contact-Jacobian part gains a v* field:
  //     Phi = sum_r f_r J_r w - mu_r J_r (v+ + e_r v*).
  // Since the reverse sweep is bilinear in (multiplier field, acceleration field) this is the usual sweep with (w, realised acceleration) PLUS a
  // second sweep with (-nu_e, UNCONSTRAINED acceleration) that also carries the injections of the v* term (bounce_pass2_*, run by the kernel
  // after the first B3).  The reference reaches the same Jacobians through getBounceDiagonals (BackpropSnapshot.cpp:2624-2680, 3088-3146).
  const bool bounce = BOUNCE && (fstatus & NB2_ST_BOUNCE) != 0;
  if (!BOUNCE && (fstatus & NB2_ST_BOUNCE)) { cd.error = 5; cd.active = 0; NB2_BWD_DRAIN(); return cd; }  // (cannot happen: the launcher picks BOUNCE from the model)
  Ws ws = *wsm;
  Dims d = d_s;
  TreeSrc S; S.scr = nullptr; S.Iinv = nullptr; S.sv = sv; S.st = st; S.nb = nb; S.nfree = M.nfree;
  S.L = fwd_layout(nb, n, M.nslots, M.nfree);
  const double dt = M.dt;
  const int kQdd = nb * 21 + M.nfree * 33;
  const double* mapping_r = rec + 2; const double* xr = rec + 2 + NB2_MAX_ROWS; const double* dqd_imp = rec + 2 + 2 * NB2_MAX_ROWS;
  // ---- contacts and row wrenches re-generated from the saved transforms (same code as the forward => same rows)
  CW_PROF_DECL;
  if (bounce) {  // body velocities at v* = v + dt qdd (unconstrained): the rows re-decide which of them bounced
    CW_FOR(dd, n) ws.vplus[dd] = (double)st[n + dd] + dt * sv[kQdd + dd];
    CW_SYNC();
  }
  fk_collision_bodies(M, C, S, bounce ? ws.vplus : nullptr, ws);
  CW_PROF(21);
  CW_PHASE(); ph++;  // 1
  collide_and_filter(C, ws, d, &M, st);
  CW_PROF(22);
  double* ws_big = ws.meta[3] ? pool_acquire(pool) : nullptr;
  if (ws_big) {
    const Ws wb = carve(ws_big, d_b);
    CW_FOR(e, C.ncb * 12) wb.Wcb[e] = ws.Wcb[e];
    if (bounce) { CW_FOR(e, C.ncb * 6) wb.Vcb[e] = ws.Vcb[e]; CW_FOR(dd, n) wb.vplus[dd] = ws.vplus[dd]; }
    CW_SYNC();
    CW_ONE *wsm = wb;
    CW_SYNC();
    ws = wb; d = d_b;
    collide_and_filter(C, ws, d, &M, st);
  }
  if (ws.meta[3] || ws.meta[0] != m) { cd.error = 3; cd.active = 0; NB2_BWD_DRAIN(); return cd; }
  CW_PHASE(); ph++;  // 2
  const int nc = ws.meta[1];
  double* eeff = ws.v11;
  build_rows(M, C, ws, m, false, bounce ? eeff : nullptr);
  cd.aeff.p = ws.aeff; cd.vplus.p = ws.vplus; cd.JcTmu.p = ws.JcTmu; cd.inj.p = ws.inj;
  double* dVb = ws.M1 + (size_t)C.ncb * C.max_chain_dofs;
  double* Aacc = dVb + (size_t)nb * 6; double* Uplus = Aacc + (size_t)nb * 6;
  // bounce only: field of v*, field of nu_e, w before the swap, nu_e, v*; and the scratch of the dual pass (kept clear of them)
  double* Ustar = Uplus + (size_t)nb * 6; double* dVbE = Ustar + (size_t)nb * 6;
  double* wold = dVbE + (size_t)nb * 6; double* nue = wold + n; double* vstar = nue + n; double* gpart = vstar + n;
  cd.Aacc.p = Aacc; cd.Uplus.p = Uplus;
  // ---- clamping / upper-bound sets from the saved labels
  int* mapping = ws.mapping; int* clampIdx = ws.clampIdx; int* cl = ws.i1; int* ubl = ws.i2; int* rows = ws.i3;
  CW_FOR(j, m) { mapping[j] = (int)mapping_r[j]; clampIdx[j] = -1; ws.x[j] = xr[j]; }
  CW_SYNC();
  const int nCl = cw_enumerate(m, [&](int j) { return mapping[j] == NB2_MAP_CLAMPING; }, [&](int j, int r) { cl[r] = j; clampIdx[j] = r; rows[r] = j; });
  const int nUb = cw_enumerate(m, [&](int j) { return mapping[j] >= 0; }, [&](int j, int r) { ubl[r] = j; });
  CW_SYNC();
  CW_FOR(u, nUb) rows[nCl + u] = ubl[u];
  double* rdot = ws.v1; double* fbar = ws.v2; double* mu_c = ws.v3; double* Eu = ws.v4; double* coefM = ws.v5; double* coefW = ws.v7; double* coefV = ws.v8;
  double* coefH = ws.v9; double* coefE = ws.v6;  // (pinv_psd's temporaries until phase 5)
  auto Wfield = [&](int body) { return ld6<double, 1>(scr + oBody + 7 * body + 1); };
  CW_FOR(j, m) {  // J_j lambda-field: wrench of row j against the field induced on its (one or two) bodies
    const int c = ws.rowc[j];
    double a = 0;
    if (ws.cbodyA[c] >= 0) a += dot(ldv6(ws.JA + 6 * j), Wfield(ws.cbodyA[c]));
    if (ws.cbodyB[c] >= 0) a += dot(ldv6(ws.JB + 6 * j), Wfield(ws.cbodyB[c]));
    rdot[j] = a;
  }
  CW_FOR(u, nUb) {
    const int j = ubl[u], fp = mapping[j];
    const double rmu = ws.cmu[ws.rowc[j]];
    const double up = xr[fp] * rmu, low = -xr[fp] * rmu;
    Eu[u] = (fabs(xr[j] - up) < fabs(xr[j] - low)) ? rmu : -rmu;
  }
  CW_SYNC();
  CW_FOR(r, nCl) {
    double f = rdot[cl[r]];
    for (int u = 0; u < nUb; u++) if (clampIdx[mapping[ubl[u]]] == r) f += Eu[u] * rdot[ubl[u]];
    fbar[r] = f; mu_c[r] = 0;
  }
  CW_SYNC();
  CW_PROF(23);
  CW_PHASE(); ph++;  // 3
  if (nCl > 0) {
    const int ld = m | 1;
    assemble_A(M, C, S, ws, m, ld, rows, nCl + nUb);  // rows cl and ub of A, measured
  }
  CW_PROF(24);
  CW_PHASE(); ph++;  // 4
  if (nCl > 0) {
    const int ld = m | 1, lq = nCl | 1;
    // Q = A[cl,cl] + A[cl,ub] E (+ cfm on the diagonal when the forward's fallback added it); as in the forward, an entry below the
    // block diagonal is the mirror image of its measured partner
    double* Q = ws.M1;
    auto Aget = [&](int r, int c) { return (ws.rowc[c] < ws.rowc[r]) ? ws.A[(size_t)c * ld + r] : ws.A[(size_t)r * ld + c]; };
    const double cfm = (fstatus & NB2_ST_PGS) ? C.fallback_cfm : 0.0;
    CW_FOR2(r, c, nCl, nCl) {
      double q = Aget(cl[r], cl[c]);
      if (r == c) q += cfm;
      for (int u = 0; u < nUb; u++) if (clampIdx[mapping[ubl[u]]] == c) q += Aget(cl[r], ubl[u]) * Eu[u];
      ws.M2[(size_t)r * lq + c] = q;
    }
    CW_SYNC();  // (built in M2: M1 still holds the private buffers of assemble_A for lanes that are not done reading A ... they are: synced)
    if (nUb == 0) pinv_psd(nCl, ws.M2, lq, fbar, mu_c, ws.M1, ws.v5, ws.v6, ws.v9, ws.i4);
    else {  // Q^T mu = fbar  ->  mu = (Q Q^T)^+ Q fbar
      double* Qm = ws.M2; double* QQt = ws.M1; double* Qf = ws.v10;
      CW_FOR2(a, c, nCl, nCl) {
        double t = 0; for (int kx = 0; kx < nCl; kx++) t += Qm[(size_t)a * lq + kx] * Qm[(size_t)c * lq + kx];
        QQt[(size_t)a * lq + c] = t;
      }
      CW_FOR(a, nCl) { double sacc = 0; for (int c = 0; c < nCl; c++) sacc += Qm[(size_t)a * lq + c] * fbar[c]; Qf[a] = sacc; }
      CW_SYNC();
      pinv_psd(nCl, QQt, lq, Qf, mu_c, Qm /* Lf */, ws.v5, ws.v6, ws.v9, ws.i4);
    }
  }
  CW_PROF(25);
  CW_PHASE(); ph++;  // 5
  // ---- nu = M^-1 A_c mu  (one impulse response) ; w = lambda - nu ; W_i(w)
  CW_FOR(j, m) {
    const double mu = (clampIdx[j] >= 0) ? mu_c[clampIdx[j]] : 0.0, ee = (bounce && eeff[j] > 0.0) ? eeff[j] : 0.0;
    coefM[j] = mu; coefH[j] = (1.0 + ee) * mu; coefE[j] = -ee * mu;
  }
  CW_SYNC();
  if (bounce) {  // nu_e = M^-1 A_c E mu and its field, kept for the second sweep
    CW_FOR(dd, n) vstar[dd] = ws.vplus[dd];
    CW_FOR(j, m) rdot[j] = -coefE[j];
    CW_SYNC();
    net_wrenches(C, ws, m, rdot, ws.Fcb);
    impulse_response_all(M, C, S, ws, ws.Fcb, dVb);
    CW_FOR(dd, n) nue[dd] = ws.dqd[dd];
    CW_FOR(e, nb * 6) dVbE[e] = dVb[e];
    CW_SYNC();
  }
  net_wrenches(C, ws, m, coefM, ws.Fcb);
  impulse_response_all(M, C, S, ws, ws.Fcb, dVb);
  CW_FOR(dd, n) scr[oLam + dd] -= ws.dqd[dd];
  CW_FOR(e, nb * 6) { const int i = e / 6, k = e - 6 * i; scr[oBody + 7 * i + 1 + k] -= dVb[e]; }
  // ---- realised accelerations, v+, and the fields they induce
  CW_FOR(dd, n) { const double ae = sv[kQdd + dd] + dqd_imp[dd] / dt; ws.aeff[dd] = ae; ws.vplus[dd] = (double)st[n + dd] + dt * ae; }
  CW_SYNC();
  {
    V6<double> A0; A0.a = zero3<double>(); A0.l = mk3<double>(-M.gravity[0], -M.gravity[1], -M.gravity[2]);
    auto sweep = [&](int lo, int hi) {
      for (int i = lo; i < hi; i++) {
        const int jt = M.jtype[i], p = M.parent[i], o = M.dof_off[i];
        const Xf<double> T = ts_xf(M, S, i);
        const V6<double> V = ldv6(sv + i * 21);
        V6<double> Ai = AdInvT(T, (p >= 0) ? ldv6(Aacc + 6 * p) : A0);
        V6<double> Ui = (p >= 0) ? AdInvT(T, ldv6(Uplus + 6 * p)) : zero6<double>();
        V6<double> Us = (bounce && p >= 0) ? AdInvT(T, ldv6(Ustar + 6 * p)) : zero6<double>();
        if (jt != NB2_JT_FREE) {
          const V6<double> Sv = S_times<double>(jt, (double)st[n + o]);
          Ai = Ai + S_times<double>(jt, ws.aeff[o]) + ad(V, Sv);
          Ui = Ui + S_times<double>(jt, ws.vplus[o]);
          if (bounce) Us = Us + S_times<double>(jt, vstar[o]);
        } else {
          V6<double> Sv; Sv.a = mk3<double>((double)st[n + o], (double)st[n + o + 1], (double)st[n + o + 2]); Sv.l = mk3<double>((double)st[n + o + 3], (double)st[n + o + 4], (double)st[n + o + 5]);
          Ai = Ai + ldv6(ws.aeff + o) + ad(V, Sv);
          Ui = Ui + ldv6(ws.vplus + o);
          if (bounce) Us = Us + ldv6(vstar + o);
        }
        stv6(Aacc + 6 * i, Ai); stv6(Uplus + 6 * i, Ui);
        if (bounce) stv6(Ustar + 6 * i, Us);
      }
    };
    CW_FOR(l, 1) for (int r = 0; r < M.trunk_n; r++) sweep(M.trunk_lo[r], M.trunk_hi[r]);
    CW_SYNC();
    CW_FOR(l, M.lanes) for (int r = 0; r < M.limb_n[l]; r++) sweep(M.limb_lo[l][r], M.limb_hi[l][r]);
    CW_SYNC();
  }
  CW_PROF(26);
  CW_PHASE(); ph++;  // 6
  // ---- per-body injections for the reverse sweep: Uw_bar, Up_bar, G (all scaled by -1/dt: they join the (dID/dq)^T w accumulator
  // that is multiplied by -dt at the end) and H (plain: A_c mu propagated to joint space).  One collision body per lane.
  const double kap = -1.0 / dt;
  CW_FOR(j, m) {
    double cW = 0, cV = 0;
    if (clampIdx[j] >= 0) { cW = xr[j]; cV = -mu_c[clampIdx[j]]; }
    else if (mapping[j] >= 0) cW = xr[j];
    coefW[j] = cW; coefV[j] = cV;
  }
  CW_SYNC();
  CW_FOR(k, C.ncb) {
    const int t = C.cb_body[k];
    double* bj = ws.inj + 24 * k;
    for (int e = 0; e < 24; e++) bj[e] = 0;
    for (int j = 0; j < m; j++) {
      const double cW = coefW[j], cV = coefV[j], cH = coefH[j];
      if (cW == 0.0 && cV == 0.0 && cH == 0.0) continue;
      const int c = ws.rowc[j];
      for (int side = 0; side < 2; side++) {
        if ((side ? ws.cbodyB[c] : ws.cbodyA[c]) != t) continue;
        const double* F = (side ? ws.JB : ws.JA) + 6 * j;
        for (int kx = 0; kx < 6; kx++) { bj[kx] += kap * cW * F[kx]; bj[6 + kx] += kap * cV * F[kx]; bj[18 + kx] += cH * F[kx]; }
      }
    }
  }
  CW_SYNC();
  // ---- contact-frame part G: derivatives of every wrench with respect to the pose of each moving body of its pair.  Work item =
  // (pair that produced contacts, body whose pose varies); each item takes 6 lanes, one pose direction each: the contact
  // generator runs on 1-direction dual numbers.  Contacts of a pair are consecutive: groups are found from the shape indices.
  CW_PROF(27);
  CW_PHASE(); ph++;  // 7
  int* gfirst = ws.i1; int* it_g = ws.i2; int* it_dyn = ws.i4;  // cl / ubl are dead by now
  int ncr = nc;  // real contacts: the joint-limit pseudo contacts come last and have no geometry to differentiate (their rows are constant in joint space)
  while (ncr > 0 && ws.ctype[ncr - 1] >= NB2_CT_LIMIT_LOWER) ncr--;
  const int ng = cw_enumerate(ncr, [&](int c) { return c == 0 || ws.cshapeA[c] != ws.cshapeA[c - 1] || ws.cshapeB[c] != ws.cshapeB[c - 1]; },
                              [&](int c, int r) { gfirst[r] = c; });
  CW_SYNC();
  CW_ONE {
    int ni = 0;
    for (int g = 0; g < ng; g++) {
      const int c0 = gfirst[g];
      if (ws.cbodyA[c0] >= 0) { it_g[ni] = g; it_dyn[ni] = ws.cbodyA[c0]; ni++; }
      if (ws.cbodyB[c0] >= 0) { it_g[ni] = g; it_dyn[ni] = ws.cbodyB[c0]; ni++; }
    }
    ws.meta[5] = ni;
  }
  CW_SYNC();
  const int nitems = ws.meta[5];
  bool bad = false;
  for (int it0 = 0; it0 < nitems; it0 += 5) {
    const int cnt = (nitems - it0 < 5) ? nitems - it0 : 5;
    CW_FOR(q, cnt * 6) {
      const int it = it0 + q / 6, kx = q % 6;
      const int g = it_g[it], dyn = it_dyn[it];
      const int c0 = gfirst[g], c1 = (g + 1 < ng) ? gfirst[g + 1] : ncr;
      const int sa = ws.cshapeA[c0], sb = ws.cshapeB[c0], ba = ws.cbodyA[c0], bb = ws.cbodyB[c0];
      Xf<D1> WDa, WDb;
      if (ba >= 0) { const Xf<double> Wa = ldXf<double, 1>(ws.Wcb + 12 * C.cb_of_body[ba]); WDa = (ba == dyn) ? dual_pose1(Wa, kx) : lift1(Wa); }
      if (bb >= 0) { const Xf<double> Wb = ldXf<double, 1>(ws.Wcb + 12 * C.cb_of_body[bb]); WDb = (bb == dyn) ? dual_pose1(Wb, kx) : lift1(Wb); }
      const Xf<D1> TsA = lift1(ldXf<double, 1>(C.shape_T[sa])), TsB = lift1(ldXf<double, 1>(C.shape_T[sb]));
      const Xf<D1> Ta = (ba >= 0) ? gxf_mul(WDa, TsA) : TsA;
      const Xf<D1> Tb = (bb >= 0) ? gxf_mul(WDb, TsB) : TsB;
      ContactOutT<D1> co[8];
      int st2 = 0;
      const int k = pair_contacts_dual(C, sa, sb, Ta, Tb, co, &st2);
      double gsum = 0;
      int cc = c0;
      for (int c = 0; c < k; c++) {
        const double nx = co[c].normal.x.v, ny = co[c].normal.y.v, nz = co[c].normal.z.v;
        if (nx * nx + ny * ny + nz * nz < 1e-12) continue;
        if (co[c].depth.v < 0.0 || co[c].depth.v > C.clip_depth) continue;
        if (cc >= c1) { bad = true; break; }
        const bool fric = ws.cmu[cc] > 1e-3;
        V3<D1> dirs[3]; dirs[0] = co[c].normal;
        if (fric) tangent_basis<D1>(co[c].normal, &dirs[1], &dirs[2]);
        V3<D1> pA, pB;
        if (ba >= 0) pA = gxf_apply_inv(WDa, co[c].point);
        if (bb >= 0) pB = gxf_apply_inv(WDb, co[c].point);
        if (C.pen_correction && coefV[ws.crow[cc]] != 0.0 && !(bounce && eeff[ws.crow[cc]] != 0.0)) {
          // b_normal carries the penetration-correction velocity kpen * depth while it is below its cap (ContactConstraint.cpp:395-408):
          // dL/db = mu, so the pose gradient gains mu * kpen * d(depth)  (gsum is scaled by kap = -1/dt below and by -dt at the end: net +1)
          const double bv = co[c].depth.v * 0.01 * (1.0 / dt);
          if (bv > 0.0 && bv <= 1e-3) gsum -= coefV[ws.crow[cc]] * (0.01 * (1.0 / dt)) * co[c].depth.d[0];  // coefV = -mu
        }
        for (int kk = 0; kk < (fric ? 3 : 1); kk++) {
          const int r = ws.crow[cc] + kk;
          const double cW = coefW[r], cV = coefV[r], cE = bounce ? coefE[r] : 0.0;
          if (cW == 0.0 && cV == 0.0) continue;
          for (int side = 0; side < 2; side++) {
            const int body = side ? bb : ba;
            if (body < 0) continue;
            const V3<D1> dd = side ? mulT(WDb.R_, -dirs[kk]) : mulT(WDa.R_, dirs[kk]);
            const V3<D1> mo = cross(side ? pB : pA, dd);
            const V6<double> Ww = Wfield(body);
            V6<double> Up = ldv6(Uplus + 6 * body) * cV;
            if (cE != 0.0) Up = Up + ldv6(Ustar + 6 * body) * cE;   // - mu_r J_r (v+ + e_r v*)
            gsum += mo.x.d[0] * (cW * Ww.a.x + Up.a.x) + mo.y.d[0] * (cW * Ww.a.y + Up.a.y) + mo.z.d[0] * (cW * Ww.a.z + Up.a.z)
                  + dd.x.d[0] * (cW * Ww.l.x + Up.l.x) + dd.y.d[0] * (cW * Ww.l.y + Up.l.y) + dd.z.d[0] * (cW * Ww.l.z + Up.l.z);
          }
        }
        cc++;
      }
      if (cc != c1) bad = true;
      gpart[q] = kap * gsum;
    }
    CW_SYNC();
    CW_ONE { for (int q = 0; q < cnt * 6; q++) ws.inj[24 * C.cb_of_body[it_dyn[it0 + q / 6]] + 12 + q % 6] += gpart[q]; }
    CW_SYNC();
  }
  CW_PROF(28);
  if (cw_any(bad)) { cd.error = 3; cd.active = 0; }
  else if (bounce) {
    cd.bounce = 1;
    CW_ONE { ws.meta[6] = m; ws.meta[7] = (int)(dVb - ws.M1); }  // for bounce_pass2_begin (which re-derives the array addresses)
    CW_SYNC();
  }
  return cd;
}

// Second reverse sweep of a bouncing world.  begin: all lanes, after the first B3 (trunk included) and before the assembly: the scratch takes
// the field of -nu_e, the injections become those of the v* term, and the returned view makes bwd_B3 read the unconstrained accelerations
// and ADD its results.  end: the multiplier of the assembly becomes w_B = w - nu_e.
NB2_HD BwdContactData<1> bounce_pass2_begin(const Nb2ModelDev<double>& M, const Nb2ContactDev& C, const Ws& ws, const BwdContactData<1>& cd, double* scr,
                                            int oLam, int oBody) {
  const int nb = M.nb, n = M.ndof, m = ws.meta[6];
  double* dVb = ws.M1 + ws.meta[7];
  double* Ustar = dVb + (size_t)nb * 18; double* dVbE = Ustar + (size_t)nb * 6;
  double* wold = dVbE + (size_t)nb * 6; double* nue = wold + n; double* vstar = nue + n;
  const double* coefE = ws.v6;
  const double kap = -1.0 / M.dt;
  CW_FOR(dd, n) { wold[dd] = scr[oLam + dd]; scr[oLam + dd] = -nue[dd]; }
  CW_FOR(e, nb * 6) { const int i = e / 6, k = e - 6 * i; scr[oBody + 7 * i + 1 + k] = -dVbE[e]; }
  CW_FOR(k, C.ncb) {
    const int t = C.cb_body[k];
    double* bj = ws.inj + 24 * k;
    for (int e = 0; e < 24; e++) bj[e] = 0;
    for (int j = 0; j < m; j++) {
      const double cE = coefE[j];
      if (cE == 0.0) continue;
      const int c = ws.rowc[j];
      for (int side = 0; side < 2; side++) {
        if ((side ? ws.cbodyB[c] : ws.cbodyA[c]) != t) continue;
        const double* F = (side ? ws.JB : ws.JA) + 6 * j;
        for (int kx = 0; kx < 6; kx++) bj[6 + kx] += kap * cE * F[kx];
      }
    }
  }
  CW_SYNC();
  BwdContactData<1> c2 = cd;
  c2.pass2 = 1; c2.Uplus.p = Ustar; c2.vplus.p = vstar;
  return c2;
}
NB2_HD void bounce_pass2_end(const Nb2ModelDev<double>& M, const Ws& ws, double* scr, int oLam) {
  const int nb = M.nb, n = M.ndof;
  double* dVb = ws.M1 + ws.meta[7];
  double* wold = dVb + (size_t)nb * 30; double* nue = wold + n;
  CW_SYNC();
  CW_FOR(dd, n) scr[oLam + dd] = wold[dd] - nue[dd];
  CW_SYNC();
}

}  // namespace cw
}  // namespace nb2
