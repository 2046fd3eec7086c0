// libnb2.so — kernels + C ABI (include/nb2.h).  sm_90a only.
//
// Kernel shape (contact-free step): ONE THREAD PER WORLD, 32 worlds per warp.  The model is a __grid_constant__
// kernel parameter (constant-bank, warp-uniform loads); per-world working storage lives in dynamic shared memory,
// interleaved [word][lane] so every access is bank-conflict free; the only HBM traffic is the fp32 state/action
// rows, the outputs and the saved-for-backward stream ([word][B]: coalesced).  All branches depend on the model
// only, so warps never diverge.  See DESIGN.md for the roofline discussion (the path is FP32-latency bound).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/nb2.h"
#include "nb2_dyn.cuh"
#include "nb2_cw.cuh"
#include "nb2_host_model.h"

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

#define NB2_CUDA(call)                                                                           \
  do {                                                                                           \
    cudaError_t e_ = (call);                                                                     \
    if (e_ != cudaSuccess) {                                                                     \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                                \
      return NB2_ERR_CUDA;                                                                       \
    }                                                                                            \
  } while (0)

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
  for (int k = threadIdx.x; k < M.nb * NB2_BT_WORDS; k += blockDim.x) {
    const int i = k / NB2_BT_WORDS, j = k - i * NB2_BT_WORDS;
    tab[k] = (j < 12) ? M.Xtree[i][j] : M.inertia[i][j - 12];
  }
  __syncthreads();
  return tab;
  }
}

// ---- bulk (TMA) staging of a group's input rows.  The rows of the worlds of one warp are contiguous in global memory, so
// ONE thread hands each block of rows to the copy engine of the SM (cp.async.bulk, completion counted on an mbarrier) instead
// of 32 threads looping over vector loads: the requests are as wide as they can be — which is what matters when `src` is
// mapped host memory behind PCIe — and cost two instructions.  The scatter into the [word][slot] scratch then reads shared
// memory.  Needs 16-byte aligned sources and sizes; otherwise the vector-load path is used.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  for (int it = 0; it < (1 << 20); it++) {  // bounded: a copy that never lands must not hang the GPU
    unsigned ok;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (ok) return;
  }
  __trap();
}
__device__ __forceinline__ bool bulk_ok(const void* p, size_t bytes) { return ((reinterpret_cast<size_t>(p) | bytes) & 15) == 0 && bytes > 0; }
// bytes of staging per warp: rows of `nrows` floats per world, rounded to 16 + the mbarrier
template <int K> __host__ __device__ constexpr size_t staging_bytes(int floats_per_world) {
  return (((size_t)floats_per_world * CoopShape<K>::WPW * sizeof(float) + 15) & ~(size_t)15) + 16;
}

// PW: the variant with a per-world inertia table (nb2_step_forward_pw).  A compile-time switch: as a run-time pointer test it cost the
// shared-table kernels registers (fp32) and spills (fp64).
template <class R, int K, bool PW>
__global__ void __launch_bounds__(128)
k_step_fwd(const __grid_constant__ Nb2ModelDev<R> M, int B, int w0, int count, const float* __restrict__ state,
           const float* __restrict__ action, float* __restrict__ next, R* __restrict__ saved, int words,
           float* __restrict__ state_copy, float* __restrict__ action_copy, const double* __restrict__ winertia) {
  // worlds [w0, w0 + count) of a batch of B (B is the stride of the saved stream and of the per-world inertia; the host entry points launch chunks)
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  constexpr int WPW = CoopShape<K>::WPW, ST = CoopShape<K>::ST;
  const int li = threadIdx.x & 31, slot = li / K, lane = li % K;
  const int g0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * WPW;  // first world of this warp's group
  const int nworlds = min(WPW, count - g0);                                      // <= 0: idle warp (grid tail)
  const bool valid = slot < nworlds;
  const size_t wg = (size_t)w0 + (nworlds > 0 ? g0 : 0);
  const R* bt = stage_body_table<R, K>(M, reinterpret_cast<R*>(nb2_smem));
  R* scr0 = reinterpret_cast<R*>(nb2_smem) + body_table_words<K>(M.nb) + (size_t)(threadIdx.x >> 5) * words * ST;
  R* scr = scr0 + slot;
  R* sv = saved ? saved + wg + (valid ? slot : 0) : nullptr;
  const double* wi = PW ? winertia + wg + (valid ? slot : 0) : nullptr;
  constexpr unsigned sync_mask = (K > 1) ? NB2_FWD_SYNC_MASK : NB2_FWD_SYNC_MASK_1LANE;
  // input rows of the group: through the bulk-copy staging buffer when they qualify, else read in place
  const float* st_src = state + wg * 2 * M.ndof;
  const float* act_src = action + wg * M.na;
  if (nworlds > 0) {
    const size_t sb = (size_t)nworlds * 2 * M.ndof * sizeof(float), ab = (size_t)nworlds * M.na * sizeof(float);
    if (bulk_ok(st_src, sb) && bulk_ok(act_src, ab)) {
      unsigned char* stg = nb2_smem + (((size_t)body_table_words<K>(M.nb) + (size_t)(blockDim.x >> 5) * words * ST) * sizeof(R) + 15 & ~(size_t)15) +
                           (size_t)(threadIdx.x >> 5) * staging_bytes<K>(2 * M.ndof + M.na);
      unsigned long long* bar = reinterpret_cast<unsigned long long*>(stg + staging_bytes<K>(2 * M.ndof + M.na) - 16);
      if (li == 0) {
        mbar_init(bar);
        mbar_expect_tx(bar, (unsigned)(sb + ab));
        bulk_g2s(stg, st_src, (unsigned)sb, bar);
        bulk_g2s(stg + sb, act_src, (unsigned)ab, bar);
      }
      __syncwarp();
      mbar_wait(bar, 0);
      st_src = reinterpret_cast<const float*>(stg);
      act_src = reinterpret_cast<const float*>(stg + sb);
    }
  }
#pragma unroll 1
  for (int sg = 0; sg < NB2_FWD_STAGES; sg++) {
    if (sg == 0) {
      if (nworlds > 0) nb2::fwd_load<R, ST>(M, scr0, st_src, act_src, nworlds, li, 32,
                                            state_copy ? state_copy + wg * 2 * M.ndof : nullptr, action_copy ? action_copy + wg * M.na : nullptr);
    }
    else if (sg == NB2_FWD_STAGES - 1) { if (nworlds > 0) nb2::fwd_store<R, ST>(M, scr0, next + wg * 2 * M.ndof, nworlds, li, 32); }
    else if (valid) nb2::world_forward_stage<R, ST>(M, scr, sv, (size_t)B, saved != nullptr, lane, sg, bt, nullptr, wi, (size_t)B);
    if ((sync_mask >> sg) & 1u) __syncwarp();
  }
}

template <class R, int K, bool PW>
__global__ void __launch_bounds__(128)
k_step_bwd(const __grid_constant__ Nb2ModelDev<R> M, int B, int w0, int count, const float* __restrict__ state,
           const float* __restrict__ action, const R* __restrict__ saved, const float* __restrict__ gnext,
           float* __restrict__ gstate, float* __restrict__ gaction, float* __restrict__ ginertia, int words,
           int stage_saved, int accumulate_state, unsigned in_stage_off, const double* __restrict__ winertia, double* __restrict__ ginertia_acc) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  constexpr int WPW = CoopShape<K>::WPW, ST = CoopShape<K>::ST;
  const int li = threadIdx.x & 31, slot = li / K, lane = li % K;
  const int g0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * WPW;
  const int nworlds = min(WPW, count - g0);
  const bool valid = slot < nworlds;
  const size_t wg = (size_t)w0 + (nworlds > 0 ? g0 : 0);
  const size_t w = wg + (valid ? slot : 0);
  const R* bt = stage_body_table<R, K>(M, reinterpret_cast<R*>(nb2_smem));
  R* scr0 = reinterpret_cast<R*>(nb2_smem) + body_table_words<K>(M.nb) + (size_t)(threadIdx.x >> 5) * words * ST;
  R* scr = scr0 + slot;
  // The sweeps walk the saved stream body by body, every access a dependent DRAM round trip.  When the launch leaves room
  // (small batches: the regime where latency is all that matters) each warp first pulls its group's rows of the stream
  // into shared memory with one burst of asynchronous 16-byte copies ([word][B] layout: the group's worlds are adjacent),
  // and the sweeps then read `svp` with stride `svB` = WPW instead of the global stream with stride B.
  const R* svp = saved + wg + (valid ? slot : 0);
  size_t svB = (size_t)B;
  if (stage_saved && nworlds == WPW) {
    const int sw = nb2_saved_words(M.nb, M.ndof, M.nfree);
    R* svs = reinterpret_cast<R*>(nb2_smem) + ((body_table_words<K>(M.nb) + (size_t)(blockDim.x >> 5) * words * ST + 3) & ~(size_t)3)  // 16-byte aligned
             + (size_t)(threadIdx.x >> 5) * sw * WPW;
    constexpr int CH = (WPW * (int)sizeof(R)) / 16;  // 16-byte chunks per row of the group
    const unsigned dst0 = (unsigned)__cvta_generic_to_shared(svs);
    const char* src0 = reinterpret_cast<const char*>(saved + wg);
    for (int idx = li; idx < sw * CH; idx += 32) {
      const int k = idx / CH, c = idx - k * CH;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst0 + (unsigned)(k * WPW * (int)sizeof(R) + c * 16)),
                   "l"(src0 + (size_t)k * B * sizeof(R) + c * 16));
    }
    asm volatile("cp.async.commit_group;");
    svp = svs + slot;
    svB = WPW;
  }
  constexpr unsigned sync_mask = (K > 1) ? NB2_BWD_SYNC_MASK : NB2_BWD_SYNC_MASK_1LANE;
  // input rows (dL/dx', x, u) of the group through the bulk-copy staging buffer when they qualify (see k_step_fwd)
  const float* g_src = gnext + wg * 2 * M.ndof;
  const float* st_src = state + wg * 2 * M.ndof;
  const float* act_src = action + wg * M.na;
  if (nworlds > 0 && in_stage_off) {
    const size_t sb = (size_t)nworlds * 2 * M.ndof * sizeof(float), ab = (size_t)nworlds * M.na * sizeof(float);
    if (bulk_ok(g_src, sb) && bulk_ok(st_src, sb) && bulk_ok(act_src, ab)) {
      unsigned char* stg = nb2_smem + in_stage_off + (size_t)(threadIdx.x >> 5) * staging_bytes<K>(4 * M.ndof + M.na);
      unsigned long long* bar = reinterpret_cast<unsigned long long*>(stg + staging_bytes<K>(4 * M.ndof + M.na) - 16);
      if (li == 0) {
        mbar_init(bar);
        mbar_expect_tx(bar, (unsigned)(2 * sb + ab));
        bulk_g2s(stg, g_src, (unsigned)sb, bar);
        bulk_g2s(stg + sb, st_src, (unsigned)sb, bar);
        bulk_g2s(stg + 2 * sb, act_src, (unsigned)ab, bar);
      }
      __syncwarp();
      mbar_wait(bar, 0);
      g_src = reinterpret_cast<const float*>(stg);
      st_src = reinterpret_cast<const float*>(stg + sb);
      act_src = reinterpret_cast<const float*>(stg + 2 * sb);
    }
  }
#pragma unroll 1
  for (int sg = 0; sg < NB2_BWD_STAGES; sg++) {
    if (sg == 0) { if (nworlds > 0) nb2::bwd_load<R, ST, false>(M, scr0, st_src, act_src, g_src, nworlds, li, 32); }
    else if (sg == NB2_BWD_STAGES - 1) {
      if (nworlds > 0) nb2::bwd_store<R, ST, false>(M, scr0, gstate + wg * 2 * M.ndof, gaction + wg * M.na, false, nworlds, li, 32, accumulate_state != 0);
    } else if (valid) nb2::world_backward_stage<R, ST>(M, scr, svp, svB, lane, sg, ginertia ? ginertia + w : nullptr, bt, (size_t)B, nullptr,
                                                       (PW && winertia) ? winertia + w : nullptr, (size_t)B, (PW && ginertia_acc) ? ginertia_acc + w : nullptr);
    if (sg == 0 && stage_saved) asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (((sync_mask >> sg) & 1u) || (sg == 0 && stage_saved)) __syncwarp();
  }
}

// ---- fused step kernels of worlds WITH a contact stage (fp64): ONE WARP PER WORLD.
// Forward: group load -> the three ABA sweeps on the first M.lanes lanes (trunk / limb schedule) -> the warp-cooperative contact /
// boxed-LCP stage on all 32 lanes (nb2_cw.cuh) -> store.  Everything a world needs — ABA scratch, contact list, LCP matrix and its
// factors — sits in that warp's slice of shared memory; HBM sees the fp32 rows, the LCP warm start and what the backward needs
// (the saved stream, world-major, and a ~1 KB record).  Backward: the lambda sweeps, the contact adjoint, the reverse RNEA sweep.
// Blocks are one warp: no block-level barrier exists in these kernels, and a warp whose world is out of range simply leaves.
#define NB2_WS_DESC_DOUBLES ((int)((sizeof(nb2::cw::Ws) + 15) / 16 * 2))  // the workspace descriptor sits in front of the arrays
// the warp's contact workspace at `at`: lane 0 carves the arrays after the descriptor and writes it, the warp syncs before reading it
__device__ __forceinline__ nb2::cw::Ws* warp_workspace(void* at, const nb2::cw::Dims& d, int lane) {
  nb2::cw::Ws* wsm = reinterpret_cast<nb2::cw::Ws*>(at);
  if (lane == 0) *wsm = nb2::cw::carve(reinterpret_cast<double*>(wsm) + NB2_WS_DESC_DOUBLES, d);
  __syncwarp();
  return wsm;
}
#ifndef NB2_CSTEP_MINB
#define NB2_CSTEP_MINB 1   // resident warps per SM the register allocation of the fused contact kernels aims at
#endif
struct CStepArgs {
  int B, fwd_words, bwd_words, saved_words;
  size_t ws_small_doubles;   // doubles of the shared contact workspace (after the scratch)
  nb2::cw::Dims ds, db;
  nb2::cw::BigPool pool;
  size_t rec_doubles;
  // three-kernel forward: exchange records and the workspace shapes of the solve / apply kernels
  double* exch; size_t exch_stride;
  nb2::cw::Dims ds_solve, db_solve, ds_apply, db_apply;
  nb2::cw::BigPool pool_solve, pool_solve_b, pool_apply;
  int *todo, *todo_count;
};
__global__ void __launch_bounds__(32, NB2_CSTEP_MINB)
k_cstep_fwd(const __grid_constant__ Nb2ModelDev<double> M, const __grid_constant__ Nb2ContactDev C, const __grid_constant__ CStepArgs P,
            const float* __restrict__ state, const float* __restrict__ action, float* __restrict__ next, double* __restrict__ saved,
            double* __restrict__ x_lcp, int* __restrict__ m_lcp, int* __restrict__ labels, int* __restrict__ status,
            int* __restrict__ ncontacts, float* __restrict__ cinfo, double* __restrict__ crec, int* __restrict__ status_accum,
            const double* __restrict__ winertia) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int w = blockIdx.x, lane = threadIdx.x & 31;
  if (w >= P.B) return;
  const double* wi = winertia ? winertia + w : nullptr;
  double* scr = reinterpret_cast<double*>(nb2_smem);
  nb2::cw::Ws* wsm = warp_workspace(scr + ((P.fwd_words + 1) & ~1), P.ds, lane);
  const nb2::cw::Ws& ws0 = *wsm;
  const float* st = state + (size_t)w * 2 * M.ndof;
  double* sv = saved ? saved + (size_t)w * P.saved_words : nullptr;
  using namespace nb2::cw;
  CW_PROF_DECL;
  nb2::fwd_load<double, 1>(M, scr, st, action + (size_t)w * M.na, 1, lane, 32);
  __syncwarp();
#pragma unroll 1
  for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++) {
    if (lane < M.lanes) nb2::world_forward_stage<double, 1>(M, scr, sv, 1, sv != nullptr, lane, sg, nullptr, ws0.Iinv, wi, (size_t)P.B);
    if ((NB2_FWD_SYNC_MASK >> sg) & 1u) __syncwarp();
  }
  __syncwarp();
  CW_PROF(0);
  nb2::cw::FwdIO io;
  io.x_io = x_lcp + (size_t)w * NB2_MAX_ROWS; io.m_io = m_lcp + w; io.labels = labels + (size_t)w * NB2_MAX_ROWS; io.status = status + w;
  io.nc = ncontacts + w; io.cinfo = cinfo ? cinfo + (size_t)w * NB2_MAX_CONTACTS * 10 : nullptr; io.rec = crec ? crec + (size_t)w * P.rec_doubles : nullptr;
  nb2::cw::contact_forward(M, C, scr, st, wsm, P.ds, P.pool, P.db, ws0.Iinv, io);
  __syncwarp();
  if (status_accum && lane == 0) status_accum[w] |= status[w];  // sticky copy: one word per world, owned by this warp
  CW_PROF(7);
  nb2::fwd_store<double, 1>(M, scr, next + (size_t)w * 2 * M.ndof, 1, lane, 32);
  CW_PROF(8);
}

// ---- the forward step as three kernels (nb2_cw.cuh: build | solve | apply): same arithmetic as k_cstep_fwd.  Several worlds per
// block, one warp each, phases in lockstep (see k_csolve).
#define NB2_CBUILD_MAXW 8
__global__ void __launch_bounds__(32 * NB2_CBUILD_MAXW, 1)
k_cbuild(const __grid_constant__ Nb2ModelDev<double> M, const __grid_constant__ Nb2ContactDev C, const __grid_constant__ CStepArgs P,
         const float* __restrict__ state, const float* __restrict__ action, float* __restrict__ next, double* __restrict__ saved,
         int* __restrict__ m_lcp, int* __restrict__ status, int* __restrict__ ncontacts, float* __restrict__ cinfo, double* __restrict__ crec,
         size_t smem_per_warp, const double* __restrict__ winertia) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int w = blockIdx.x * wpb + warp;
  const bool live = w < P.B;
  const int wc = live ? w : P.B - 1;  // a warp without a world redoes the last one (reads only) so that it walks the same code
  const double* wi = winertia ? winertia + wc : nullptr;
  double* scr = reinterpret_cast<double*>(nb2_smem + (size_t)warp * smem_per_warp);
  nb2::cw::Ws* wsm = warp_workspace(scr + ((P.fwd_words + 1) & ~1), P.ds, lane);
  const nb2::cw::Ws& ws0 = *wsm;
  const float* st = state + (size_t)wc * 2 * M.ndof;
  double* sv = live ? saved + (size_t)w * P.saved_words : nullptr;
  using namespace nb2::cw;
  CW_PROF_DECL;
  nb2::fwd_load<double, 1>(M, scr, st, action + (size_t)wc * M.na, 1, lane, 32);
  __syncwarp();
#pragma unroll 1
  for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++) {
    __syncthreads();  // lockstep: every warp of the block sweeps the same stage
    if (lane < M.lanes) nb2::world_forward_stage<double, 1>(M, scr, sv, 1, sv != nullptr, lane, sg, nullptr, ws0.Iinv, wi, (size_t)P.B);
    if ((NB2_FWD_SYNC_MASK >> sg) & 1u) __syncwarp();
  }
  __syncwarp();
  __syncthreads();
  CW_PROF(0);
  nb2::cw::FwdIO io;
  io.x_io = nullptr; io.m_io = m_lcp + wc; io.labels = nullptr; io.status = status + wc;
  io.nc = ncontacts + wc; io.cinfo = cinfo ? cinfo + (size_t)wc * NB2_MAX_CONTACTS * 10 : nullptr; io.rec = crec ? crec + (size_t)wc * P.rec_doubles : nullptr;
  nb2::cw::contact_build(M, C, scr, st, wsm, P.ds, P.pool, P.db, io, live ? P.exch + (size_t)w * P.exch_stride : nullptr);
  __syncwarp();
  if (live) nb2::fwd_store<double, 1>(M, scr, next + (size_t)w * 2 * M.ndof, 1, lane, 32);  // [q+ ; v*]: the apply kernel replaces v* by v+ where there are contacts
}
// Several worlds per block (one warp each): the warps run the phases of the chain in LOCKSTEP (CW_PHASE = __syncthreads), so that the
// SM fetches each piece of code once for all of them.  The warp count per block is chosen at launch (shared memory, batch size).
#define NB2_CSOLVE_MAXW 12
// solve kernel A (every world: warm start + short-circuit classification) / B (the worlds A listed in `todo`: the rest of the chain)
template <int PART>
__global__ void __launch_bounds__(32 * NB2_CSOLVE_MAXW, 1)
k_csolve(const __grid_constant__ Nb2ContactDev C, const __grid_constant__ CStepArgs P, int ndof, double* __restrict__ x_lcp, int* __restrict__ m_lcp,
         int* __restrict__ labels, int* __restrict__ status, double* __restrict__ crec, int* __restrict__ status_accum, size_t smem_per_warp,
         int* __restrict__ todo, int* __restrict__ todo_count) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int idx = blockIdx.x * wpb + warp;
  int w = idx;
  bool live = idx < P.B;
  if (PART == 1) {
    const int cnt = *todo_count;
    if (blockIdx.x * wpb >= cnt) return;  // the whole block has nothing to do
    live = idx < cnt;
    w = live ? todo[idx] : 0;
  }
  double* X = live ? P.exch + (size_t)w * P.exch_stride : nullptr;
  nb2::cw::Ws* wsm = warp_workspace(nb2_smem + (size_t)warp * smem_per_warp, P.ds_solve, lane);
  nb2::cw::FwdIO io;
  const int wc = live ? w : 0;
  io.x_io = x_lcp + (size_t)wc * NB2_MAX_ROWS; io.m_io = m_lcp + wc; io.labels = labels + (size_t)wc * NB2_MAX_ROWS; io.status = status + wc;
  io.nc = nullptr; io.cinfo = nullptr; io.rec = crec ? crec + (size_t)wc * P.rec_doubles : nullptr;
  if (PART == 0) nb2::cw::contact_solve_a(C, ndof, wsm, P.ds_solve, P.pool_solve, P.db_solve, io, X, status_accum ? status_accum + wc : nullptr, w, todo, todo_count);
  else nb2::cw::contact_solve_b(C, ndof, wsm, P.ds_solve, P.pool_solve_b, P.db_solve, io, X, status_accum ? status_accum + wc : nullptr);
}
#define NB2_CAPPLY_MAXW 16
__global__ void __launch_bounds__(32 * NB2_CAPPLY_MAXW, 1)
k_capply(const __grid_constant__ Nb2ModelDev<double> M, const __grid_constant__ Nb2ContactDev C, const __grid_constant__ CStepArgs P,
         const float* __restrict__ state, float* __restrict__ next, const double* __restrict__ saved, double* __restrict__ x_lcp,
         int* __restrict__ labels, double* __restrict__ crec, size_t smem_per_warp) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int w = blockIdx.x * wpb + warp;
  const bool live = w < P.B;
  const int wc = live ? w : 0;
  const double* X = live ? P.exch + (size_t)w * P.exch_stride : nullptr;
  nb2::cw::Ws* wsm = warp_workspace(nb2_smem + (size_t)warp * smem_per_warp, P.ds_apply, lane);
  nb2::cw::FwdIO io;
  io.x_io = x_lcp + (size_t)wc * NB2_MAX_ROWS; io.m_io = nullptr; io.labels = labels + (size_t)wc * NB2_MAX_ROWS; io.status = nullptr;
  io.nc = nullptr; io.cinfo = nullptr; io.rec = crec ? crec + (size_t)wc * P.rec_doubles : nullptr;
  nb2::cw::contact_apply(M, C, state + (size_t)wc * 2 * M.ndof, saved + (size_t)wc * P.saved_words, wsm, P.ds_apply, P.pool_apply, P.db_apply, io, X,
                         next + (size_t)wc * 2 * M.ndof + M.ndof);
}

#define NB2_CBWD_MAXW 8
template <bool BOUNCE>
__global__ void __launch_bounds__(32 * NB2_CBWD_MAXW, 1)
k_cstep_bwd(const __grid_constant__ Nb2ModelDev<double> M, const __grid_constant__ Nb2ContactDev C, const __grid_constant__ CStepArgs P,
            const float* __restrict__ state, const float* __restrict__ action, const double* __restrict__ saved, const double* __restrict__ crec,
            const float* __restrict__ gnext, float* __restrict__ gstate, float* __restrict__ gaction, float* __restrict__ ginertia,
            int* __restrict__ status, size_t smem_per_warp, int stage_saved, int accumulate_state, const double* __restrict__ winertia,
            double* __restrict__ ginertia_acc) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int w = blockIdx.x * wpb + warp;
  const bool live = w < P.B;
  const int wc = live ? w : P.B - 1;  // a warp without a world redoes the last one without storing anything
  double* scr = reinterpret_cast<double*>(nb2_smem + (size_t)warp * smem_per_warp);
  nb2::cw::Ws* wsm = warp_workspace(scr + ((P.bwd_words + 1) & ~1), P.ds, lane);
  double* wsb = reinterpret_cast<double*>(wsm) + NB2_WS_DESC_DOUBLES;
  const float* st = state + (size_t)wc * 2 * M.ndof;
  // when shared memory allows it WITHOUT costing a resident world, the world's saved stream (world-major, ~5 KB) is pulled into shared
  // memory by one bulk copy (TMA) while the group load runs: the sweeps walk it body by body, each a dependent L2 / DRAM round trip
  // otherwise.  (Measured: +2 % on half-cheetah; on Atlas it would cost one of seven worlds per SM and lose 4 %.)
  const double* sv = saved + (size_t)wc * P.saved_words;
  double* svs = wsb + ((P.ws_small_doubles + 1) & ~(size_t)1);  // 16-byte aligned destination of the bulk copy
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(svs + ((P.saved_words + 1) & ~1));
  const unsigned sv_bytes = (unsigned)(P.saved_words * sizeof(double));
  const bool staged = stage_saved && bulk_ok(sv, sv_bytes);
  if (staged && lane == 0) { mbar_init(bar); mbar_expect_tx(bar, sv_bytes); bulk_g2s(svs, sv, sv_bytes, bar); }
  const nb2::BwdLayout L = nb2::bwd_layout(M.nb, M.ndof, M.nslots, M.nfree, 42);
  using namespace nb2::cw;
  CW_PROF_DECL;
  nb2::bwd_load<double, 1, true>(M, scr, st, action + (size_t)wc * M.na, gnext + (size_t)wc * 2 * M.ndof, 1, lane, 32);
  __syncwarp();
  if (staged) { mbar_wait(bar, 0); sv = svs; }
  nb2::BwdContactData<1> cd; cd.active = 0; cd.error = 0; cd.inj_of_body = nullptr;
  nb2::BwdContactData<1> c2 = cd;
  float* gI = (ginertia && live) ? ginertia + w : nullptr;
  double* gIa = (ginertia_acc && live) ? ginertia_acc + w : nullptr;
  const double* wi = winertia ? winertia + wc : nullptr;
  // stage order: nb2::cbwd_iter.  One call site for all of them (code size), one block-wide barrier per entry (lockstep, see k_csolve):
  // worlds without a bounce only wait at the two extra barriers.
#pragma unroll 1
  for (int it = 0; it < NB2_CBWD_ITERS; it++) {
    const auto [sg, second] = nb2::cbwd_iter(it);
    if (!BOUNCE && second) continue;
    if (it == 4) {  // lambda and its fields are complete: the contact adjoint turns them into w and prepares the injections
      __syncwarp();
      CW_PROF(20);
#ifndef NB2_DEV_NO_CBWD
      cd = nb2::cw::contact_backward<BOUNCE>(M, C, st, sv, wsm, P.ds, P.pool, P.db, crec + (size_t)wc * P.rec_doubles, scr, L.oLam, L.oBody);
#endif
      __syncwarp();
      CW_PROF(29);
    }
    __syncthreads();
#ifdef NB2_DEV_NO_B3
    if (sg == 5 || sg == 7) continue;
#endif
    if (BOUNCE) {
      if (second && !cd.bounce) continue;
      if (it == 6) c2 = nb2::cw::bounce_pass2_begin(M, C, *wsm, cd, scr, L.oLam, L.oBody);
      if (it == 8 && cd.bounce) nb2::cw::bounce_pass2_end(M, *wsm, scr, L.oLam);
    }
    if (lane < M.lanes) nb2::world_backward_stage<double, 1, true>(M, scr, sv, 1, lane, sg, gI, nullptr, (size_t)P.B, (BOUNCE && second) ? &c2 : &cd,
                                                                   wi, (size_t)P.B, gIa);
    __syncwarp();
  }
  __syncwarp();
  if (live) {
    nb2::bwd_store<double, 1, true>(M, scr, gstate + (size_t)w * 2 * M.ndof, gaction + (size_t)w * M.na, cd.error != 0, 1, lane, 32, accumulate_state != 0);
    if (cd.error && status && lane == 0) atomicOr(status + w, NB2_ST_BWD_ERROR);
  }
  CW_PROF(30);
}


// =====================================================================================================
// IKMapping (row f4): world poses / spatial velocities of chosen bodies as a function of the state, and the VJP.
// reference: neural/IKMapping.cpp:146-237 (getPositionsInPlace / getVelocitiesInPlace), :371-476 (getPosJacobian / getVelJacobian built from
// Skeleton::getWorldPositionJacobian / getWorldJacobian), python/nimblephysics/mapping.py:23-114 (map_to_pos / map_to_vel and their backward).
// One thread per (world, entry) forward; one thread per world backward (it owns the gradient row: deterministic sums, no atomics).  Every
// entry walks its own root -> body chain (depth ~10), so nothing but the state row is read and nothing is staged.
// =====================================================================================================
struct IkEntryDev { int type, body, pos_off, vel_off; double T[12]; };  // body: canonical owner (-1 = static); T: owner frame <- entry body frame
#define NB2_IK_SPATIAL 0
#define NB2_IK_LINEAR 1
#define NB2_IK_ANGULAR 2
#define NB2_IK_COM 3

using nb2::V3; using nb2::V6; using nb2::Xf; using nb2::M3;
// parent <- child transform of body j at generalized position q (fwd_pass1's three cases)
__device__ __forceinline__ Xf<double> ik_joint_xf(const Nb2ModelDev<double>& M, int j, const float* q) {
  const int jt = M.jtype[j], o = M.dof_off[j];
  if (jt == NB2_JT_REV) { double s, c; sincos((double)q[o], &s, &c); return nb2::xf_rev<double>(M, j, s, c); }
  if (jt == NB2_JT_PRIS) return nb2::xf_pris<double>(M, j, (double)q[o]);
  Xf<double> X = nb2::xtree<double>(M, j), T;
  T.R_ = nb2::mul(X.R_, nb2::expmap(nb2::mk3<double>(q[o], q[o + 1], q[o + 2])));
  T.p = nb2::mul(X.R_, nb2::mk3<double>(q[o + 3], q[o + 4], q[o + 5])) + X.p;
  return T;
}
__device__ __forceinline__ int ik_chain(const Nb2ModelDev<double>& M, int body, unsigned char* chain) {
  int d = 0;
  for (int j = body; j >= 0; j = M.parent[j]) chain[d++] = (unsigned char)j;
  return d;  // chain[d-1] is the root
}
// world transform W and body-frame spatial velocity V of canonical body `body`
__device__ __forceinline__ void ik_fk(const Nb2ModelDev<double>& M, int body, const float* q, const float* qd, Xf<double>* W, V6<double>* V) {
  unsigned char chain[NB2_MAX_BODIES];
  const int d = ik_chain(M, body, chain);
  Xf<double> Wc; V6<double> Vc = nb2::zero6<double>();
  for (int k = d - 1; k >= 0; k--) {
    const int j = chain[k], jt = M.jtype[j], o = M.dof_off[j];
    const Xf<double> T = ik_joint_xf(M, j, q);
    Wc = (k == d - 1) ? T : nb2::gxf_mul(Wc, T);
    Vc = (k == d - 1) ? nb2::zero6<double>() : nb2::AdInvT(T, Vc);
    if (jt == NB2_JT_REV) Vc.a.z += (double)qd[o];
    else if (jt == NB2_JT_PRIS) Vc.l.z += (double)qd[o];
    else { Vc.a = Vc.a + nb2::mk3<double>(qd[o], qd[o + 1], qd[o + 2]); Vc.l = Vc.l + nb2::mk3<double>(qd[o + 3], qd[o + 4], qd[o + 5]); }
  }
  *W = Wc; *V = Vc;
}
// adjoint of ik_fk for one body: world wrenches about the WORLD ORIGIN (torque n, force f) paired with position perturbations (np, fp) and with
// velocities (nv, fv) -> += into the gradient row g = [g_q ; g_qdot]
__device__ __forceinline__ void ik_fk_vjp(const Nb2ModelDev<double>& M, int body, const float* q, const V3<double>& np, const V3<double>& fp,
                                          const V3<double>& nv, const V3<double>& fv, float* g) {
  unsigned char chain[NB2_MAX_BODIES];
  const int d = ik_chain(M, body, chain), n = M.ndof;
  Xf<double> Wc;
  for (int k = d - 1; k >= 0; k--) {
    const int j = chain[k], jt = M.jtype[j], o = M.dof_off[j];
    const Xf<double> T = ik_joint_xf(M, j, q);
    Wc = (k == d - 1) ? T : nb2::gxf_mul(Wc, T);
    // wrench in the frame of body j: the generalized force on its dofs is S^T of it
    const V3<double> cpa = nb2::mulT(Wc.R_, np - nb2::cross(Wc.p, fp)), cpl = nb2::mulT(Wc.R_, fp);
    const V3<double> cva = nb2::mulT(Wc.R_, nv - nb2::cross(Wc.p, fv)), cvl = nb2::mulT(Wc.R_, fv);
    if (jt == NB2_JT_REV) { g[o] += (float)cpa.z; g[n + o] += (float)cva.z; }
    else if (jt == NB2_JT_PRIS) { g[o] += (float)cpl.z; g[n + o] += (float)cvl.z; }
    else {
      // positions: R = exp(phi), p in the parent frame: body-frame twist of (d phi, d p) is (Jr(phi) d phi, R^T d p) (cf. bwd_B3)
      const V3<double> phi = nb2::mk3<double>(q[o], q[o + 1], q[o + 2]);
      const V3<double> ga = nb2::mulT(nb2::so3_Jr(phi), cpa), gl = nb2::mul(nb2::expmap(phi), cpl);
      g[o] += (float)ga.x; g[o + 1] += (float)ga.y; g[o + 2] += (float)ga.z; g[o + 3] += (float)gl.x; g[o + 4] += (float)gl.y; g[o + 5] += (float)gl.z;
      g[n + o] += (float)cva.x; g[n + o + 1] += (float)cva.y; g[n + o + 2] += (float)cva.z;
      g[n + o + 3] += (float)cvl.x; g[n + o + 4] += (float)cvl.y; g[n + o + 5] += (float)cvl.z;
    }
  }
}
__device__ __forceinline__ int ik_root(const Nb2ModelDev<double>& M, int j) { while (M.parent[j] >= 0) j = M.parent[j]; return j; }

__global__ void __launch_bounds__(128)
k_ik_forward(const __grid_constant__ Nb2ModelDev<double> M, int B, int nent, int pos_dim, int vel_dim, const IkEntryDev* __restrict__ ent,
             const float* __restrict__ state, float* __restrict__ pos, float* __restrict__ vel) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * nent) return;
  const int w = t / nent, e = t - w * nent;
  const IkEntryDev E = ent[e];
  const float* q = state + (size_t)w * 2 * M.ndof; const float* qd = q + M.ndof;
  float* po = pos ? pos + (size_t)w * pos_dim + E.pos_off : nullptr;
  float* vo = vel ? vel + (size_t)w * vel_dim + E.vel_off : nullptr;
  if (E.type == NB2_IK_COM) {  // Skeleton::getCOM / getCOMLinearVelocity of the tree rooted at E.body
    double mt = 0; V3<double> c = nb2::zero3<double>(), cv = nb2::zero3<double>();
    for (int i = 0; i < M.nb; i++) {
      if (ik_root(M, i) != E.body) continue;
      Xf<double> W; V6<double> V; ik_fk(M, i, q, qd, &W, &V);
      const double m = M.inertia[i][0];
      const V3<double> h = nb2::mul(W.R_, nb2::mk3<double>(M.inertia[i][1], M.inertia[i][2], M.inertia[i][3]));  // m * (com - origin), world axes
      mt += m; c = c + W.p * m + h;
      cv = cv + nb2::mul(W.R_, V.l) * m + nb2::cross(nb2::mul(W.R_, V.a), h);
    }
    const double inv = mt > 0 ? 1.0 / mt : 0.0;
    if (po) { po[0] = (float)(c.x * inv); po[1] = (float)(c.y * inv); po[2] = (float)(c.z * inv); }
    if (vo) { vo[0] = (float)(cv.x * inv); vo[1] = (float)(cv.y * inv); vo[2] = (float)(cv.z * inv); }
    return;
  }
  Xf<double> Toff = nb2::ldXf<double, 1>(E.T), We; V3<double> om = nb2::zero3<double>(), vl = nb2::zero3<double>();
  if (E.body >= 0) {
    Xf<double> W; V6<double> V; ik_fk(M, E.body, q, qd, &W, &V);
    We = nb2::gxf_mul(W, Toff);
    om = nb2::mul(W.R_, V.a);
    vl = nb2::mul(W.R_, V.l) + nb2::cross(om, We.p - W.p);
  } else We = Toff;
  int k = 0;
  if (po) {
    if (E.type != NB2_IK_LINEAR) { const V3<double> phi = nb2::logmap(We.R_); po[0] = (float)phi.x; po[1] = (float)phi.y; po[2] = (float)phi.z; k = 3; }
    if (E.type != NB2_IK_ANGULAR) { po[k] = (float)We.p.x; po[k + 1] = (float)We.p.y; po[k + 2] = (float)We.p.z; }
  }
  if (vo) {
    k = 0;
    if (E.type != NB2_IK_LINEAR) { vo[0] = (float)om.x; vo[1] = (float)om.y; vo[2] = (float)om.z; k = 3; }
    if (E.type != NB2_IK_ANGULAR) { vo[k] = (float)vl.x; vo[k + 1] = (float)vl.y; vo[k + 2] = (float)vl.z; }
  }
}

// grad_state[w] = J_pos^T grad_pos[w] (into the position half) and J_vel^T grad_vel[w] (into the velocity half): exactly what
// MapToPosLayer.backward / MapToVelLayer.backward return (mapping.py:36-47, 84-95: positions feed only d/dq, velocities only d/dqdot).
__global__ void __launch_bounds__(128)
k_ik_backward(const __grid_constant__ Nb2ModelDev<double> M, int B, int nent, int pos_dim, int vel_dim, const IkEntryDev* __restrict__ ent,
              const float* __restrict__ state, const float* __restrict__ gpos, const float* __restrict__ gvel, float* __restrict__ gstate) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= B) return;
  const float* q = state + (size_t)w * 2 * M.ndof; const float* qd = q + M.ndof;
  float* g = gstate + (size_t)w * 2 * M.ndof;
  for (int d = 0; d < 2 * M.ndof; d++) g[d] = 0.f;
  const V3<double> z3 = nb2::zero3<double>();
  for (int e = 0; e < nent; e++) {
    const IkEntryDev E = ent[e];
    const float* gp = gpos ? gpos + (size_t)w * pos_dim + E.pos_off : nullptr;
    const float* gv = gvel ? gvel + (size_t)w * vel_dim + E.vel_off : nullptr;
    if (E.type == NB2_IK_COM) {
      double mt = 0;
      for (int i = 0; i < M.nb; i++) if (ik_root(M, i) == E.body) mt += M.inertia[i][0];
      const double inv = mt > 0 ? 1.0 / mt : 0.0;
      const V3<double> fp = gp ? nb2::mk3<double>(gp[0], gp[1], gp[2]) * inv : z3, fv = gv ? nb2::mk3<double>(gv[0], gv[1], gv[2]) * inv : z3;
      for (int i = 0; i < M.nb; i++) {
        if (ik_root(M, i) != E.body) continue;
        Xf<double> W; V6<double> V; ik_fk(M, i, q, qd, &W, &V);
        const double m = M.inertia[i][0];
        const V3<double> h = nb2::mul(W.R_, nb2::mk3<double>(M.inertia[i][1], M.inertia[i][2], M.inertia[i][3]));
        // d(m p + R h) = m dp + dtheta x h  ->  force m f at the origin, torque h x f; about the world origin: + p x (m f)
        ik_fk_vjp(M, i, q, nb2::cross(h, fp) + nb2::cross(W.p, fp * m), fp * m, nb2::cross(h, fv) + nb2::cross(W.p, fv * m), fv * m, g);
      }
      continue;
    }
    if (E.body < 0) continue;  // static body: constants
    Xf<double> W; V6<double> V; ik_fk(M, E.body, q, qd, &W, &V);
    const Xf<double> We = nb2::gxf_mul(W, nb2::ldXf<double, 1>(E.T));
    V3<double> np = z3, fp = z3, nv = z3, fv = z3;
    int k = 0;
    if (E.type != NB2_IK_LINEAR) {
      // log(exp(dtheta) R) = phi + Jl^-1(phi) dtheta, and Jl^-T = Jr^-1
      if (gp) np = nb2::mul(nb2::so3_Jr_inv(nb2::logmap(We.R_)), nb2::mk3<double>(gp[0], gp[1], gp[2]));
      if (gv) nv = nb2::mk3<double>(gv[0], gv[1], gv[2]);
      k = 3;
    }
    if (E.type != NB2_IK_ANGULAR) {
      if (gp) fp = nb2::mk3<double>(gp[k], gp[k + 1], gp[k + 2]);
      if (gv) fv = nb2::mk3<double>(gv[k], gv[k + 1], gv[k + 2]);
    }
    ik_fk_vjp(M, E.body, q, np + nb2::cross(We.p, fp), fp, nv + nb2::cross(We.p, fv), fv, g);
  }
}

// ---- pointer-style forward dynamics (row a5: SimpleFeatherstone::forwardDynamics(pos, vel, force, accel), dynamics/SimpleFeatherstone.hpp:61-65):
// fp64 in, fp64 out, one thread per world with its scratch in global memory — a convenience / parity entry, not a hot path.
__global__ void __launch_bounds__(64)
k_forward_dynamics(const __grid_constant__ Nb2ModelDev<double> M, int B, int words, const double* __restrict__ pos, const double* __restrict__ vel,
                   const double* __restrict__ force, double* __restrict__ accel, double* __restrict__ scratch) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= B) return;
  double* scr = scratch + (size_t)w * words;
  const nb2::FwdLayout L = nb2::fwd_layout(M.nb, M.ndof, M.nslots, M.nfree);
  const int n = M.ndof;
  for (int d = 0; d < n; d++) { scr[L.oQ + d] = pos[(size_t)w * n + d]; scr[L.oV + d] = vel[(size_t)w * n + d]; }
  for (int a = 0; a < M.na; a++) scr[L.oAct + a] = force[(size_t)w * n + M.action_map[a]];
  for (int sg = 1; sg < NB2_FWD_STAGES - 1; sg++)
    for (int lane = 0; lane < M.lanes; lane++) nb2::world_forward_stage<double, 1>(M, scr, nullptr, 1, false, lane, sg);
  // pass 3 left v + dt * qdd in the velocity slots
  for (int d = 0; d < n; d++) accel[(size_t)w * n + d] = (scr[L.oV + d] - vel[(size_t)w * n + d]) / M.dt;
}

// ---- batched boxed-LCP entry (the reference's pointer-style lower boundary: BoxedLcpSolver::solve, constraint/BoxedLcpSolver.hpp:125-135,
// and BoxedLcpConstraintSolver::solveLcp): one warp per problem, the same device code the contact stage runs.
//   mode 0: Dantzig only (DantzigBoxedLcpSolver::solve -> dSolveLCP);  mode 1: the whole solve chain with classification
__global__ void __launch_bounds__(32)
k_lcp_batch(nb2::cw::Dims d, int B, int mcap, double cfm, int mode, int early_termination, const int* __restrict__ ms, const double* __restrict__ A,
            const double* __restrict__ b, const double* __restrict__ lo, const double* __restrict__ hi, const int* __restrict__ findex,
            const double* __restrict__ x0, double* __restrict__ x, int* __restrict__ labels, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char nb2_smem[];
  const int w = blockIdx.x, lane = threadIdx.x & 31;
  if (w >= B) return;
  nb2::cw::Ws* wsm = warp_workspace(nb2_smem, d, lane);
  const nb2::cw::Ws ws = *wsm;
  const int m = ms[w], ld = m | 1;
  const size_t ov = (size_t)w * mcap;
  for (int e = lane; e < m * m; e += 32) { const int r = e / m, c = e - r * m; ws.A[(size_t)r * ld + c] = A[((size_t)w * mcap + r) * mcap + c]; }
  for (int i = lane; i < m; i += 32) { ws.b[i] = b[ov + i]; ws.lo[i] = lo[ov + i]; ws.hi[i] = hi[ov + i]; ws.findex[i] = findex[ov + i]; }
  __syncwarp();
  int st;
  if (mode == 0) {
    nb2::cw::DzWork W;
    for (int e = lane; e < m * ld; e += 32) ws.M1[e] = ws.A[e];
    for (int i = lane; i < m; i += 32) { ws.v1[i] = ws.b[i]; ws.v2[i] = ws.lo[i]; ws.v3[i] = ws.hi[i]; ws.i1[i] = ws.findex[i]; }
    __syncwarp();
    W.A = ws.M1; W.ld = ld; W.x = ws.x; W.b = ws.v1; W.w = ws.v5; W.lo = ws.v2; W.hi = ws.v3; W.L = ws.M2; W.d = ws.v6; W.delta_x = ws.v7; W.delta_w = ws.v8;
    W.Dell = ws.v9; W.ell = ws.v10; W.tmp = ws.v11; W.findex = ws.i1; W.p = ws.clampIdx; W.C = ws.ubIdx; W.state = ws.i4;
    st = nb2::cw::dantzig_solve(W, m, early_termination != 0);
  } else {
    st = nb2::cw::lcp_chain(m, ws, *wsm, cfm, x0 ? x0 + ov : nullptr);
  }
  __syncwarp();
  for (int i = lane; i < m; i += 32) { x[ov + i] = ws.x[i]; if (labels) labels[ov + i] = (mode == 1) ? ws.mapping[i] : 0; }
  if (lane == 0) status[w] = st;
}

constexpr int kMaxSmem = 227 * 1024;

}  // namespace

// Calls f with the lane count as a compile-time std::integral_constant (the step kernels are instantiated for 1, 2, 4 and 8 lanes).
template <class F> static int with_lanes(int lanes, F&& f) {
  switch (lanes) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 4: return f(std::integral_constant<int, 4>());
    case 8: return f(std::integral_constant<int, 8>());
  }
  g_err = "bad lane count"; return NB2_ERR_INVALID;
}
// Calls f with a value of the real type of `precision`: NB2_FP64 runs the fp64 kernels, any other value the fp32 ones.
template <class F> static int with_precision(int precision, F&& f) { return precision == NB2_FP64 ? f(double()) : f(float()); }
// The dynamic shared-memory limit of a kernel is a per-device attribute (a model may be used from several GPUs of one process): raise it
// to kMaxSmem once per kernel and device.
template <auto Kern> static int allow_max_smem() {
  static std::atomic<bool> done[64];
  int dev = 0; NB2_CUDA(cudaGetDevice(&dev));
  if (!done[dev & 63].load(std::memory_order_acquire)) {
    NB2_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    done[dev & 63].store(true, std::memory_order_release);
  }
  return NB2_OK;
}

// one sweep schedule of the model (same bodies, different lane count / slot assignment)
struct LaunchShape { int warps_per_block = 0; int resident_warps = 0; };  // filled lazily from the occupancy API
struct nb2_variant {
  Nb2ModelDev<float> mf;
  Nb2ModelDev<double> md;
  int fwd_words, bwd_words;
  int depth;                 // bodies on the sequential path of one sweep: |trunk| + longest lane
  LaunchShape shape[2][2];   // [forward/backward][fp32/fp64]
};

struct nb2_model {
  Nb2ModelDev<float> mf;   // the schedule given to nb2_model_create (also what the contact kernels use)
  Nb2ModelDev<double> md;
  Nb2ContactDev contact;
  bool has_contacts = false;
  bool contact_restitution = false;  // any shape-carrying body with a restitution coefficient > 0
  int contact_mc = 0;      // contact capacity of the shared-memory workspace of the fused contact kernels (rows: 3x)
  int contact_variant = 0; // schedule the fused contact kernels sweep the tree with
  int saved_words;
  int sm_count;
  std::vector<nb2_variant> variants;  // [0] = the create-time schedule
  int forced_lanes = 0;               // 0: pick per launch from the batch size
  // device buffers owned by the *_host entry points
  float *d_state = nullptr, *d_action = nullptr, *d_next = nullptr, *d_gnext = nullptr,
        *d_gstate = nullptr, *d_gaction = nullptr;
  void* d_saved = nullptr;  // sized for fp64 words
  int host_cap = 0;
  int host_B = 0;  // batch of the last forward_host kept for backward
  // contact path of the *_host entry points: solver cache (flows from call to call), per-step outputs, record, workspace
  void* hc_ws = nullptr; double *hc_x = nullptr, *hc_rec = nullptr; int32_t *hc_m = nullptr, *hc_labels = nullptr, *hc_status = nullptr, *hc_nc = nullptr, *hc_sticky = nullptr;
  int hc_cap = 0;
  cudaStream_t host_streams[4] = {nullptr, nullptr, nullptr, nullptr};
  std::mutex mu;
};

template <class R> static const Nb2ModelDev<R>& model_of(const nb2_variant& v);
template <> const Nb2ModelDev<float>& model_of<float>(const nb2_variant& v) { return v.mf; }
template <> const Nb2ModelDev<double>& model_of<double>(const nb2_variant& v) { return v.md; }

static void init_variant(nb2_variant& v) {
  v.fwd_words = nb2::fwd_layout(v.mf.nb, v.mf.ndof, v.mf.nslots, v.mf.nfree).total;
  v.bwd_words = nb2::bwd_layout(v.mf.nb, v.mf.ndof, v.mf.nslots, v.mf.nfree).total;
  int trunk = 0, longest = 0;
  for (int r = 0; r < v.mf.trunk_n; r++) trunk += v.mf.trunk_hi[r] - v.mf.trunk_lo[r];
  for (int l = 0; l < v.mf.lanes; l++) {
    int len = 0;
    for (int r = 0; r < v.mf.limb_n[l]; r++) len += v.mf.limb_hi[l][r] - v.mf.limb_lo[l][r];
    if (len > longest) longest = len;
  }
  v.depth = trunk + longest;
}

// ---- launch shape.  The kernels are latency bound (one dependent chain per world), so a launch costs about
//   (sequential depth of the schedule) x (number of waves the batch needs at that schedule's occupancy).
// Occupancy is limited by the per-warp scratch in shared memory; blocks of 1, 2 or 4 warps are tried and the shape
// that keeps most warps resident wins.  Small batches use 1-warp blocks so that they spread over all SMs.
template <class Kern>
static LaunchShape occupancy_shape(Kern kern, size_t bytes_per_warp, size_t bytes_per_block) {
  LaunchShape best;
  for (int w = 1; w <= 4; w *= 2) {
    const size_t smem = bytes_per_warp * w + bytes_per_block;
    if (smem > (size_t)kMaxSmem) break;
    int blocks = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, w * 32, smem) != cudaSuccess) { cudaGetLastError(); continue; }
    if (blocks * w > best.resident_warps) { best.resident_warps = blocks * w; best.warps_per_block = w; }
  }
  return best;
}

// warps per block for one launch: a batch that fits in one wave is spread so that every SM gets about the same number of
// warps in as few blocks as possible (measured: 4 warps in one block beat 4 one-warp blocks on the same SM); beyond one
// wave the occupancy-optimal shape is used.
static int block_warps(int total_warps, int sm_count, const LaunchShape& sh, size_t per_warp) {
  if ((long long)total_warps > (long long)sm_count * sh.resident_warps) return sh.warps_per_block;
  int w = 1;
  while (w < 4 && total_warps > sm_count * w && (size_t)(2 * w) * per_warp <= (size_t)kMaxSmem) w *= 2;
  return w;
}

template <class R, int K>
static int prepare_k(nb2_variant& v, int dir) {  // dir 0 forward, 1 backward
  constexpr int ST = CoopShape<K>::ST;
  LaunchShape& sh = v.shape[dir][sizeof(R) == 8];
  // the occupancy query sizes a warp with its scratch AND its input-staging buffer, in both directions
  const size_t scratch_and_staging = (size_t)(dir ? v.bwd_words : v.fwd_words) * ST * sizeof(R) +
                                     (dir ? staging_bytes<K>(4 * v.mf.ndof + v.mf.na) : staging_bytes<K>(2 * v.mf.ndof + v.mf.na));
  const size_t per_block = (size_t)body_table_words<K>(v.mf.nb) * sizeof(R) + 16;
  if (scratch_and_staging + per_block > (size_t)kMaxSmem) {
    g_err = "model needs " + std::to_string(scratch_and_staging) + " B of shared memory per warp (> 227 KB)"; return NB2_ERR_UNSUPPORTED;
  }
  int rc;
  if (dir == 0) {  // the per-world-inertia variant launches with the shape of the shared-table kernel
    if ((rc = allow_max_smem<k_step_fwd<R, K, false>>()) || (rc = allow_max_smem<k_step_fwd<R, K, true>>())) return rc;
    if (!sh.warps_per_block) sh = occupancy_shape(k_step_fwd<R, K, false>, scratch_and_staging, per_block);
  } else {
    if ((rc = allow_max_smem<k_step_bwd<R, K, false>>()) || (rc = allow_max_smem<k_step_bwd<R, K, true>>())) return rc;
    if (!sh.warps_per_block) sh = occupancy_shape(k_step_bwd<R, K, false>, scratch_and_staging, per_block);
  }
  if (!sh.warps_per_block) { g_err = "no launch shape fits this model"; return NB2_ERR_UNSUPPORTED; }
  return NB2_OK;
}
template <class R>
static int prepare_variant(nb2_variant& v, int dir) {
  return with_lanes(v.mf.lanes, [&](auto k) { return prepare_k<R, decltype(k)::value>(v, dir); });
}

template <class R>
static int pick_variant(nb2_model* m, int B, int dir, nb2_variant** out) {
  nb2_variant* best = nullptr;
  double best_cost = 0;
  for (auto& v : m->variants) {
    if (m->forced_lanes && v.mf.lanes != m->forced_lanes) continue;
    int rc = prepare_variant<R>(v, dir);
    if (rc) { if (m->variants.size() == 1 || m->forced_lanes) return rc; continue; }
    const LaunchShape& sh = v.shape[dir][sizeof(R) == 8];
    const double warps = ((double)B * v.mf.lanes + 31) / 32;
    double waves = warps / ((double)m->sm_count * sh.resident_warps);
    if (waves < 1) waves = 1;
    const double cost = (v.depth + 3) * waves;   // +3: per-sweep fixed part (loads, stores, barriers)
    if (!best || cost < best_cost - 1e-9) { best = &v; best_cost = cost; }
  }
  if (!best) { g_err = "no usable schedule"; return NB2_ERR_UNSUPPORTED; }
  *out = best;
  return NB2_OK;
}

template <class R, int K>
static int launch_fwd_k(const nb2_variant& v, int sm_count, int Btot, int w0, int B, const float* state, const float* action,
                        float* next, R* saved, cudaStream_t st, float* state_copy, float* action_copy, const double* wi) {
  constexpr int WPW = CoopShape<K>::WPW, ST = CoopShape<K>::ST;
  const LaunchShape& sh = v.shape[0][sizeof(R) == 8];
  const size_t per_warp = (size_t)v.fwd_words * ST * sizeof(R) + staging_bytes<K>(2 * v.mf.ndof + v.mf.na);  // scratch + input staging
  const int total_warps = (B + WPW - 1) / WPW;
  const int warps = block_warps(total_warps, sm_count, sh, per_warp);
  const int blocks = (total_warps + warps - 1) / warps;
  const size_t smem = per_warp * warps + (size_t)body_table_words<K>(v.mf.nb) * sizeof(R) + 16;
  if (wi) k_step_fwd<R, K, true><<<blocks, warps * 32, smem, st>>>(model_of<R>(v), Btot, w0, B, state, action, next, saved, v.fwd_words, state_copy, action_copy, wi);
  else k_step_fwd<R, K, false><<<blocks, warps * 32, smem, st>>>(model_of<R>(v), Btot, w0, B, state, action, next, saved, v.fwd_words, state_copy, action_copy, nullptr);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
template <class R>
static int launch_fwd(nb2_model* m, int B, const float* state, const float* action, float* next, R* saved, cudaStream_t st,
                      int Btot = -1, int w0 = 0, float* state_copy = nullptr, float* action_copy = nullptr, const double* wi = nullptr) {
  if (Btot < 0) Btot = B;
  nb2_variant* pv = nullptr;
  int rc = pick_variant<R>(m, B, 0, &pv);
  if (rc) return rc;
  return with_lanes(pv->mf.lanes, [&](auto k) {
    return launch_fwd_k<R, decltype(k)::value>(*pv, m->sm_count, Btot, w0, B, state, action, next, saved, st, state_copy, action_copy, wi);
  });
}
static bool no_stage_saved() {
  static const bool off = [] { const char* e = getenv("NB2_NO_STAGE_SAVED"); return e && atoi(e); }();
  return off;
}
template <class R, int K>
static int launch_bwd_k(const nb2_variant& v, int sm_count, int Btot, int w0, int B, const float* state, const float* action,
                        const R* saved, const float* gnext, float* gstate, float* gaction, float* ginertia, cudaStream_t st, int accumulate,
                        const double* wi, double* gIa) {
  constexpr int WPW = CoopShape<K>::WPW, ST = CoopShape<K>::ST;
  const LaunchShape& sh = v.shape[1][sizeof(R) == 8];
  // the warps per block are sized with the scratch only, while prepare_k's occupancy query (scratch_and_staging) also counts the input staging
  const size_t scratch_per_warp = (size_t)v.bwd_words * ST * sizeof(R);
  const int total_warps = (B + WPW - 1) / WPW;
  const int warps = block_warps(total_warps, sm_count, sh, scratch_per_warp);
  const int blocks = (total_warps + warps - 1) / warps;
  const size_t tab = (size_t)body_table_words<K>(v.mf.nb) * sizeof(R);
  // stage the saved stream in shared memory when the whole batch is resident at once anyway (see the kernel)
  const size_t stage_per_warp = (size_t)nb2_saved_words(v.mf.nb, v.mf.ndof, v.mf.nfree) * WPW * sizeof(R);
  const bool aligned = (((size_t)Btot * sizeof(R)) % 16 == 0) && (((size_t)w0 * sizeof(R)) % 16 == 0) && ((reinterpret_cast<size_t>(saved) & 15) == 0) &&
                       ((WPW * sizeof(R)) % 16 == 0);
  const size_t in_per_warp = staging_bytes<K>(4 * v.mf.ndof + v.mf.na);  // bulk-copy staging of dL/dx', x, u rows
  const size_t smem_staged = (scratch_per_warp + stage_per_warp) * warps + tab + 16;
  const int blocks_per_sm = (blocks + sm_count - 1) / sm_count;
  const bool stage = aligned && (smem_staged + in_per_warp * warps) * blocks_per_sm + 1024 * blocks_per_sm <= (size_t)kMaxSmem && !no_stage_saved();
  const size_t base = ((stage ? smem_staged : scratch_per_warp * warps + tab) + 15) & ~(size_t)15;
  const bool in_stage = base + in_per_warp * warps <= (size_t)kMaxSmem;
  const size_t smem = in_stage ? base + in_per_warp * warps : base;
  if (wi || gIa) k_step_bwd<R, K, true><<<blocks, warps * 32, smem, st>>>(model_of<R>(v), Btot, w0, B, state, action, saved, gnext, gstate, gaction, ginertia,
                                                                   v.bwd_words, stage ? 1 : 0, accumulate, in_stage ? (unsigned)base : 0u, wi, gIa);
  else k_step_bwd<R, K, false><<<blocks, warps * 32, smem, st>>>(model_of<R>(v), Btot, w0, B, state, action, saved, gnext, gstate, gaction, ginertia,
                                                                 v.bwd_words, stage ? 1 : 0, accumulate, in_stage ? (unsigned)base : 0u, nullptr, nullptr);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
template <class R>
static int launch_bwd(nb2_model* m, int B, const float* state, const float* action,
                      const R* saved, const float* gnext, float* gstate, float* gaction, float* ginertia, cudaStream_t st,
                      int Btot = -1, int w0 = 0, int accumulate = 0, const double* wi = nullptr, double* gIa = nullptr) {
  if (Btot < 0) Btot = B;
  nb2_variant* pv = nullptr;
  int rc = pick_variant<R>(m, B, 1, &pv);
  if (rc) return rc;
  return with_lanes(pv->mf.lanes, [&](auto k) {
    return launch_bwd_k<R, decltype(k)::value>(*pv, m->sm_count, Btot, w0, B, state, action, saved, gnext, gstate, gaction, ginertia, st, accumulate, wi, gIa);
  });
}

// The host entry points take host buffers.  When every buffer of a call is page-locked memory visible to the device
// (cudaHostAlloc / cudaHostRegister, e.g. torch pin_memory()), the kernels read and write it DIRECTLY: the group load /
// store of every warp is a coalesced, deeply pipelined stream over PCIe, so the transfer overlaps the sweeps warp by warp
// and no copy is ever queued (the forward kernel also leaves a device copy of state / action for the backward pass).
// Pageable buffers go through staged cudaMemcpyAsync on up to NB2_HOST_CHUNKS streams (default 1).
static int host_chunks(int B) {
  static const int forced = [] { const char* e = getenv("NB2_HOST_CHUNKS"); return e ? atoi(e) : 1; }();
  return (forced >= 1 && forced <= 4 && forced <= B) ? forced : 1;
}
static bool zero_copy_enabled() {
  static const bool on = [] { const char* e = getenv("NB2_NO_ZEROCOPY"); return !(e && atoi(e)); }();
  return on;
}
// device-side alias of a page-locked host buffer, or nullptr when the buffer is pageable
template <class T> static T* mapped_alias(const T* host) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, host) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (a.type != cudaMemoryTypeHost || !a.devicePointer) return nullptr;
  return (T*)a.devicePointer;
}

// ---- fused contact kernels: launch plumbing
static nb2::cw::Dims cdims(const nb2_model* m, int MC, int bwd, int mode = NB2_WS_FULL) {
  return nb2::cw::make_dims(m->md.nb, m->md.ndof, m->md.nfree, MC, 3 * MC, m->contact.ncb, m->contact.max_chain_dofs, bwd, mode);
}
// worlds (warps) per block of a lockstep kernel: as many as shared memory allows (one block per SM), fewer for batches that would
// otherwise leave SMs idle
static int wpb_cap(int which) {  // dev knob: NB2_WPB="build,solve,apply,bwd" caps the worlds per block of the lockstep kernels (0 = default)
  static int caps[4] = {0, 0, 0, 0};
  static const bool init = [] { const char* e = getenv("NB2_WPB"); if (e) sscanf(e, "%d,%d,%d,%d", &caps[0], &caps[1], &caps[2], &caps[3]); return true; }();
  (void)init;
  return caps[which];
}
static int pick_wpb(int B, int sm_count, size_t smem_per_warp, int max_warps, int which = -1) {
  int w = (int)((size_t)kMaxSmem / (smem_per_warp ? smem_per_warp : 1));
  if (which >= 0 && wpb_cap(which) > 0 && wpb_cap(which) < max_warps) max_warps = wpb_cap(which);
  if (w > max_warps) w = max_warps;
  const int spread = (B + sm_count - 1) / sm_count;
  if (w > spread) w = spread;
  return w < 1 ? 1 : w;
}
static bool contact_fused() {
  static const bool on = [] { const char* e = getenv("NB2_CONTACT_FUSED"); return e && atoi(e); }();
  return on;
}
static int pool_slots(int B) { int s = B / 16; if (s < 32) s = 32; if (s > 4096) s = 4096; return s; }
static size_t pool_stride(const nb2_model* m) { return (nb2::cw::ws_doubles(cdims(m, NB2_MAX_CONTACTS, 1)) + 1) & ~(size_t)1; }
static CStepArgs cstep_args(const nb2_model* m, const nb2_variant& v, int B, void* workspace, int bwd) {
  CStepArgs P;
  P.B = B;
  P.fwd_words = v.fwd_words;
  P.bwd_words = nb2::bwd_layout(v.md.nb, v.md.ndof, v.md.nslots, v.md.nfree, 42).total;
  P.saved_words = m->saved_words;
  P.ds = cdims(m, m->contact_mc, bwd);
  P.db = cdims(m, NB2_MAX_CONTACTS, bwd);
  P.ws_small_doubles = nb2::cw::ws_doubles(P.ds);
  P.pool.counter = (int*)workspace;
  P.pool.base = (double*)((char*)workspace + 64);
  P.pool.stride = pool_stride(m);
  P.pool.nslots = pool_slots(B);
  P.rec_doubles = nb2::cw::record_doubles(m->md.ndof);
  P.exch = P.pool.base + (size_t)P.pool.nslots * P.pool.stride;
  P.exch_stride = nb2::cw::xlayout(m->md.ndof).total;
  P.ds_solve = cdims(m, m->contact_mc, 0, NB2_WS_SOLVE); P.db_solve = cdims(m, NB2_MAX_CONTACTS, 0, NB2_WS_SOLVE);
  P.ds_apply = cdims(m, m->contact_mc, 0, NB2_WS_APPLY); P.db_apply = cdims(m, NB2_MAX_CONTACTS, 0, NB2_WS_APPLY);
  P.pool_solve = P.pool; P.pool_solve.counter = (int*)workspace + 1;  // the kernels run one after the other: same slots, own counter
  P.pool_apply = P.pool; P.pool_apply.counter = (int*)workspace + 2;
  P.pool_solve_b = P.pool; P.pool_solve_b.counter = (int*)workspace + 3;
  P.todo_count = (int*)workspace + 4;
  P.todo = (int*)(P.exch + (size_t)B * P.exch_stride);  // list of the worlds the first solve kernel hands to the second
  return P;
}
template <auto Kern> static int cstep_smem_attr(size_t smem) {
  if (int rc = allow_max_smem<Kern>()) return rc;
  if (smem > (size_t)kMaxSmem) { g_err = "the fused contact kernel needs " + std::to_string(smem) + " B of shared memory per world (> 227 KB)"; return NB2_ERR_UNSUPPORTED; }
  return NB2_OK;
}

extern "C" {

const char* nb2_last_error(void) { return g_err.c_str(); }
const char* nb2_version(void) { return "nb2 0.2 (sm_90a; cooperative-lane ABA + adjoint, warp-per-world contact / boxed-LCP stage)"; }
long long nb2_launch_count(void) { return g_launches.load(); }

int nb2_model_create(const nb2_model_desc* desc, nb2_model** out) {
  if (!desc || !out) { g_err = "null argument"; return NB2_ERR_INVALID; }
  nb2_model* m = new nb2_model();
  std::string err;
  if (!nb2_fill_model(*desc, m->mf, err) || !nb2_fill_model(*desc, m->md, err)) {
    g_err = err; delete m;
    return (desc->nb > NB2_MAX_BODIES || desc->ndof > NB2_MAX_DOFS) ? NB2_ERR_UNSUPPORTED : NB2_ERR_INVALID;
  }
  if ((desc->nshapes > 0 && desc->npairs > 0) || desc->nlimits > 0) {
    if (!nb2_fill_contact(*desc, m->contact, err)) { g_err = err; delete m; return NB2_ERR_UNSUPPORTED; }
    m->has_contacts = true;
    for (int p = 0; p < desc->npairs; p++)  // a pair bounces when the product of its shapes' coefficients exceeds 1e-3 (ContactConstraint.cpp:112-123)
      if (m->contact.shape_rest[desc->pair_a[p]] * m->contact.shape_rest[desc->pair_b[p]] > 1e-3) m->contact_restitution = true;
    // contacts the shared-memory workspace is sized for: a box-box pair yields up to 4 in the common face-face case (8 at most), every
    // other supported pair at most one; worlds that exceed it fall back to a global-memory workspace (nb2_cw.cuh BigPool)
    int mc = 0;
    for (int p = 0; p < desc->npairs; p++) mc += (desc->shape_type[desc->pair_a[p]] == 0 && desc->shape_type[desc->pair_b[p]] == 0) ? 4 : 1;
    mc += desc->nlimits;  // an active joint limit takes the slot of one contact (one row)
    if (const char* e = getenv("NB2_CONTACT_MC")) mc = atoi(e);
    m->contact_mc = mc < 2 ? 2 : (mc > NB2_MAX_CONTACTS ? NB2_MAX_CONTACTS : mc);
  }
  {
    nb2_variant v;
    v.mf = m->mf; v.md = m->md;
    init_variant(v);
    m->variants.push_back(v);
  }
  m->saved_words = nb2_saved_words(m->mf.nb, m->mf.ndof, m->mf.nfree);
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    g_err = "no CUDA device available: nimblephysics_b200 has no CPU fallback";
    delete m;
    return NB2_ERR_CUDA;
  }
  m->sm_count = prop.multiProcessorCount;
  *out = m;
  return NB2_OK;
}

int nb2_model_add_schedule(nb2_model* m, const nb2_model_desc* desc) {
  if (!m || !desc) { g_err = "null argument"; return NB2_ERR_INVALID; }
  nb2_variant v;
  std::string err;
  if (!nb2_fill_model(*desc, v.mf, err) || !nb2_fill_model(*desc, v.md, err)) { g_err = err; return NB2_ERR_INVALID; }
  // same bodies, same numbering: only the sweep schedule (lanes, slots, handoff flags) may differ
  bool same = v.md.nb == m->md.nb && v.md.ndof == m->md.ndof && v.md.na == m->md.na && v.md.nfree == m->md.nfree && v.md.dt == m->md.dt;
  for (int i = 0; same && i < m->md.nb; i++) {
    same = v.md.parent[i] == m->md.parent[i] && v.md.jtype[i] == m->md.jtype[i] && v.md.dof_off[i] == m->md.dof_off[i];
    for (int k = 0; same && k < 12; k++) same = v.md.Xtree[i][k] == m->md.Xtree[i][k];
    for (int k = 0; same && k < 10; k++) same = v.md.inertia[i][k] == m->md.inertia[i][k];
  }
  if (!same) { g_err = "nb2_model_add_schedule: the descriptor describes a different model"; return NB2_ERR_INVALID; }
  for (const auto& o : m->variants) if (o.mf.lanes == v.mf.lanes) { g_err = "nb2_model_add_schedule: a schedule with this lane count exists"; return NB2_ERR_INVALID; }
  init_variant(v);
  std::lock_guard<std::mutex> lk(m->mu);
  m->variants.push_back(v);
  // the fused contact kernels have a whole warp per world: they sweep the tree with the shallowest schedule registered
  for (size_t k = 0; k < m->variants.size(); k++) if (m->variants[k].depth < m->variants[m->contact_variant].depth) m->contact_variant = (int)k;
  return NB2_OK;
}
int nb2_model_set_inertia(nb2_model* m, const double* inertia) {
  if (!m || !inertia) { g_err = "null argument"; return NB2_ERR_INVALID; }
  for (int i = 0; i < m->md.nb; i++)
    if (!(inertia[10 * i] > 0)) { g_err = "nb2_model_set_inertia: body " + std::to_string(i) + " has non-positive mass"; return NB2_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(m->mu);
  auto put = [&](Nb2ModelDev<float>& mf, Nb2ModelDev<double>& md) {
    for (int i = 0; i < md.nb; i++)
      for (int k = 0; k < 10; k++) { md.inertia[i][k] = inertia[10 * i + k]; mf.inertia[i][k] = (float)inertia[10 * i + k]; }
  };
  put(m->mf, m->md);
  for (auto& v : m->variants) put(v.mf, v.md);
  return NB2_OK;
}
int nb2_model_set_lanes(nb2_model* m, int lanes) {
  if (!m) { g_err = "null argument"; return NB2_ERR_INVALID; }
  if (lanes != 0) {
    bool found = false;
    for (const auto& o : m->variants) found = found || o.mf.lanes == lanes;
    if (!found) { g_err = "nb2_model_set_lanes: no schedule with " + std::to_string(lanes) + " lanes was added"; return NB2_ERR_INVALID; }
  }
  m->forced_lanes = lanes;
  return NB2_OK;
}
int nb2_model_lanes_for(nb2_model* m, int B, int backward, int precision) {
  if (!m || B <= 0) return -1;
  nb2_variant* pv = nullptr;
  const int rc = with_precision(precision, [&](auto r) { return pick_variant<decltype(r)>(m, B, backward ? 1 : 0, &pv); });
  return rc ? -1 : pv->mf.lanes;
}

void nb2_model_destroy(nb2_model* m) {
  if (!m) return;
  cudaFree(m->d_state); cudaFree(m->d_action); cudaFree(m->d_next); cudaFree(m->d_saved);
  cudaFree(m->d_gnext); cudaFree(m->d_gstate); cudaFree(m->d_gaction);
  cudaFree(m->hc_ws); cudaFree(m->hc_x); cudaFree(m->hc_rec); cudaFree(m->hc_m); cudaFree(m->hc_labels); cudaFree(m->hc_status); cudaFree(m->hc_nc); cudaFree(m->hc_sticky);
  for (auto& hs : m->host_streams) if (hs) cudaStreamDestroy(hs);
  delete m;
}
int nb2_model_has_contacts(const nb2_model* m) { return (m && m->has_contacts) ? 1 : 0; }
size_t nb2_contact_workspace_bytes(const nb2_model* m, int B) {
  if (!m || !m->has_contacts || B <= 0) return 0;
  // [64 B: pool counters] [pool of large workspaces] [exchange records of the three-kernel forward, one per world]
  return 64 + ((size_t)pool_slots(B) * pool_stride(m) + (size_t)B * nb2::cw::xlayout(m->md.ndof).total) * sizeof(double) + (size_t)B * sizeof(int);
}
int nb2_step_forward_contact(const nb2_model* cm, int B, const float* state, const float* action, float* next_state,
                             void* saved_fp64, void* workspace, double* x_lcp, int32_t* m_lcp, int32_t* labels,
                             int32_t* status, int32_t* ncontacts, float* cinfo, double* contact_record, int32_t* status_accum, void* stream) {
  return nb2_step_forward_contact_pw(cm, B, state, action, nullptr, next_state, saved_fp64, workspace, x_lcp, m_lcp, labels, status, ncontacts, cinfo,
                                     contact_record, status_accum, stream);
}
int nb2_step_forward_contact_pw(const nb2_model* cm, int B, const float* state, const float* action, const double* world_inertia, float* next_state,
                                void* saved_fp64, void* workspace, double* x_lcp, int32_t* m_lcp, int32_t* labels,
                                int32_t* status, int32_t* ncontacts, float* cinfo, double* contact_record, int32_t* status_accum, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (m && B == 0) return NB2_OK;  // an empty batch has no buffers to check
  if (!m || B < 0 || !state || !action || !next_state || !workspace || !x_lcp || !m_lcp || !labels || !status || !ncontacts) {
    g_err = "nb2_step_forward_contact: bad argument"; return NB2_ERR_INVALID;
  }
  if (!m->has_contacts) { g_err = "nb2_step_forward_contact: the model has no collision pairs"; return NB2_ERR_INVALID; }
  if (contact_record && !saved_fp64) { g_err = "nb2_step_forward_contact: a contact record without the saved stream cannot be back-propagated"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const nb2_variant& v = m->variants[m->contact_variant];
  const CStepArgs P = cstep_args(m, v, B, workspace, 0);
  const size_t smem = ((((size_t)P.fwd_words + 1) & ~(size_t)1) + NB2_WS_DESC_DOUBLES + P.ws_small_doubles) * sizeof(double);
  int rc = cstep_smem_attr<k_cstep_fwd>(smem);
  if (rc) return rc;
  NB2_CUDA(cudaMemsetAsync(workspace, 0, 64, st));  // pool counters
  if (contact_fused() || !saved_fp64) {
    // one kernel does everything (also the only form that runs without a saved stream: the apply kernel reads the tree data from it)
    k_cstep_fwd<<<B, 32, smem, st>>>(v.md, m->contact, P, state, action, next_state, (double*)saved_fp64, x_lcp, m_lcp, labels, status, ncontacts, cinfo,
                                     contact_record, status_accum, world_inertia);
    g_launches++;
    NB2_CUDA(cudaGetLastError());
    return NB2_OK;
  }
  const size_t smem_s = (NB2_WS_DESC_DOUBLES + nb2::cw::ws_doubles(P.ds_solve)) * sizeof(double);
  const size_t smem_a = (NB2_WS_DESC_DOUBLES + nb2::cw::ws_doubles(P.ds_apply)) * sizeof(double);
  if ((rc = cstep_smem_attr<k_cbuild>(smem)) || (rc = cstep_smem_attr<k_csolve<0>>(smem_s)) || (rc = cstep_smem_attr<k_csolve<1>>(smem_s)) ||
      (rc = cstep_smem_attr<k_capply>(smem_a)))
    return rc;
  const int wpb_b = pick_wpb(B, m->sm_count, smem, NB2_CBUILD_MAXW, 0), wpb_s = pick_wpb(B, m->sm_count, smem_s, NB2_CSOLVE_MAXW, 1),
            wpb_a = pick_wpb(B, m->sm_count, smem_a, NB2_CAPPLY_MAXW, 2);
  k_cbuild<<<(B + wpb_b - 1) / wpb_b, 32 * wpb_b, smem * wpb_b, st>>>(v.md, m->contact, P, state, action, next_state, (double*)saved_fp64, m_lcp, status, ncontacts, cinfo,
                                                                      contact_record, smem, world_inertia);
  k_csolve<0><<<(B + wpb_s - 1) / wpb_s, 32 * wpb_s, smem_s * wpb_s, st>>>(m->contact, P, m->md.ndof, x_lcp, m_lcp, labels, status, contact_record, status_accum, smem_s,
                                                                         P.todo, P.todo_count);
  k_csolve<1><<<(B + wpb_s - 1) / wpb_s, 32 * wpb_s, smem_s * wpb_s, st>>>(m->contact, P, m->md.ndof, x_lcp, m_lcp, labels, status, contact_record, status_accum, smem_s,
                                                                         P.todo, P.todo_count);
  k_capply<<<(B + wpb_a - 1) / wpb_a, 32 * wpb_a, smem_a * wpb_a, st>>>(v.md, m->contact, P, state, next_state, (const double*)saved_fp64, x_lcp, labels, contact_record,
                                                                        smem_a);
  g_launches += 4;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
size_t nb2_contact_record_bytes(const nb2_model* m, int B) {
  if (!m || !m->has_contacts || B <= 0) return 0;
  return nb2::cw::record_doubles(m->mf.ndof) * sizeof(double) * (size_t)B;
}
}  // extern "C"
// accumulate: grad_state += clip(J^T grad_next_state) instead of = (rollouts: the loss gradient of x_t is already in the buffer)
static int cbwd_launch(nb2_model* m, int B, const float* state, const float* action, const void* saved_fp64, const double* contact_record, void* workspace,
                       const float* grad_next_state, float* grad_state, float* grad_action, float* grad_inertia, int32_t* status_accum, cudaStream_t st,
                       int accumulate, const double* wi = nullptr, double* gIa = nullptr) {
  const nb2_variant& v = m->variants[m->contact_variant];
  const CStepArgs P = cstep_args(m, v, B, workspace, 1);
  const size_t smem_base = ((((size_t)P.bwd_words + 1) & ~(size_t)1) + NB2_WS_DESC_DOUBLES + ((P.ws_small_doubles + 1) & ~(size_t)1)) * sizeof(double);
  const size_t smem_staged = smem_base + ((((size_t)P.saved_words + 1) & ~(size_t)1) + 2) * sizeof(double);
  const int stage = pick_wpb(B, m->sm_count, smem_staged, NB2_CBWD_MAXW, 3) == pick_wpb(B, m->sm_count, smem_base, NB2_CBWD_MAXW, 3);
  const size_t smem = stage ? smem_staged : smem_base;
  const bool bounce = m->contact_restitution;  // some body has a restitution coefficient: the kernel with the second reverse sweep
  int rc = bounce ? cstep_smem_attr<k_cstep_bwd<true>>(smem) : cstep_smem_attr<k_cstep_bwd<false>>(smem);
  if (rc) return rc;
  NB2_CUDA(cudaMemsetAsync(workspace, 0, 64, st));
  const int wpb = pick_wpb(B, m->sm_count, smem, NB2_CBWD_MAXW, 3);
  if (bounce)
    k_cstep_bwd<true><<<(B + wpb - 1) / wpb, 32 * wpb, smem * wpb, st>>>(v.md, m->contact, P, state, action, (const double*)saved_fp64, contact_record, grad_next_state,
                                                                         grad_state, grad_action, grad_inertia, status_accum, smem, stage, accumulate, wi, gIa);
  else
    k_cstep_bwd<false><<<(B + wpb - 1) / wpb, 32 * wpb, smem * wpb, st>>>(v.md, m->contact, P, state, action, (const double*)saved_fp64, contact_record, grad_next_state,
                                                                          grad_state, grad_action, grad_inertia, status_accum, smem, stage, accumulate, wi, gIa);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
extern "C" {
int nb2_step_backward_contact(const nb2_model* cm, int B, const float* state, const float* action, const void* saved_fp64,
                              const double* contact_record, void* workspace, const float* grad_next_state, float* grad_state,
                              float* grad_action, float* grad_inertia, int32_t* status_accum, void* stream) {
  return nb2_step_backward_contact_pw(cm, B, state, action, nullptr, saved_fp64, contact_record, workspace, grad_next_state, grad_state, grad_action,
                                      grad_inertia, status_accum, stream);
}
int nb2_step_backward_contact_pw(const nb2_model* cm, int B, const float* state, const float* action, const double* world_inertia, const void* saved_fp64,
                                 const double* contact_record, void* workspace, const float* grad_next_state, float* grad_state,
                                 float* grad_action, float* grad_inertia, int32_t* status_accum, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (m && B == 0) return NB2_OK;
  if (!m || B < 0 || !state || !action || !saved_fp64 || !contact_record || !workspace || !grad_next_state || !grad_state || !grad_action) {
    g_err = "nb2_step_backward_contact: bad argument"; return NB2_ERR_INVALID;
  }
  if (!m->has_contacts) { g_err = "nb2_step_backward_contact: the model has no collision pairs"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  return cbwd_launch(m, B, state, action, saved_fp64, contact_record, workspace, grad_next_state, grad_state, grad_action, grad_inertia, status_accum,
                     (cudaStream_t)stream, 0, world_inertia);
}

// ---- whole-horizon rollouts of contact worlds (row f1): the T steps are queued from C, the LCP cache flows on the device, and the tape of
// saved streams / contact records is either complete (checkpoint_every <= 0 or >= T) or holds ONE segment of `checkpoint_every` steps that the
// reverse sweep refills by re-running the segment's forward from the stored state and the LCP-cache snapshot taken at its start.
struct RolloutTape {
  int k, nseg, nslots;
  size_t slot_doubles, saved_doubles, rec_doubles, snap_doubles, x_doubles;
  size_t o_slots, o_snaps, o_next, o_labels, o_status, o_nc, total_doubles;
  double* base;  // the tape buffer (nullptr when only its size is wanted)
  // slot i holds a step's saved stream followed by its contact record
  double* saved(int i) const { return base + o_slots + slot_doubles * i; }
  double* record(int i) const { return saved(i) + saved_doubles; }
  int32_t* labels() const { return reinterpret_cast<int32_t*>(base + o_labels); }
  int32_t* status() const { return reinterpret_cast<int32_t*>(base + o_status); }
  int32_t* nc() const { return reinterpret_cast<int32_t*>(base + o_nc); }
  float* next_scratch() const { return reinterpret_cast<float*>(base + o_next); }
  // snapshot i of the LCP cache: x, then m
  double* snap_x(int i) const { return base + o_snaps + snap_doubles * i; }
  int32_t* snap_m(int i) const { return reinterpret_cast<int32_t*>(snap_x(i) + x_doubles); }
};
static RolloutTape rollout_tape(const nb2_model* m, int B, int T, int checkpoint_every, void* tape = nullptr) {
  RolloutTape L;
  L.base = (double*)tape;
  L.k = (checkpoint_every <= 0 || checkpoint_every >= T) ? (T > 0 ? T : 1) : checkpoint_every;
  L.nseg = T > 0 ? (T + L.k - 1) / L.k : 0;
  L.nslots = L.k;
  L.saved_doubles = (size_t)m->saved_words * B;
  L.rec_doubles = (size_t)nb2::cw::record_doubles(m->mf.ndof) * B;
  L.slot_doubles = L.saved_doubles + L.rec_doubles;
  L.x_doubles = (size_t)NB2_MAX_ROWS * B;
  L.snap_doubles = L.x_doubles + ((size_t)B + 1) / 2;
  const bool ckpt = L.nseg > 1;
  size_t o = 0;
  L.o_slots = o; o += L.slot_doubles * L.nslots;
  L.o_snaps = o; o += ckpt ? L.snap_doubles * (L.nseg + 1) : 0;   // one per segment start + the cache after the last step
  L.o_next = o; o += ckpt ? ((size_t)2 * m->mf.ndof * B + 1) / 2 : 0;
  L.o_labels = o; o += ((size_t)NB2_MAX_ROWS * B + 1) / 2;
  L.o_status = o; o += ((size_t)B + 1) / 2;
  L.o_nc = o; o += ((size_t)B + 1) / 2;
  L.total_doubles = o;
  return L;
}
size_t nb2_rollout_contact_tape_bytes(const nb2_model* m, int B, int T, int checkpoint_every) {
  if (!m || !m->has_contacts || B <= 0 || T < 0) return 0;
  return rollout_tape(m, B, T, checkpoint_every).total_doubles * sizeof(double);
}
static int snap_copy(const RolloutTape& L, int idx, double* x_lcp, int32_t* m_lcp, int B, bool restore, cudaStream_t st) {
  double* sx = L.snap_x(idx);
  int32_t* sm = L.snap_m(idx);
  if (restore) {
    NB2_CUDA(cudaMemcpyAsync(x_lcp, sx, L.x_doubles * sizeof(double), cudaMemcpyDeviceToDevice, st));
    NB2_CUDA(cudaMemcpyAsync(m_lcp, sm, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  } else {
    NB2_CUDA(cudaMemcpyAsync(sx, x_lcp, L.x_doubles * sizeof(double), cudaMemcpyDeviceToDevice, st));
    NB2_CUDA(cudaMemcpyAsync(sm, m_lcp, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  return NB2_OK;
}
int nb2_rollout_forward_contact(const nb2_model* cm, int B, int T, float* states, const float* actions, double* x_lcp, int32_t* m_lcp, void* tape_,
                                int checkpoint_every, void* workspace, int32_t* status_accum, void* stream) {
  return nb2_rollout_forward_contact_pw(cm, B, T, states, actions, nullptr, x_lcp, m_lcp, tape_, checkpoint_every, workspace, status_accum, stream);
}
int nb2_rollout_forward_contact_pw(const nb2_model* cm, int B, int T, float* states, const float* actions, const double* world_inertia, double* x_lcp,
                                   int32_t* m_lcp, void* tape_, int checkpoint_every, void* workspace, int32_t* status_accum, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (m && (B == 0 || T == 0)) return NB2_OK;
  if (!m || B < 0 || T < 0 || !states || (!actions && T > 0) || !x_lcp || !m_lcp || !tape_ || !workspace) { g_err = "nb2_rollout_forward_contact: bad argument"; return NB2_ERR_INVALID; }
  if (!m->has_contacts) { g_err = "nb2_rollout_forward_contact: the model has no collision pairs (use nb2_rollout_forward)"; return NB2_ERR_INVALID; }
  if (B == 0 || T == 0) return NB2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const RolloutTape L = rollout_tape(m, B, T, checkpoint_every, tape_);
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  const bool ckpt = L.nseg > 1;
  for (int t = 0; t < T; t++) {
    int rc;
    if (ckpt && t % L.k == 0 && (rc = snap_copy(L, t / L.k, x_lcp, m_lcp, B, false, st))) return rc;
    const int slot = t % L.nslots;
    // with checkpoints the forward's records are thrown away (the reverse sweep regenerates them): do not write them
    rc = nb2_step_forward_contact_pw(m, B, states + n2 * B * t, actions + na * B * t, world_inertia, states + n2 * B * (t + 1), L.saved(slot), workspace,
                                     x_lcp, m_lcp, L.labels(), L.status(), L.nc(), nullptr, ckpt ? nullptr : L.record(slot), status_accum, stream);
    if (rc) return rc;
  }
  if (ckpt) return snap_copy(L, L.nseg, x_lcp, m_lcp, B, false, st);
  return NB2_OK;
}
int nb2_rollout_backward_contact(const nb2_model* cm, int B, int T, const float* states, const float* actions, double* x_lcp, int32_t* m_lcp, void* tape_,
                                 int checkpoint_every, float* grad_states, float* grad_actions, void* workspace, int32_t* status_accum, void* stream) {
  return nb2_rollout_backward_contact_pw(cm, B, T, states, actions, nullptr, x_lcp, m_lcp, tape_, checkpoint_every, grad_states, grad_actions, nullptr,
                                         workspace, status_accum, stream);
}
int nb2_rollout_backward_contact_pw(const nb2_model* cm, int B, int T, const float* states, const float* actions, const double* world_inertia, double* x_lcp,
                                    int32_t* m_lcp, void* tape_, int checkpoint_every, float* grad_states, float* grad_actions, double* grad_inertia,
                                    void* workspace, int32_t* status_accum, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (m && (B == 0 || T == 0)) return NB2_OK;
  if (!m || B < 0 || T < 0 || !states || (!actions && T > 0) || !x_lcp || !m_lcp || !tape_ || !grad_states || (!grad_actions && T > 0) || !workspace) {
    g_err = "nb2_rollout_backward_contact: bad argument"; return NB2_ERR_INVALID;
  }
  if (!m->has_contacts) { g_err = "nb2_rollout_backward_contact: the model has no collision pairs (use nb2_rollout_backward)"; return NB2_ERR_INVALID; }
  if (B == 0 || T == 0) return NB2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const RolloutTape L = rollout_tape(m, B, T, checkpoint_every, tape_);
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  const bool ckpt = L.nseg > 1;
  for (int seg = L.nseg - 1; seg >= 0; seg--) {
    const int t0 = seg * L.k, t1 = (t0 + L.k < T) ? t0 + L.k : T;
    int rc;
    if (ckpt) {
      // refill the tape: the segment's forward again, from the stored states and the LCP cache as it was at the segment start.  The stored
      // trajectory is NOT overwritten (the recomputed next states go to a scratch row; they are the same bits).
      if ((rc = snap_copy(L, seg, x_lcp, m_lcp, B, true, st))) return rc;
      for (int t = t0; t < t1; t++) {
        rc = nb2_step_forward_contact_pw(m, B, states + n2 * B * t, actions + na * B * t, world_inertia, L.next_scratch(), L.saved(t - t0), workspace, x_lcp,
                                         m_lcp, L.labels(), L.status(), L.nc(), nullptr, L.record(t - t0), nullptr, stream);
        if (rc) return rc;
      }
    }
    for (int t = t1 - 1; t >= t0; t--) {
      rc = cbwd_launch(m, B, states + n2 * B * t, actions + na * B * t, L.saved(t - t0), L.record(t - t0), workspace, grad_states + n2 * B * (t + 1),
                       grad_states + n2 * B * t, grad_actions + na * B * t, nullptr, status_accum, st, 1, world_inertia, grad_inertia);
      if (rc) return rc;
    }
  }
  if (ckpt) return snap_copy(L, L.nseg, x_lcp, m_lcp, B, true, st);  // leave the solver cache as the forward left it
  return NB2_OK;
}
int nb2_model_set_contact_capacity(nb2_model* m, int max_contacts_in_shared_memory) {
  if (!m || !m->has_contacts) { g_err = "nb2_model_set_contact_capacity: the model has no collision pairs"; return NB2_ERR_INVALID; }
  if (max_contacts_in_shared_memory < 1 || max_contacts_in_shared_memory > NB2_MAX_CONTACTS) { g_err = "nb2_model_set_contact_capacity: capacity must be in [1, NB2_MAX_CONTACTS]"; return NB2_ERR_INVALID; }
  m->contact_mc = max_contacts_in_shared_memory;
  return NB2_OK;
}
int nb2_model_contact_capacity(const nb2_model* m) { return (m && m->has_contacts) ? m->contact_mc : 0; }
/* dev builds (-DNB2_CW_PROFILE): per-phase cycle counters of the fused contact kernels; returns 0 when not compiled in */
int nb2_cw_profile_read(unsigned long long* out64, int reset) {
#ifdef NB2_CW_PROFILE
  if (out64 && cudaMemcpyFromSymbol(out64, nb2::cw::nb2_cw_prof, 64 * sizeof(unsigned long long)) != cudaSuccess) return 0;
  if (reset) { unsigned long long z[64] = {}; cudaMemcpyToSymbol(nb2::cw::nb2_cw_prof, z, sizeof(z)); }
  return 1;
#else
  (void)out64; (void)reset; return 0;
#endif
}
// ---- IKMapping entry points
struct nb2_ik_map { const nb2_model* m; int n, pos_dim, vel_dim; IkEntryDev* d_ent; };
int nb2_ik_create(const nb2_model* m, int nentries, const int32_t* type, const int32_t* body, const double* T_owner_from_body, nb2_ik_map** out) {
  if (!m || nentries <= 0 || !type || !body || !T_owner_from_body || !out) { g_err = "nb2_ik_create: bad argument"; return NB2_ERR_INVALID; }
  std::vector<IkEntryDev> ent(nentries);
  int po = 0, vo = 0;
  for (int e = 0; e < nentries; e++) {
    if (type[e] < 0 || type[e] > NB2_IK_COM || body[e] >= m->md.nb || (type[e] == NB2_IK_COM && (body[e] < 0 || m->md.parent[body[e]] >= 0))) {
      g_err = "nb2_ik_create: entry " + std::to_string(e) + " has a bad type / body (a COM entry names the root body of its tree)"; return NB2_ERR_INVALID;
    }
    ent[e].type = type[e]; ent[e].body = body[e]; ent[e].pos_off = po; ent[e].vel_off = vo;
    for (int k = 0; k < 12; k++) ent[e].T[k] = T_owner_from_body[12 * e + k];
    const int d = type[e] == NB2_IK_SPATIAL ? 6 : 3;
    po += d; vo += d;
  }
  nb2_ik_map* ik = new nb2_ik_map{m, nentries, po, vo, nullptr};
  if (cudaMalloc(&ik->d_ent, sizeof(IkEntryDev) * nentries) != cudaSuccess ||
      cudaMemcpy(ik->d_ent, ent.data(), sizeof(IkEntryDev) * nentries, cudaMemcpyHostToDevice) != cudaSuccess) {
    g_err = std::string("nb2_ik_create: ") + cudaGetErrorString(cudaGetLastError()); cudaFree(ik->d_ent); delete ik; return NB2_ERR_CUDA;
  }
  *out = ik;
  return NB2_OK;
}
void nb2_ik_destroy(nb2_ik_map* ik) { if (ik) { cudaFree(ik->d_ent); delete ik; } }
int nb2_ik_pos_dim(const nb2_ik_map* ik) { return ik ? ik->pos_dim : -1; }
int nb2_ik_vel_dim(const nb2_ik_map* ik) { return ik ? ik->vel_dim : -1; }
int nb2_ik_forward(const nb2_ik_map* ik, int B, const float* state, float* mapped_pos, float* mapped_vel, void* stream) {
  if (!ik || B < 0 || !state || (!mapped_pos && !mapped_vel)) { g_err = "nb2_ik_forward: bad argument"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  const long long threads = (long long)B * ik->n;
  k_ik_forward<<<(unsigned)((threads + 127) / 128), 128, 0, (cudaStream_t)stream>>>(ik->m->md, B, ik->n, ik->pos_dim, ik->vel_dim, ik->d_ent, state, mapped_pos, mapped_vel);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
int nb2_ik_backward(const nb2_ik_map* ik, int B, const float* state, const float* grad_pos, const float* grad_vel, float* grad_state, void* stream) {
  if (!ik || B < 0 || !state || !grad_state) { g_err = "nb2_ik_backward: bad argument"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  k_ik_backward<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ik->m->md, B, ik->n, ik->pos_dim, ik->vel_dim, ik->d_ent, state, grad_pos, grad_vel, grad_state);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}

int nb2_forward_dynamics(const nb2_model* cm, int B, const double* pos, const double* vel, const double* force, double* accel, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (!m || B < 0 || !pos || !vel || !force || !accel) { g_err = "nb2_forward_dynamics: bad argument"; return NB2_ERR_INVALID; }
  if (m->md.na != m->md.ndof) { g_err = "nb2_forward_dynamics: the action space must cover every dof (force is given per dof)"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  const nb2_variant& v = m->variants[0];
  double* scratch = nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  NB2_CUDA(cudaMallocAsync((void**)&scratch, (size_t)B * v.fwd_words * sizeof(double), st));
  k_forward_dynamics<<<(B + 63) / 64, 64, 0, st>>>(v.md, B, v.fwd_words, pos, vel, force, accel, scratch);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  NB2_CUDA(cudaFreeAsync(scratch, st));
  return NB2_OK;
}
int nb2_lcp_solve_batch(int B, int mcap, int mode, int early_termination, double fallback_cfm, const int32_t* m, const double* A, const double* b,
                        const double* lo, const double* hi, const int32_t* findex, const double* x0, double* x, int32_t* labels, int32_t* status,
                        void* stream) {
  if (B < 0 || mcap < 1 || mcap > NB2_MAX_ROWS || !m || !A || !b || !lo || !hi || !findex || !x || !status || (mode != 0 && mode != 1)) {
    g_err = "nb2_lcp_solve_batch: bad argument (1 <= mcap <= NB2_MAX_ROWS)"; return NB2_ERR_INVALID;
  }
  if (B == 0) return NB2_OK;
  const nb2::cw::Dims d = nb2::cw::make_dims(1, 1, 0, (mcap + 2) / 3 + 1, mcap < 3 ? 3 : mcap, 1, 1, 0, NB2_WS_SOLVE);
  const size_t smem = (NB2_WS_DESC_DOUBLES + nb2::cw::ws_doubles(d)) * sizeof(double);
  int rc = cstep_smem_attr<k_lcp_batch>(smem);
  if (rc) return rc;
  k_lcp_batch<<<B, 32, smem, (cudaStream_t)stream>>>(d, B, mcap, fallback_cfm, mode, early_termination, m, A, b, lo, hi, findex, x0, x, labels, status);
  g_launches++;
  NB2_CUDA(cudaGetLastError());
  return NB2_OK;
}
int nb2_model_ndof(const nb2_model* m) { return m ? m->mf.ndof : -1; }
int nb2_model_na(const nb2_model* m) { return m ? m->mf.na : -1; }
int nb2_saved_words_per_world(const nb2_model* m) { return m ? m->saved_words : -1; }

int nb2_step_forward(const nb2_model* cm, int B, const float* state, const float* action, float* next_state,
                     void* saved, int precision, void* stream) {
  return nb2_step_forward_pw(cm, B, state, action, nullptr, next_state, saved, precision, stream);
}
int nb2_step_forward_pw(const nb2_model* cm, int B, const float* state, const float* action, const double* world_inertia, float* next_state,
                        void* saved, int precision, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (!m || B < 0 || !state || !action || !next_state) { g_err = "nb2_step_forward: bad argument"; return NB2_ERR_INVALID; }
  if (m->has_contacts) { g_err = "nb2_step_forward: the model has collision pairs: use nb2_step_forward_contact (or build the model without shapes for a contact-free step)"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  return with_precision(precision, [&](auto r) {
    using R = decltype(r);
    return launch_fwd<R>(m, B, state, action, next_state, (R*)saved, st, -1, 0, nullptr, nullptr, world_inertia);
  });
}

int nb2_step_backward(const nb2_model* cm, int B, const float* state, const float* action, const void* saved,
                      const float* grad_next_state, float* grad_state, float* grad_action, float* grad_inertia,
                      int precision, void* stream) {
  return nb2_step_backward_pw(cm, B, state, action, nullptr, saved, grad_next_state, grad_state, grad_action, grad_inertia, precision, stream);
}
int nb2_step_backward_pw(const nb2_model* cm, int B, const float* state, const float* action, const double* world_inertia, const void* saved,
                         const float* grad_next_state, float* grad_state, float* grad_action, float* grad_inertia,
                         int precision, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (!m || B < 0 || !state || !action || !saved || !grad_next_state || !grad_state || !grad_action) {
    g_err = "nb2_step_backward: bad argument"; return NB2_ERR_INVALID;
  }
  if (m->has_contacts) { g_err = "nb2_step_backward: the model has collision pairs: use nb2_step_backward_contact"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  return with_precision(precision, [&](auto r) {
    using R = decltype(r);
    return launch_bwd<R>(m, B, state, action, (const R*)saved, grad_next_state, grad_state, grad_action, grad_inertia, st, -1, 0, 0, world_inertia);
  });
}

int nb2_rollout_forward(const nb2_model* cm, int B, int T, float* states, const float* actions, void* saved, int precision, void* stream) {
  return nb2_rollout_forward_pw(cm, B, T, states, actions, nullptr, saved, precision, stream);
}
int nb2_rollout_forward_pw(const nb2_model* cm, int B, int T, float* states, const float* actions, const double* world_inertia, void* saved, int precision,
                           void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (!m || B < 0 || T < 0 || !states || (!actions && T > 0)) { g_err = "nb2_rollout_forward: bad argument"; return NB2_ERR_INVALID; }
  if (m->has_contacts) { g_err = "nb2_rollout_forward: contact worlds roll out through nb2_step_forward_contact (one call per step)"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  const size_t sv_step = (size_t)m->saved_words * B * (precision == NB2_FP64 ? sizeof(double) : sizeof(float));
  for (int t = 0; t < T; t++) {  // x_{t+1} = step(x_t, u_t): every launch reads the rows the previous one wrote (stream order)
    void* sv = saved ? (char*)saved + sv_step * t : nullptr;
    int rc = nb2_step_forward_pw(m, B, states + n2 * B * t, actions + na * B * t, world_inertia, states + n2 * B * (t + 1), sv, precision, stream);
    if (rc) return rc;
  }
  return NB2_OK;
}

int nb2_rollout_backward(const nb2_model* cm, int B, int T, const float* states, const float* actions, const void* saved,
                         float* grad_states, float* grad_actions, int precision, void* stream) {
  return nb2_rollout_backward_pw(cm, B, T, states, actions, nullptr, saved, grad_states, grad_actions, nullptr, precision, stream);
}
int nb2_rollout_backward_pw(const nb2_model* cm, int B, int T, const float* states, const float* actions, const double* world_inertia, const void* saved,
                            float* grad_states, float* grad_actions, double* grad_inertia, int precision, void* stream) {
  nb2_model* m = const_cast<nb2_model*>(cm);
  if (!m || B < 0 || T < 0 || !states || !saved || !grad_states || (!actions && T > 0) || (!grad_actions && T > 0)) { g_err = "nb2_rollout_backward: bad argument"; return NB2_ERR_INVALID; }
  if (m->has_contacts) { g_err = "nb2_rollout_backward: contact worlds back-propagate through nb2_step_backward_contact"; return NB2_ERR_INVALID; }
  if (B == 0) return NB2_OK;
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  cudaStream_t st = (cudaStream_t)stream;
  return with_precision(precision, [&](auto r) {
    using R = decltype(r);
    for (int t = T - 1; t >= 0; t--) {  // grad_states[t] += clip(J_t^T grad_states[t+1]) ; grad_actions[t] = ...
      const R* sv = (const R*)saved + (size_t)m->saved_words * B * t;
      int rc = launch_bwd<R>(m, B, states + n2 * B * t, actions + na * B * t, sv, grad_states + n2 * B * (t + 1), grad_states + n2 * B * t,
                             grad_actions + na * B * t, nullptr, st, -1, 0, 1, world_inertia, grad_inertia);
      if (rc) return rc;
    }
    return (int)NB2_OK;
  });
}

static int ensure_host_buffers(nb2_model* m, int B) {
  for (auto& hs : m->host_streams) if (!hs) NB2_CUDA(cudaStreamCreateWithFlags(&hs, cudaStreamNonBlocking));
  if (B <= m->host_cap) return NB2_OK;
  cudaFree(m->d_state); cudaFree(m->d_action); cudaFree(m->d_next); cudaFree(m->d_saved);
  cudaFree(m->d_gnext); cudaFree(m->d_gstate); cudaFree(m->d_gaction);
  m->d_state = m->d_action = m->d_next = m->d_gnext = m->d_gstate = m->d_gaction = nullptr;
  m->d_saved = nullptr;
  m->host_cap = 0;
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)(m->mf.na > 0 ? m->mf.na : 1);
  NB2_CUDA(cudaMalloc(&m->d_state, n2 * B * sizeof(float)));
  NB2_CUDA(cudaMalloc(&m->d_action, na * B * sizeof(float)));
  NB2_CUDA(cudaMalloc(&m->d_next, n2 * B * sizeof(float)));
  NB2_CUDA(cudaMalloc(&m->d_saved, (size_t)m->saved_words * B * sizeof(double)));
  NB2_CUDA(cudaMalloc(&m->d_gnext, n2 * B * sizeof(float)));
  NB2_CUDA(cudaMalloc(&m->d_gstate, n2 * B * sizeof(float)));
  NB2_CUDA(cudaMalloc(&m->d_gaction, na * B * sizeof(float)));
  m->host_cap = B;
  return NB2_OK;
}

int nb2_step_forward_host(nb2_model* m, int B, const float* state, const float* action, float* next_state,
                          int keep_for_backward, int precision) {
  if (!m || B <= 0 || !state || !action || !next_state) { g_err = "nb2_step_forward_host: bad argument"; return NB2_ERR_INVALID; }
  if (m->has_contacts) { g_err = "nb2_step_forward_host: the model has collision pairs: use nb2_step_forward_contact_host"; return NB2_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(m->mu);
  int rc = ensure_host_buffers(m, B);
  if (rc) return rc;
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  if (zero_copy_enabled()) {
    const float* zs = mapped_alias(state); const float* za = mapped_alias(action); float* zn = mapped_alias(next_state);
    if (zs && za && zn) {
      cudaStream_t st = m->host_streams[0];
      rc = with_precision(precision, [&](auto r) {
        using R = decltype(r);
        return launch_fwd<R>(m, B, zs, za, zn, keep_for_backward ? (R*)m->d_saved : nullptr, st, B, 0, m->d_state, m->d_action);
      });
      if (rc) return rc;
      NB2_CUDA(cudaStreamSynchronize(st));
      m->host_B = keep_for_backward ? B : 0;
      return NB2_OK;
    }
  }
  const int C = host_chunks(B);
  for (int c = 0; c < C; c++) {
    const int lo = (int)((long long)B * c / C), cnt = (int)((long long)B * (c + 1) / C) - lo;
    cudaStream_t st = m->host_streams[c];
    NB2_CUDA(cudaMemcpyAsync(m->d_state + n2 * lo, state + n2 * lo, n2 * cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    NB2_CUDA(cudaMemcpyAsync(m->d_action + na * lo, action + na * lo, na * cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    rc = with_precision(precision, [&](auto r) {
      using R = decltype(r);
      return launch_fwd<R>(m, cnt, m->d_state, m->d_action, m->d_next, keep_for_backward ? (R*)m->d_saved : nullptr, st, B, lo);
    });
    if (rc) return rc;
    NB2_CUDA(cudaMemcpyAsync(next_state + n2 * lo, m->d_next + n2 * lo, n2 * cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  for (int c = 0; c < C; c++) NB2_CUDA(cudaStreamSynchronize(m->host_streams[c]));
  m->host_B = keep_for_backward ? B : 0;
  return NB2_OK;
}

int nb2_step_backward_host(nb2_model* m, int B, const float* grad_next_state, float* grad_state, float* grad_action,
                           int precision) {
  if (!m || !grad_next_state || !grad_state || !grad_action) { g_err = "nb2_step_backward_host: bad argument"; return NB2_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(m->mu);
  if (B <= 0 || B != m->host_B) { g_err = "nb2_step_backward_host: no matching forward_host(keep_for_backward=1) precedes this call"; return NB2_ERR_INVALID; }
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  if (zero_copy_enabled()) {
    const float* zg = mapped_alias(grad_next_state); float* zgs = mapped_alias(grad_state); float* zga = mapped_alias(grad_action);
    if (zg && zgs && zga) {
      cudaStream_t st = m->host_streams[0];
      int rc = with_precision(precision, [&](auto r) {
        using R = decltype(r);
        return launch_bwd<R>(m, B, m->d_state, m->d_action, (const R*)m->d_saved, zg, zgs, zga, nullptr, st);
      });
      if (rc) return rc;
      NB2_CUDA(cudaStreamSynchronize(st));
      return NB2_OK;
    }
  }
  const int C = host_chunks(B);
  for (int c = 0; c < C; c++) {
    const int lo = (int)((long long)B * c / C), cnt = (int)((long long)B * (c + 1) / C) - lo;
    cudaStream_t st = m->host_streams[c];
    NB2_CUDA(cudaMemcpyAsync(m->d_gnext + n2 * lo, grad_next_state + n2 * lo, n2 * cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    int rc = with_precision(precision, [&](auto r) {
      using R = decltype(r);
      return launch_bwd<R>(m, cnt, m->d_state, m->d_action, (const R*)m->d_saved, m->d_gnext, m->d_gstate, m->d_gaction, nullptr, st, B, lo);
    });
    if (rc) return rc;
    NB2_CUDA(cudaMemcpyAsync(grad_state + n2 * lo, m->d_gstate + n2 * lo, n2 * cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
    NB2_CUDA(cudaMemcpyAsync(grad_action + na * lo, m->d_gaction + na * lo, na * cnt * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  for (int c = 0; c < C; c++) NB2_CUDA(cudaStreamSynchronize(m->host_streams[c]));
  return NB2_OK;
}

// ---- host entry points of the contact path (pageable or pinned host buffers; staged copies on one stream, synchronised on return).  The solver
// cache, the saved stream, the contact record and the sticky status live in the model between the calls.
static int ensure_host_contact_buffers(nb2_model* m, int B) {
  int rc = ensure_host_buffers(m, B);
  if (rc) return rc;
  if (B <= m->hc_cap) return NB2_OK;
  cudaFree(m->hc_ws); cudaFree(m->hc_x); cudaFree(m->hc_rec); cudaFree(m->hc_m); cudaFree(m->hc_labels); cudaFree(m->hc_status); cudaFree(m->hc_nc); cudaFree(m->hc_sticky);
  m->hc_ws = nullptr; m->hc_x = m->hc_rec = nullptr; m->hc_m = m->hc_labels = m->hc_status = m->hc_nc = m->hc_sticky = nullptr; m->hc_cap = 0;
  const int cap = m->host_cap;  // (ensure_host_buffers sized the state / saved buffers for this many worlds)
  NB2_CUDA(cudaMalloc(&m->hc_ws, nb2_contact_workspace_bytes(m, cap)));
  NB2_CUDA(cudaMalloc(&m->hc_x, (size_t)cap * NB2_MAX_ROWS * sizeof(double)));
  NB2_CUDA(cudaMalloc(&m->hc_rec, nb2_contact_record_bytes(m, cap)));
  NB2_CUDA(cudaMalloc(&m->hc_m, (size_t)cap * sizeof(int32_t)));
  NB2_CUDA(cudaMalloc(&m->hc_labels, (size_t)cap * NB2_MAX_ROWS * sizeof(int32_t)));
  NB2_CUDA(cudaMalloc(&m->hc_status, (size_t)cap * sizeof(int32_t)));
  NB2_CUDA(cudaMalloc(&m->hc_nc, (size_t)cap * sizeof(int32_t)));
  NB2_CUDA(cudaMalloc(&m->hc_sticky, (size_t)cap * sizeof(int32_t)));
  NB2_CUDA(cudaMemset(m->hc_m, 0xff, (size_t)cap * sizeof(int32_t)));  // -1: no cached solution
  NB2_CUDA(cudaMemset(m->hc_x, 0, (size_t)cap * NB2_MAX_ROWS * sizeof(double)));
  NB2_CUDA(cudaMemset(m->hc_sticky, 0, (size_t)cap * sizeof(int32_t)));
  m->hc_cap = cap;
  return NB2_OK;
}
int nb2_step_forward_contact_host(nb2_model* m, int B, const float* state, const float* action, float* next_state, int keep_for_backward,
                                  int reset_cache, int32_t* status_out) {
  if (!m || B <= 0 || !state || !action || !next_state) { g_err = "nb2_step_forward_contact_host: bad argument"; return NB2_ERR_INVALID; }
  if (!m->has_contacts) { g_err = "nb2_step_forward_contact_host: the model has no collision pairs (use nb2_step_forward_host)"; return NB2_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(m->mu);
  int rc = ensure_host_contact_buffers(m, B);
  if (rc) return rc;
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  cudaStream_t st = m->host_streams[0];
  if (reset_cache) NB2_CUDA(cudaMemsetAsync(m->hc_m, 0xff, (size_t)B * sizeof(int32_t), st));
  NB2_CUDA(cudaMemcpyAsync(m->d_state, state, n2 * B * sizeof(float), cudaMemcpyHostToDevice, st));
  NB2_CUDA(cudaMemcpyAsync(m->d_action, action, na * B * sizeof(float), cudaMemcpyHostToDevice, st));
  rc = nb2_step_forward_contact(m, B, m->d_state, m->d_action, m->d_next, m->d_saved, m->hc_ws, m->hc_x, m->hc_m, m->hc_labels, m->hc_status, m->hc_nc, nullptr,
                                keep_for_backward ? m->hc_rec : nullptr, m->hc_sticky, st);
  if (rc) return rc;
  NB2_CUDA(cudaMemcpyAsync(next_state, m->d_next, n2 * B * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (status_out) NB2_CUDA(cudaMemcpyAsync(status_out, m->hc_status, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NB2_CUDA(cudaStreamSynchronize(st));
  m->host_B = keep_for_backward ? B : 0;
  return NB2_OK;
}
int nb2_step_backward_contact_host(nb2_model* m, int B, const float* grad_next_state, float* grad_state, float* grad_action, int32_t* sticky_out) {
  if (!m || B <= 0 || !grad_next_state || !grad_state || !grad_action) { g_err = "nb2_step_backward_contact_host: bad argument"; return NB2_ERR_INVALID; }
  if (!m->has_contacts) { g_err = "nb2_step_backward_contact_host: the model has no collision pairs"; return NB2_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(m->mu);
  if (m->host_B != B) { g_err = "nb2_step_backward_contact_host: no forward of this batch size was kept (keep_for_backward)"; return NB2_ERR_INVALID; }
  const size_t n2 = (size_t)2 * m->mf.ndof, na = (size_t)m->mf.na;
  cudaStream_t st = m->host_streams[0];
  NB2_CUDA(cudaMemcpyAsync(m->d_gnext, grad_next_state, n2 * B * sizeof(float), cudaMemcpyHostToDevice, st));
  int rc = nb2_step_backward_contact(m, B, m->d_state, m->d_action, m->d_saved, m->hc_rec, m->hc_ws, m->d_gnext, m->d_gstate, m->d_gaction, nullptr, m->hc_sticky, st);
  if (rc) return rc;
  NB2_CUDA(cudaMemcpyAsync(grad_state, m->d_gstate, n2 * B * sizeof(float), cudaMemcpyDeviceToHost, st));
  NB2_CUDA(cudaMemcpyAsync(grad_action, m->d_gaction, na * B * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (sticky_out) {  // read-and-clear: the OR of every step's status word since the last read
    NB2_CUDA(cudaMemcpyAsync(sticky_out, m->hc_sticky, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    NB2_CUDA(cudaMemsetAsync(m->hc_sticky, 0, (size_t)B * sizeof(int32_t), st));
  }
  NB2_CUDA(cudaStreamSynchronize(st));
  return NB2_OK;
}

}  // extern "C"
