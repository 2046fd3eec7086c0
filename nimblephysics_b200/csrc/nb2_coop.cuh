// The group shape of the contact-free kernels (step, inverse and forward dynamics), shared by nb2_kernels.cu and nb2_fd.cu.
#pragma once
#include <cuda_runtime.h>

#include "nb2_dyn.cuh"

namespace {

// A GROUP is 32 consecutive worlds worked on by K warps (K = M.lanes, compile-time here so that the shape is a constant): warp r
// of the group plays lane r of the schedule for all 32 worlds, and thread t of every warp is world slot t.  So no warp ever
// holds two bodies at once: every per-body read of the model (the __grid_constant__ kernel parameter) has a warp-uniform index
// and is one constant-bank broadcast.  The group's scratch is [word][slot] with stride 33: the sweeps (consecutive threads on
// consecutive slots) and the group I/O (consecutive threads on consecutive words of a world's row, which keeps the global rows
// coalesced) both spread over the banks (a bound reasoned from the access pattern, not measured).  K = 1 keeps stride 32, the one-warp
// shape's stride before groups existed: its footprint and code stay those of that shape.  A block holds one group when K > 1 (so the
// group's barrier is the block's named barrier 1 and no group index stays live in the sweeps, which kept the fp64 kernels at their
// spill counts) and up to four one-warp groups when K = 1.
// W = NARROW_W<K> = 32/K (K > 1): a NARROW group (slots W..31 idle, stride W + 1) for a K-lane schedule whose 32-world scratch
// does not fit shared memory: its scratch is about 1/K of a 32-world group's, what one warp of the same schedule needs.
template <int K> constexpr int NARROW_W = 32 / K;
template <int K, int W = 32> struct GroupShape {
  static constexpr int WPG = W;                             // worlds per group
  static constexpr int ST = (K == 1) ? 32 : W + 1;          // scratch stride in words (see above for K = 1)
  static constexpr int THREADS = 32 * K;                    // threads per group
  static constexpr int MAX_GROUPS = (K >= 2) ? 1 : 4;        // groups per block
  static constexpr int MAX_THREADS = THREADS * MAX_GROUPS;  // threads per block (the kernels' launch bound)
};

// A stage barrier over the K warps of the group: the block's named barrier 1 (0 is __syncthreads').  barrier.sync, not bar.sync:
// the threads of a partial group's missing slots skip the sweeps, so a warp may reach it diverged.
template <int K> __device__ __forceinline__ void group_sync() {
  if constexpr (K == 1) __syncwarp();
  else asm volatile("barrier.sync 1, %0;" ::"n"(32 * K) : "memory");
}

// Where thread threadIdx.x sits in the group shape, and the worlds its group covers: [w0 + g0, w0 + g0 + nworlds) of a launch over
// `count` worlds.  nworlds <= 0: an idle group (grid tail).
template <int K, int W = 32> struct GroupPos {
  int gb, tid, lane, slot, gi, g0, nworlds;
  __device__ __forceinline__ GroupPos(int count) {
    gb = (GroupShape<K, W>::MAX_GROUPS == 1) ? 0 : threadIdx.x / GroupShape<K, W>::THREADS;  // group of the block
    tid = threadIdx.x - gb * GroupShape<K, W>::THREADS;    // thread of the group (its group I/O index)
    lane = tid >> 5;
    slot = tid & 31;
    gi = blockIdx.x * (blockDim.x / GroupShape<K, W>::THREADS) + gb;  // group of the grid
    g0 = gi * W;
    nworlds = min(W, count - g0);
  }
  __device__ __forceinline__ bool valid() const { return slot < nworlds; }
};

}  // namespace
