// The mbarrier stage ring of the warp-specialized kernels (gemm_ws.cu, attention_wgmma.cu): one producer thread fills S
// shared-memory stages by TMA, consumer warps read them with wgmma, and both count the blocks g = 0, 1, ... in one order.
// Block g sits in stage g % S.  full[s] takes 1 arrival (arrive_expect_tx) plus the TMA bytes: block g has landed once the
// full phase of parity (g / S) & 1 has completed.  empty[s] takes one arrival per consumer warp, once wgmma.wait_group has
// retired the MMAs that read the stage: the producer refills stage g % S with block g >= S after the empty phase
// ((g / S) - 1) & 1, the release of block g - S.  Waits are mbar_wait<false>: a printf there would make ptxas serialize the
// caller's wgmma (see ptx.cuh).  tools/kernel_models.py reads these rules from here.
#pragma once
#include "ptx.cuh"

namespace av2v {

template <int S>
struct StageRing {  // declared __shared__
  uint64_t full[S], empty[S];
  static __device__ __forceinline__ int stage(int g) { return g % S; }
  // one thread; the caller then issues fence_mbar_init() once, after any other barriers it inits
  __device__ __forceinline__ void init(int consumer_warps) {
#pragma unroll
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], consumer_warps);
    }
  }
  // producer: waits until stage(g) is free and posts block g's bytes; returns the barrier its TMA loads complete on
  __device__ __forceinline__ uint64_t* produce(int g, uint32_t bytes) {
    if (g >= S) mbar_wait<false>(&empty[stage(g)], ((g / S) - 1) & 1);
    mbar_arrive_expect_tx(&full[stage(g)], bytes);
    return &full[stage(g)];
  }
  __device__ __forceinline__ void wait(int g) { mbar_wait<false>(&full[stage(g)], (g / S) & 1); }
  // a whole consumer warp, once the MMAs that read block g have retired
  __device__ __forceinline__ void release(int g) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage(g)]);
  }
};

// Two consumer warpgroups wg = 0, 1 (256 threads) taking turns: wg waits on named barrier 1 + wg, hands over on the other's.
__device__ __forceinline__ void turn_open(int wg) { if (wg == 1) named_bar_arrive(1, 256); }  // so warpgroup 0 goes first
__device__ __forceinline__ void turn_take(int wg) { if (wg == 0) named_bar_sync(1, 256); else named_bar_sync(2, 256); }
__device__ __forceinline__ void turn_hand_over(int wg) { if (wg == 0) named_bar_arrive(2, 256); else named_bar_arrive(1, 256); }

}  // namespace av2v
