// Pieces of the GEMM epilogues shared by gemm_wgmma.cu and conv_halo.cu: cluster rank / barrier and the warp
// butterflies behind the fused BatchNorm column statistics.
#pragma once
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Column sums of a 32 x 32 register block held one ROW per lane.  Butterfly: at every step a lane keeps one
// half of its remaining columns and trades the other half with its partner, so after 5 steps (31 shuffles)
// lane j owns the complete sum of column j.
#define COLSUM_STEP(OFF, HALF)                                                  \
  {                                                                             \
    const bool upper = (lane & (OFF)) != 0;                                     \
    _Pragma("unroll") for (int i = 0; i < (HALF); ++i) {                        \
      const float keep = upper ? t[i + (HALF)] : t[i];                          \
      const float send = upper ? t[i] : t[i + (HALF)];                          \
      t[i] = keep + __shfl_xor_sync(0xffffffffu, send, (OFF));                  \
    }                                                                           \
  }
__device__ __forceinline__ float warp_colsum32(float (&t)[32]) {
  const uint32_t lane = lane_id();
  COLSUM_STEP(16, 16) COLSUM_STEP(8, 8) COLSUM_STEP(4, 4) COLSUM_STEP(2, 2) COLSUM_STEP(1, 1)
  return t[0];
}
#undef COLSUM_STEP

// Same butterflies, but the warp's column sums go to shared memory (`sbuf[0:BN]` sums, `sbuf[BN:2BN]` sums of squares of
// ONE warp): the four epilogue warps of a CTA are combined there and the CTA issues ONE global atomic per statistic
// instead of four -- with 256 CTAs (ResNet stem) the atomics of a launch pile up on 2 N addresses and serialise in L2.
__device__ __forceinline__ void stage_col_stats(float* sbuf, int BNv, int c, const float (&v)[32]) {
  float s[32], q[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float r = __bfloat162float(__float2bfloat16_rn(v[j]));
    s[j] = r;
    q[j] = r * r;
  }
  const float cs = warp_colsum32(s), cq = warp_colsum32(q);
  const int lane = static_cast<int>(lane_id());
  sbuf[c + lane] = cs;
  sbuf[BNv + c + lane] = cq;
}

}  // namespace b200
