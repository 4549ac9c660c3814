// Row-kernel helpers shared by the LayerNorm / softmax kernels of norm.cu and their dropout forms in dropout.cu:
// warp and lane-group reductions, bf16x8 <-> fp32 conversions, and the (LPR, VPL) dispatch of the vectorised row
// kernels.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

constexpr int LN_MAX_PER_LANE = 32;  // supports C <= 1024 * ... (C / 32 elements per lane, <= 32)

// ---- vectorised row kernels
// A row of C elements (C % 8 == 0, C <= 1024) is owned by a group of LPR adjacent lanes (8, 16 or 32), each
// holding VPL 16-byte vectors entirely in registers: 128-bit coalesced loads/stores, no local memory, group
// reductions by xor-shuffles that stay inside the group.
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int LPR>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int o = LPR >> 1; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
__device__ __forceinline__ void load8f(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// (LPR, VPL) for a row length: the smallest group that covers the row with at most 4 vectors per lane
#define ROW_DISPATCH(C, CALL)                                     \
  do {                                                           \
    const int nvec_ = (C) >> 3;                                  \
    if (nvec_ <= 8) { CALL(8, 1); }                              \
    else if (nvec_ <= 16) { CALL(16, 1); }                       \
    else if (nvec_ <= 32) { CALL(32, 1); }                       \
    else if (nvec_ <= 64) { CALL(32, 2); }                       \
    else if (nvec_ <= 96) { CALL(32, 3); }                       \
    else { CALL(32, 4); }                                        \
  } while (0)
static inline bool row_vec_ok(int C, const void* a, const void* b, const void* c) {
  return C % 8 == 0 && C <= 1024 && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                                       reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}
static inline int rows_per_block(int C) {   // 8 warps x rows per warp
  const int nvec = C >> 3;
  return 8 * (nvec <= 8 ? 4 : (nvec <= 16 ? 2 : 1));
}

}  // namespace b200
