// Row-kernel helpers shared by the LayerNorm / softmax kernels of norm.cu and their dropout forms in dropout.cu:
// warp and lane-group reductions, bf16x8 <-> fp32 conversions, and the (LPR, VPL) dispatch of the vectorised row
// kernels.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "pdl.cuh"
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

// ---- vectorised LayerNorm bodies: the kernels of norm.cu (SUM = false) and the pre-LN add + LayerNorm of vit.cu
// SUM (pre-LN transformer blocks): s = bf16(x + res) is written to `sum` and normalised as rounded, so y = LN(s)
// holds for the stored s that the backward re-reads
template <int LPR, int VPL, bool SUM>
__device__ __forceinline__ void
layernorm_fwd_vec_body(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                       __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ mean, float* __restrict__ rstd, long long rows, int C, float eps,
                       __nv_bfloat16* __restrict__ sum) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int RPW = 32 / LPR;                       // rows per warp
  const int gl = threadIdx.x & (LPR - 1);
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW +
                        ((threadIdx.x & 31) / LPR);
  const bool row_ok = row < rows;                     // lanes of a dead row still join the shuffles
  const int nvec = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (row_ok ? row : 0) * C);
  const uint4* rr = res != nullptr ? reinterpret_cast<const uint4*>(res + (row_ok ? row : 0) * C) : nullptr;
  float v[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (row_ok && idx < nvec) {
      unpack8(xr[idx], v[k]);
      if (rr != nullptr) {
        float r8[8];
        unpack8(rr[idx], r8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[k][j] += r8[j];
      }
      if constexpr (SUM) {
        const uint4 sv = pack8(v[k]);
        reinterpret_cast<uint4*>(sum + row * C)[idx] = sv;
        unpack8(sv, v[k]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[k][j];
    }
  }
  const float mu = group_sum<LPR>(s) / C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (row_ok && gl + k * LPR < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[k][j] - mu;
        q = fmaf(d, d, q);
      }
    }
  const float rs = rsqrtf(group_sum<LPR>(q) / C + eps);
  if (!row_ok) return;
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (idx < nvec) {
      float g8[8], b8[8], o[8];
      load8f(gamma + idx * 8, g8);
      load8f(beta + idx * 8, b8);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf((v[k][j] - mu) * rs, g8[j], b8[j]);
      yr[idx] = pack8(o);
    }
  }
  if (gl == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
}
// SUM: dx = LN_bwd(dy) + ds, rounded once -- the gradient of both summands of a pre-LN block's residual add
template <int LPR, int VPL, bool SUM>
__device__ __forceinline__ void
layernorm_bwd_vec_body(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                       __nv_bfloat16* __restrict__ dx, const float* __restrict__ gamma, const float* __restrict__ mean,
                       const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                       long long rows, int C, const __nv_bfloat16* __restrict__ ds) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // dgamma[C], dbeta[C] partials of this block
  float* sg = sm;
  float* sb = sm + C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { sg[c] = 0.f; sb[c] = 0.f; }
  __syncthreads();
  constexpr int RPW = 32 / LPR;
  const int gl = threadIdx.x & (LPR - 1);
  const int nvec = C >> 3;
  const long long groups = static_cast<long long>(gridDim.x) * (blockDim.x >> 5) * RPW;
  const long long g0 = (blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW +
                       ((threadIdx.x & 31) / LPR);
  float dg[VPL][8], db[VPL][8];
#pragma unroll
  for (int k = 0; k < VPL; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) { dg[k][j] = 0.f; db[k][j] = 0.f; }
  // trip count is uniform across the warp (dead rows are predicated), so the shuffles stay legal
  for (long long base = 0; base < rows; base += groups) {
    const long long row = base + g0;
    const bool row_ok = row < rows;
    const uint4* xr = reinterpret_cast<const uint4*>(x + (row_ok ? row : 0) * C);
    const uint4* gr = reinterpret_cast<const uint4*>(dy + (row_ok ? row : 0) * C);
    uint4 xu[VPL], gu[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int idx = gl + k * LPR;
      if (row_ok && idx < nvec) {
        xu[k] = __ldcs(xr + idx);
        gu[k] = __ldcs(gr + idx);
      }
    }
    const float mu = row_ok ? mean[row] : 0.f, rs = row_ok ? rstd[row] : 0.f;
    float xh[VPL][8], gw[VPL][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int idx = gl + k * LPR;
      if (row_ok && idx < nvec) {
        float g8[8], gm[8];
        unpack8(xu[k], xh[k]);
        unpack8(gu[k], g8);
        load8f(gamma + idx * 8, gm);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float h = (xh[k][j] - mu) * rs;
          xh[k][j] = h;
          dg[k][j] = fmaf(g8[j], h, dg[k][j]);
          db[k][j] += g8[j];
          const float w = g8[j] * gm[j];
          gw[k][j] = w;
          s1 += w;
          s2 = fmaf(w, h, s2);
        }
      }
    }
    s1 = group_sum<LPR>(s1) / C;
    s2 = group_sum<LPR>(s2) / C;
    if (row_ok) {
      uint4* dr = reinterpret_cast<uint4*>(dx + row * C);
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const int idx = gl + k * LPR;
        if (idx < nvec) {
          float o[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = rs * (gw[k][j] - s1 - xh[k][j] * s2);
          if constexpr (SUM) {
            float d8[8];
            unpack8(__ldcs(reinterpret_cast<const uint4*>(ds + row * C) + idx), d8);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += d8[j];
          }
          dr[idx] = pack8(o);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (idx < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(sg + idx * 8 + j, dg[k][j]);
        atomicAdd(sb + idx * 8 + j, db[k][j]);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(dgamma + c, sg[c]);
    atomicAdd(dbeta + c, sb[c]);
  }
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
