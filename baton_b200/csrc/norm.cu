// Normalisation kernels (K6): BatchNorm forward/backward over NHWC activations viewed as a
// [rows, C] bf16 matrix (fused residual add + ReLU, running-stat update), LayerNorm forward /
// backward (fused residual add) and row softmax for attention.  Statistics and gradients in fp32.
#define B200_TU_TAG 10
#include <atomic>

#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"
#include "rows.cuh"

namespace b200 {

// cluster helpers (BatchNorm backward cluster kernel)
__device__ __forceinline__ uint32_t cluster_ctarank_any() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank_y() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive_norm() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_norm() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_sync_all_norm() {
  cluster_arrive_norm();
  cluster_wait_norm();
}
__device__ __forceinline__ float ld_dsmem_f1(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_smem_addr), "r"(cta_rank));
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

// ------------------------------------------------------------------ BatchNorm statistics
// sums[0:C] += sum_r x[r,c] ; sums[C:2C] += sum_r x[r,c]^2.  Block = 32 channel pairs x 8 row lanes.
__global__ void __launch_bounds__(256)
bn_stats_kernel(const __nv_bfloat162* __restrict__ x, float* __restrict__ sums, long long rows, int C) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s[4][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int C2 = C >> 1;
  const int c2 = blockIdx.x * 32 + tx;
  float a0 = 0.f, a1 = 0.f, q0 = 0.f, q1 = 0.f;
  if (c2 < C2) {
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + ty; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      const float2 v = __bfloat1622float2(x[r * C2 + c2]);
      a0 += v.x; a1 += v.y;
      q0 = fmaf(v.x, v.x, q0); q1 = fmaf(v.y, v.y, q1);
    }
  }
  s[0][ty][tx] = a0; s[1][ty][tx] = a1; s[2][ty][tx] = q0; s[3][ty][tx] = q1;
  __syncthreads();
  if (ty < 4 && c2 < C2) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += s[ty][j][tx];
    const int c = c2 * 2 + (ty & 1);
    atomicAdd(sums + (ty >> 1) * C + c, t);
  }
}

// y = relu?( gamma * (x - mean) * rstd + beta + residual? ).  Every block derives per-channel
// scale/shift from the global sums into shared memory, then streams 16-byte vectors.
__global__ void __launch_bounds__(256)
bn_apply_kernel(const uint4* __restrict__ x, const uint4* __restrict__ res, uint4* __restrict__ y,
                const float* __restrict__ sums, const float* __restrict__ gamma, const float* __restrict__ beta,
                float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ save_mean,
                float* __restrict__ save_rstd, long long* __restrict__ nbt, long long rows, int C, float eps,
                float momentum, int relu, int training) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // scale[C], shift[C]
  // the activation (and residual) do not depend on the statistics: issue this thread's first loads BEFORE the
  // scale / shift phase, so the two global round trips of this latency-bound kernel overlap instead of adding up
  const int C8 = C >> 3;
  const long long total = rows * C8;
  const long long i_first = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  uint4 xv0 = make_uint4(0u, 0u, 0u, 0u), rv0 = make_uint4(0u, 0u, 0u, 0u);
  if (i_first < total) {
    xv0 = x[i_first];
    if (res != nullptr) rv0 = res[i_first];
  }
  if (training && nbt != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *nbt += 1;  // num_batches_tracked
  float* scale = sm;
  float* shift = sm + C;
  const float inv_rows = 1.f / static_cast<float>(rows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mean, var;
    if (training) {
      mean = sums[c] * inv_rows;
      var = fmaxf(sums[C + c] * inv_rows - mean * mean, 0.f);
    } else {
      mean = running_mean[c];
      var = running_var[c];
    }
    const float rstd = rsqrtf(var + eps);
    const float g = gamma != nullptr ? gamma[c] : 1.f;
    scale[c] = g * rstd;
    shift[c] = (beta != nullptr ? beta[c] : 0.f) - mean * g * rstd;
    if (training && blockIdx.x == 0) {
      save_mean[c] = mean;
      save_rstd[c] = rstd;
      if (running_mean != nullptr) {
        const float unbiased = rows > 1 ? var * static_cast<float>(rows) / static_cast<float>(rows - 1) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      }
    }
  }
  __syncthreads();
  for (long long i = i_first; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % C8) * 8;
    uint4 xv = xv0, rv = rv0;
    if (i != i_first) {
      xv = x[i];
      if (res != nullptr) rv = res[i];
    }
    const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w};
    const uint32_t rs[4] = {rv.x, rv.y, rv.z, rv.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 p = unpack_bf16x2(xs[j]);
      const float2 q = unpack_bf16x2(rs[j]);
      float u = fmaf(p.x, scale[c0 + 2 * j], shift[c0 + 2 * j]) + q.x;
      float v = fmaf(p.y, scale[c0 + 2 * j + 1], shift[c0 + 2 * j + 1]) + q.y;
      if (relu) { u = fmaxf(u, 0.f); v = fmaxf(v, 0.f); }
      o[j] = pack_bf16x2(u, v);
    }
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// backward reduce: sums[0:C] += sum dy' ; sums[C:2C] += sum dy' * xhat   with dy' = dy * (y > 0) if relu
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const __nv_bfloat162* __restrict__ x, const __nv_bfloat162* __restrict__ y,
                     const __nv_bfloat162* __restrict__ dy, const float* __restrict__ mean,
                     const float* __restrict__ rstd, float* __restrict__ sums, long long rows, int C, int relu) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s[4][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int C2 = C >> 1;
  const int c2 = blockIdx.x * 32 + tx;
  float a0 = 0.f, a1 = 0.f, q0 = 0.f, q1 = 0.f;
  if (c2 < C2) {
    const float m0 = mean[2 * c2], m1 = mean[2 * c2 + 1], r0 = rstd[2 * c2], r1 = rstd[2 * c2 + 1];
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + ty; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      float2 g = __bfloat1622float2(dy[r * C2 + c2]);
      if (relu) {
        const float2 o = __bfloat1622float2(y[r * C2 + c2]);
        if (!(o.x > 0.f)) g.x = 0.f;
        if (!(o.y > 0.f)) g.y = 0.f;
      }
      const float2 v = __bfloat1622float2(x[r * C2 + c2]);
      a0 += g.x; a1 += g.y;
      q0 = fmaf(g.x, (v.x - m0) * r0, q0);
      q1 = fmaf(g.y, (v.y - m1) * r1, q1);
    }
  }
  s[0][ty][tx] = a0; s[1][ty][tx] = a1; s[2][ty][tx] = q0; s[3][ty][tx] = q1;
  __syncthreads();
  if (ty < 4 && c2 < C2) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += s[ty][j][tx];
    const int c = c2 * 2 + (ty & 1);
    atomicAdd(sums + (ty >> 1) * C + c, t);
  }
}

// dx = gamma * rstd * (dy' - sum_dy/rows - xhat * sum_dy_xhat/rows) ; dres = dy' ;
// block 0 accumulates dgamma += sum_dy_xhat, dbeta += sum_dy into the fp32 gradient arena.
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const uint4* __restrict__ x, const uint4* __restrict__ y, const uint4* __restrict__ dy,
                    uint4* __restrict__ dx, uint4* __restrict__ dres, const float* __restrict__ gamma,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ sums,
                    float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C, int relu) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // a[C], b[C], m[C], r[C]
  float* ka = sm;
  float* kb = sm + C;
  float* km = sm + 2 * C;
  float* kr = sm + 3 * C;
  const float inv_rows = 1.f / static_cast<float>(rows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float g = gamma != nullptr ? gamma[c] : 1.f;
    const float r = rstd[c];
    ka[c] = g * r;                       // multiplies (dy' - mean_dy - xhat * mean_dy_xhat)
    kb[c] = sums[c] * inv_rows;          // mean_dy
    km[c] = mean[c];
    kr[c] = r;
    if (blockIdx.x == 0) {
      if (dgamma != nullptr) dgamma[c] += sums[C + c];
      if (dbeta != nullptr) dbeta[c] += sums[c];
    }
  }
  __syncthreads();
  const int C8 = C >> 3;
  const long long total = rows * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % C8) * 8;
    const uint4 xv = x[i], gv = dy[i];
    const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
    uint32_t ys[4] = {0u, 0u, 0u, 0u};
    if (relu) {
      const uint4 yv = y[i];
      ys[0] = yv.x; ys[1] = yv.y; ys[2] = yv.z; ys[3] = yv.w;
    }
    uint32_t o[4], om[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 p = unpack_bf16x2(xs[j]);
      float2 g = unpack_bf16x2(gs[j]);
      if (relu) {
        const float2 q = unpack_bf16x2(ys[j]);
        if (!(q.x > 0.f)) g.x = 0.f;
        if (!(q.y > 0.f)) g.y = 0.f;
      }
      om[j] = pack_bf16x2(g.x, g.y);
      const int ca = c0 + 2 * j, cb = ca + 1;
      const float xh0 = (p.x - km[ca]) * kr[ca], xh1 = (p.y - km[cb]) * kr[cb];
      const float d0 = ka[ca] * (g.x - kb[ca] - xh0 * sums[C + ca] * inv_rows);
      const float d1 = ka[cb] * (g.y - kb[cb] - xh1 * sums[C + cb] * inv_rows);
      o[j] = pack_bf16x2(d0, d1);
    }
    dx[i] = make_uint4(o[0], o[1], o[2], o[3]);
    if (dres != nullptr) dres[i] = make_uint4(om[0], om[1], om[2], om[3]);
  }
}

// ------------------------------------------------------------------ LayerNorm (one warp per row)

// y = LN(x + residual?) * gamma + beta ; when residual is given the sum is also written to `sum_out`
// (== y's pre-norm input, needed by backward) -- here we simply recompute it in backward from x+res
// being stored by the caller, so the kernel only emits y, mean, rstd.
__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                     __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* __restrict__ mean, float* __restrict__ rstd, long long rows, int C, float eps) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __nv_bfloat16* xr = x + row * C;
  const __nv_bfloat16* rr = res != nullptr ? res + row * C : nullptr;
  float v[LN_MAX_PER_LANE];
  float s = 0.f;
  int cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) {
    float t = __bfloat162float(xr[c]);
    if (rr != nullptr) t += __bfloat162float(rr[c]);
    v[cnt] = t;
    s += t;
  }
  const float mu = warp_sum(s) / C;
  float q = 0.f;
  for (int j = 0; j < cnt; ++j) {
    const float d = v[j] - mu;
    q = fmaf(d, d, q);
  }
  const float rs = rsqrtf(warp_sum(q) / C + eps);
  __nv_bfloat16* yr = y + row * C;
  cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt)
    yr[c] = __float2bfloat16_rn((v[cnt] - mu) * rs * gamma[c] + beta[c]);
  if (lane == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
}

// x here is the pre-norm input (x + residual if a residual was fused in forward).
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                     __nv_bfloat16* __restrict__ dx, const float* __restrict__ gamma, const float* __restrict__ mean,
                     const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                     long long rows, int C) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // dgamma[C], dbeta[C] partials of this block
  float* sg = sm;
  float* sb = sm + C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { sg[c] = 0.f; sb[c] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  for (long long row = blockIdx.x * static_cast<long long>(warps) + (threadIdx.x >> 5); row < rows;
       row += static_cast<long long>(gridDim.x) * warps) {
    const __nv_bfloat16* xr = x + row * C;
    const __nv_bfloat16* gr = dy + row * C;
    const float mu = mean[row], rs = rstd[row];
    float xh[LN_MAX_PER_LANE], gg[LN_MAX_PER_LANE];
    float s1 = 0.f, s2 = 0.f;
    int cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) {
      const float h = (__bfloat162float(xr[c]) - mu) * rs;
      const float g = __bfloat162float(gr[c]);
      atomicAdd(sg + c, g * h);
      atomicAdd(sb + c, g);
      const float gw = g * gamma[c];
      xh[cnt] = h; gg[cnt] = gw;
      s1 += gw; s2 = fmaf(gw, h, s2);
    }
    s1 = warp_sum(s1) / C;
    s2 = warp_sum(s2) / C;
    __nv_bfloat16* dr = dx + row * C;
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) dr[c] = __float2bfloat16_rn(rs * (gg[cnt] - s1 - xh[cnt] * s2));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(dgamma + c, sg[c]);
    atomicAdd(dbeta + c, sb[c]);
  }
}

// ------------------------------------------------------------------ row softmax (attention probabilities)
__global__ void __launch_bounds__(256)
softmax_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long rows, int C,
                   float scale) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __nv_bfloat16* xr = x + row * C;
  float v[LN_MAX_PER_LANE];
  float m = -INFINITY;
  int cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) {
    v[cnt] = __bfloat162float(xr[c]) * scale;
    m = fmaxf(m, v[cnt]);
  }
  m = warp_max(m);
  float s = 0.f;
  for (int j = 0; j < cnt; ++j) {
    v[j] = __expf(v[j] - m);
    s += v[j];
  }
  const float inv = 1.f / warp_sum(s);
  __nv_bfloat16* yr = y + row * C;
  cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) yr[c] = __float2bfloat16_rn(v[cnt] * inv);
}
// dx = scale * y * (dy - sum(dy * y))
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                   __nv_bfloat16* __restrict__ dx, long long rows, int C, float scale) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __nv_bfloat16* yr = y + row * C;
  const __nv_bfloat16* gr = dy + row * C;
  float p[LN_MAX_PER_LANE], g[LN_MAX_PER_LANE];
  float s = 0.f;
  int cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) {
    p[cnt] = __bfloat162float(yr[c]);
    g[cnt] = __bfloat162float(gr[c]);
    s = fmaf(p[cnt], g[cnt], s);
  }
  s = warp_sum(s);
  __nv_bfloat16* dr = dx + row * C;
  cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) dr[c] = __float2bfloat16_rn(scale * p[cnt] * (g[cnt] - s));
}


// ------------------------------------------------------------------ vectorised row kernels
// A row of C elements (C % 8 == 0, C <= 1024) is owned by a group of LPR adjacent lanes (8, 16 or 32), each
// holding VPL 16-byte vectors entirely in registers: 128-bit coalesced loads/stores, no local memory, group
// reductions by xor-shuffles that stay inside the group.  LayerNorm(768) -> LPR 32 x VPL 3; attention
// softmax over 128 keys -> LPR 16 x VPL 1 (two rows per warp).

template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
layernorm_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                         __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                         float* __restrict__ mean, float* __restrict__ rstd, long long rows, int C, float eps) {
  layernorm_fwd_vec_body<LPR, VPL, false>(x, res, y, gamma, beta, mean, rstd, rows, C, eps, nullptr);
}

// persistent: every group keeps the dgamma / dbeta partials of ITS columns in registers across all the rows
// it processes; one shared-memory and one global atomic per column per block at the very end
template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
layernorm_bwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                         __nv_bfloat16* __restrict__ dx, const float* __restrict__ gamma, const float* __restrict__ mean,
                         const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                         long long rows, int C) {
  layernorm_bwd_vec_body<LPR, VPL, false>(x, dy, dx, gamma, mean, rstd, dgamma, dbeta, rows, C, nullptr);
}

template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
softmax_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long rows, int C,
                       float scale) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int RPW = 32 / LPR;
  const int gl = threadIdx.x & (LPR - 1);
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW +
                        ((threadIdx.x & 31) / LPR);
  const bool row_ok = row < rows;
  const int nvec = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (row_ok ? row : 0) * C);
  float v[VPL][8];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (row_ok && idx < nvec) {
      unpack8(__ldcs(xr + idx), v[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] *= scale;
        m = fmaxf(m, v[k][j]);
      }
    }
  }
  m = group_max<LPR>(m);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k)
    if (row_ok && gl + k * LPR < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] = __expf(v[k][j] - m);
        s += v[k][j];
      }
    }
  s = group_sum<LPR>(s);
  if (!row_ok) return;
  const float inv = 1.f / s;
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (idx < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] *= inv;
      yr[idx] = pack8(v[k]);
    }
  }
}

template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
softmax_bwd_vec_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                       __nv_bfloat16* __restrict__ dx, long long rows, int C, float scale) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int RPW = 32 / LPR;
  const int gl = threadIdx.x & (LPR - 1);
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW +
                        ((threadIdx.x & 31) / LPR);
  const bool row_ok = row < rows;
  const int nvec = C >> 3;
  const uint4* yr = reinterpret_cast<const uint4*>(y + (row_ok ? row : 0) * C);
  const uint4* gr = reinterpret_cast<const uint4*>(dy + (row_ok ? row : 0) * C);
  float p[VPL][8], g[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (row_ok && idx < nvec) {
      unpack8(__ldcs(yr + idx), p[k]);
      unpack8(__ldcs(gr + idx), g[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s = fmaf(p[k][j], g[k][j], s);
    }
  }
  s = group_sum<LPR>(s);
  if (!row_ok) return;
  uint4* dr = reinterpret_cast<uint4*>(dx + row * C);
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (idx < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = scale * p[k][j] * (g[k][j] - s);
      dr[idx] = pack8(o);
    }
  }
}



// ---- vectorised column reductions (C % 8 == 0, C/8 a power of two <= 256): a thread owns 8 adjacent
// channels (one 16-byte load per row), TPR = C/8 threads cover a row, 256/TPR rows are in flight per pass and
// every thread issues 4 independent row loads before it accumulates.  Partials meet in shared memory; one
// global atomic per channel per CTA.  (The scalar kernels above issue 16 dependent 4-byte loads per thread.)
__device__ __forceinline__ void unpack8_bn(const uint4& u, float (&f)[8]) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void colred_finish(float (&a)[8], float (&q)[8], float* sm, int tpr, int cg, int rg,
                                              float* __restrict__ sums, int C) {
  // sm: [rows_in_flight][2 * C]
  float* mine = sm + static_cast<size_t>(rg) * 2 * C + cg * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) { mine[j] = a[j]; mine[C + j] = q[j]; }
  __syncthreads();
  const int rpp = 256 / tpr;
  for (int c = threadIdx.x; c < 2 * C; c += 256) {
    float t = 0.f;
    for (int r = 0; r < rpp; ++r) t += sm[static_cast<size_t>(r) * 2 * C + c];
    atomicAdd(sums + c, t);
  }
}

__global__ void __launch_bounds__(256)
bn_stats_vec_kernel(const uint4* __restrict__ x, float* __restrict__ sums, long long rows, int C, int rows_per_cta) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];
  const int tpr = C >> 3, rpp = 256 / tpr;
  const int cg = threadIdx.x % tpr, rg = threadIdx.x / tpr;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows) r1 = rows;
  float a[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a[j] = 0.f; q[j] = 0.f; }
  for (long long r = r0 + rg; r < r1; r += 4ll * rpp) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (r + static_cast<long long>(u) * rpp < r1) v[u] = x[(r + static_cast<long long>(u) * rpp) * tpr + cg];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (r + static_cast<long long>(u) * rpp < r1) {
        float f[8];
        unpack8_bn(v[u], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) { a[j] += f[j]; q[j] = fmaf(f[j], f[j], q[j]); }
      }
  }
  colred_finish(a, q, sm, tpr, cg, rg, sums, C);
}

__global__ void __launch_bounds__(256)
bn_bwd_reduce_vec_kernel(const uint4* __restrict__ x, const uint4* __restrict__ y, const uint4* __restrict__ dy,
                         const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ sums,
                         long long rows, int C, int relu, int rows_per_cta) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];
  const int tpr = C >> 3, rpp = 256 / tpr;
  const int cg = threadIdx.x % tpr, rg = threadIdx.x / tpr;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows) r1 = rows;
  float m[8], rs[8], a[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { m[j] = mean[cg * 8 + j]; rs[j] = rstd[cg * 8 + j]; a[j] = 0.f; q[j] = 0.f; }
  for (long long r = r0 + rg; r < r1; r += 2ll * rpp) {
    uint4 xv[2], gv[2], yv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long rr = r + static_cast<long long>(u) * rpp;
      if (rr < r1) {
        xv[u] = x[rr * tpr + cg];
        gv[u] = dy[rr * tpr + cg];
        if (relu) yv[u] = y[rr * tpr + cg];
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (r + static_cast<long long>(u) * rpp < r1) {
        float xf[8], gf[8];
        unpack8_bn(xv[u], xf);
        unpack8_bn(gv[u], gf);
        if (relu) {
          float yf[8];
          unpack8_bn(yv[u], yf);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (!(yf[j] > 0.f)) gf[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          a[j] += gf[j];
          q[j] = fmaf(gf[j], (xf[j] - m[j]) * rs[j], q[j]);
        }
      }
    }
  }
  colred_finish(a, q, sm, tpr, cg, rg, sums, C);
}


// ---- BatchNorm backward in ONE kernel, cluster edition (default path) ------------------------------------------
// A thread-block CLUSTER owns a 16-channel slice of the [rows, C] activation (32 B = one sector per row and tensor)
// and splits the rows between its CTAs.  Every thread reads its (x, y, dy) pieces ONCE and keeps them in
// registers; the per-channel sums (sum dy', sum dy' * xhat) are reduced warp -> CTA (shared memory) -> cluster
// (distributed shared memory, fixed order: deterministic), and after one cluster barrier the same registers produce
// dx (and dres = dy').  No device-wide barrier (the channel slices are independent), no second pass over global
// memory, no workspace: the two-kernel reduce + apply pair becomes one launch.
// The gradient may arrive in TWO pieces (dy = dy_a + dy_b): a ResNet block input receives the main-branch dgrad and
// the residual-branch gradient, and summing them here removes the separate add kernel.
constexpr int BNC_CW = 16;        // channels per cluster
constexpr int BNC_LANES = 128;    // row lanes per CTA (256 threads = 128 rows x 2 sixteen-byte chunks)

template <int ITER>
__global__ void __launch_bounds__(256)
bn_bwd_cluster_kernel(const uint4* __restrict__ x, const uint4* __restrict__ y, const uint4* __restrict__ dy_a,
                      const uint4* __restrict__ dy_b, uint4* __restrict__ dx, uint4* __restrict__ dres,
                      const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                      float* __restrict__ dgamma, float* __restrict__ dbeta, int rows, int C, int relu, int rows_per_cta) {
  griddep_launch_dependents();
  __shared__ float wpart[8][2][16];          // per-warp partials: [warp][chunk][8 x {sum_g, sum_gx}]
  __shared__ __align__(16) float cpart[32];  // this CTA's partial: [0:16) sum_g, [16:32) sum_gx per channel of the slice
  __shared__ float tot[32];
  const int chunk = threadIdx.x & 1, lane_r = threadIdx.x >> 1;
  const int c0 = blockIdx.x * BNC_CW + chunk * 8;            // first of this thread's 8 channels
  const int C8 = C >> 3;
  const uint32_t S = cluster_nctarank_y();
  const uint32_t me = cluster_ctarank_any();
  const int r_begin = static_cast<int>(me) * rows_per_cta;
  int r_end = r_begin + rows_per_cta;
  if (r_end > rows) r_end = rows;
  // mean / rstd come from the forward pass, but only the wait is transitive: the grid that wrote them may still run
  griddep_wait();
  float m[8], rs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { m[j] = mean[c0 + j]; rs[j] = rstd[c0 + j]; }
  constexpr int NC = ITER > 0 ? ITER : 1;          // ITER == 0: rows are NOT cached (any row count): second pass re-reads
  float xh[NC][8], g[NC][8];
  float sg[8], sgx[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sg[j] = 0.f; sgx[j] = 0.f; }
  auto load_row = [&](int r, float (&xh_)[8], float (&g_)[8]) {
    const long long i = static_cast<long long>(r) * C8 + (c0 >> 3);
    float xf[8];
    unpack8_bn(x[i], xf);
    unpack8_bn(dy_a[i], g_);
    if (dy_b != nullptr) {
      float t[8];
      unpack8_bn(dy_b[i], t);
#pragma unroll
      for (int j = 0; j < 8; ++j) g_[j] += t[j];
    }
    if (relu) {
      float yf[8];
      unpack8_bn(y[i], yf);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (!(yf[j] > 0.f)) g_[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) xh_[j] = (xf[j] - m[j]) * rs[j];
  };
  if constexpr (ITER > 0) {
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
      const int r = r_begin + it * BNC_LANES + lane_r;
      if (r < r_end) {
        load_row(r, xh[it], g[it]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sg[j] += g[it][j];
          sgx[j] = fmaf(g[it][j], xh[it][j], sgx[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { xh[it][j] = 0.f; g[it][j] = 0.f; }
      }
    }
  } else {
    for (int r = r_begin + lane_r; r < r_end; r += BNC_LANES) {
      load_row(r, xh[0], g[0]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        sg[j] += g[0][j];
        sgx[j] = fmaf(g[0][j], xh[0][j], sgx[j]);
      }
    }
  }
  // warp reduce over the 16 row lanes that share this chunk (lane bit 0 = chunk); the 16 chains are independent, so
  // each round issues all of them before the next round needs their results
#pragma unroll
  for (int o = 2; o < 32; o <<= 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sg[j] += __shfl_xor_sync(0xffffffffu, sg[j], o);
      sgx[j] += __shfl_xor_sync(0xffffffffu, sgx[j], o);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      wpart[warp][lane][j] = sg[j];
      wpart[warp][lane][8 + j] = sgx[j];
    }
  }
  __syncthreads();
  if (threadIdx.x < 32) {      // thread t: chunk = (t >> 3) & 1, j = t & 7, kind = t >> 4
    const int kind = threadIdx.x >> 4, ch = (threadIdx.x >> 3) & 1, j = threadIdx.x & 7;
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += wpart[w][ch][kind * 8 + j];
    cpart[kind * 16 + ch * 8 + j] = t;
  }
  if (S > 1) {
    cluster_sync_all_norm();
  } else {
    __syncthreads();
  }
  if (threadIdx.x < 32) {
    float t = 0.f;
    const uint32_t laddr = smem_u32(&cpart[threadIdx.x]);
    for (uint32_t r = 0; r < S; ++r) t += (S > 1) ? ld_dsmem_f1(laddr, r) : cpart[threadIdx.x];
    tot[threadIdx.x] = t;
    if (me == 0) {             // one CTA per slice owns the parameter gradients of its 16 channels
      const int c = blockIdx.x * BNC_CW + (threadIdx.x & 15);
      if (threadIdx.x < 16) {
        if (dbeta != nullptr) dbeta[c] += t;
      } else if (dgamma != nullptr) {
        dgamma[c] += t;
      }
    }
  }
  __syncthreads();
  if (S > 1) cluster_arrive_norm();          // peers may exit once everybody has read everybody's partials
  const float inv_rows = 1.f / static_cast<float>(rows);
  float ka[8], kb[8], kc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    ka[j] = (gamma != nullptr ? gamma[c0 + j] : 1.f) * rs[j];
    kb[j] = tot[chunk * 8 + j] * inv_rows;
    kc[j] = tot[16 + chunk * 8 + j] * inv_rows;
  }
  auto store_row = [&](int r, const float (&xh_)[8], const float (&g_)[8]) {
    const long long i = static_cast<long long>(r) * C8 + (c0 >> 3);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = ka[j] * (g_[j] - kb[j] - xh_[j] * kc[j]);
    dx[i] = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
    if (dres != nullptr)
      dres[i] = make_uint4(pack_bf16x2(g_[0], g_[1]), pack_bf16x2(g_[2], g_[3]), pack_bf16x2(g_[4], g_[5]),
                           pack_bf16x2(g_[6], g_[7]));
  };
  if constexpr (ITER > 0) {
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
      const int r = r_begin + it * BNC_LANES + lane_r;
      if (r < r_end) store_row(r, xh[it], g[it]);
    }
  } else {
    for (int r = r_begin + lane_r; r < r_end; r += BNC_LANES) {      // second pass: the slab is L2 (often L1) resident
      load_row(r, xh[0], g[0]);
      store_row(r, xh[0], g[0]);
    }
  }
  if (S > 1) cluster_wait_norm();
}

static inline bool colred_vec_ok(int C, const void* p0, const void* p1, const void* p2) {
  const int tpr = C >> 3;
  return C % 8 == 0 && tpr >= 1 && tpr <= 256 && (tpr & (tpr - 1)) == 0 &&
         ((reinterpret_cast<uintptr_t>(p0) | reinterpret_cast<uintptr_t>(p1) | reinterpret_cast<uintptr_t>(p2)) & 15) == 0;
}
// rows handled by one CTA: a multiple of the rows in flight per pass, ~2 CTAs per SM at most
static inline int colred_rows_per_cta(long long rows, int C, int unroll) {
  const int rpp = 256 / (C >> 3);
  long long per = (rows + 295) / 296;
  per = (per + rpp - 1) / rpp * rpp;
  if (per < rpp) per = rpp;
  const long long cap = static_cast<long long>(rpp) * unroll * 4;
  if (per > cap) per = cap;      // beyond this, more CTAs simply queue: still one short pass each
  return static_cast<int>(per);
}

static inline dim3 colred_grid(long long rows, int C) {
  long long gy = (rows + 127) / 128;
  if (gy > device_sm_count()) gy = device_sm_count();
  if (gy < 1) gy = 1;
  return dim3((C / 2 + 31) / 32, static_cast<unsigned>(gy));
}
// ------------------------------------------------------------------ ResNet stem: BatchNorm + ReLU + max-pool fused
// The stem's normalised activation y = relu(bn(z)) (32768 x 64 for 32x32 inputs) is only ever consumed by the 3x3/2
// max-pool, and the backward pass needs it only as the ReLU mask at the pooled maxima -- which the pooled output itself
// carries (p > 0  <=>  y > 0 at the argmax).  So y is never materialised:
//   forward : p, argmax = maxpool(relu(scale * z + shift))                       (one kernel instead of two, -8 MB)
//   backward: the per-channel sums of BatchNorm's backward run over the POOLED gradient (4x fewer rows; z is gathered
//             at the argmax), and the apply pass gathers the pooled gradient while it writes dz (no dense dy).
// Candidates are rounded to bf16 before they are compared, so p / argmax are bit-identical to bn_apply + maxpool.
__global__ void __launch_bounds__(256)
bn_relu_maxpool_kernel(const uint4* __restrict__ z, uint4* __restrict__ p, uint2* __restrict__ arg,
                       const float* __restrict__ sums, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ save_mean,
                       float* __restrict__ save_rstd, long long* __restrict__ nbt, int N, int H, int W, int C, int k,
                       int stride, int pad, int Ho, int Wo, float eps, float momentum) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // scale[C], shift[C]
  float* scale = sm;
  float* shift = sm + C;
  const long long rows = static_cast<long long>(N) * H * W;
  if (nbt != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *nbt += 1;
  const float inv_rows = 1.f / static_cast<float>(rows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float mean = sums[c] * inv_rows;
    const float var = fmaxf(sums[C + c] * inv_rows - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    const float g = gamma != nullptr ? gamma[c] : 1.f;
    scale[c] = g * rstd;
    shift[c] = (beta != nullptr ? beta[c] : 0.f) - mean * g * rstd;
    if (blockIdx.x == 0) {
      save_mean[c] = mean;
      save_rstd[c] = rstd;
      if (running_mean != nullptr) {
        const float unbiased = rows > 1 ? var * static_cast<float>(rows) / static_cast<float>(rows - 1) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      }
    }
  }
  __syncthreads();
  const int C8 = C >> 3;
  const long long total = static_cast<long long>(N) * Ho * Wo * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % C8);
    long long t = i / C8;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    float sc[8], sh[8], m[8];
    uint32_t a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = scale[c8 * 8 + j]; sh[j] = shift[c8 * 8 + j]; m[j] = -INFINITY; a[j] = 255u; }
    for (int kh = 0; kh < k; ++kh) {
      const int h = ho * stride - pad + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int w = wo * stride - pad + kw;
        if (w < 0 || w >= W) continue;
        float f[8];
        unpack8_bn(z[((static_cast<long long>(n) * H + h) * W + w) * C8 + c8], f);
        const uint32_t tap = static_cast<uint32_t>(kh * k + kw);
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          const float2 y = unpack_bf16x2(pack_bf16x2(fmaxf(fmaf(f[j], sc[j], sh[j]), 0.f),
                                                     fmaxf(fmaf(f[j + 1], sc[j + 1], sh[j + 1]), 0.f)));
          if (y.x > m[j]) { m[j] = y.x; a[j] = tap; }
          if (y.y > m[j + 1]) { m[j + 1] = y.y; a[j + 1] = tap; }
        }
      }
    }
    p[i] = make_uint4(pack_bf16x2(m[0], m[1]), pack_bf16x2(m[2], m[3]), pack_bf16x2(m[4], m[5]), pack_bf16x2(m[6], m[7]));
    arg[i] = make_uint2(a[0] | (a[1] << 8) | (a[2] << 16) | (a[3] << 24), a[4] | (a[5] << 8) | (a[6] << 16) | (a[7] << 24));
  }
}

// sums[0:C] += sum_o g[o, c] ;  sums[C:2C] += sum_o g[o, c] * xhat(z at the argmax of o),   g = (dy_a + dy_b) * (p > 0),
// over the pooled positions o.  Same thread layout / reduction as bn_bwd_reduce_vec_kernel.
__global__ void __launch_bounds__(256)
bn_maxpool_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ z, const uint4* __restrict__ p, const uint2* __restrict__ arg,
                             const uint4* __restrict__ dy_a, const uint4* __restrict__ dy_b,
                             const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ sums,
                             int N, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int rows_per_cta) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];
  const int tpr = C >> 3, rpp = 256 / tpr;
  const int cg = threadIdx.x % tpr, rg = threadIdx.x / tpr;
  const long long rows = static_cast<long long>(N) * Ho * Wo;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows) r1 = rows;
  float m[8], rs[8], a[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { m[j] = mean[cg * 8 + j]; rs[j] = rstd[cg * 8 + j]; a[j] = 0.f; q[j] = 0.f; }
  for (long long r = r0 + rg; r < r1; r += rpp) {
    const long long o = r * tpr + cg;
    const uint2 av = arg[o];
    float g[8], pf[8];
    unpack8_bn(dy_a[o], g);
    unpack8_bn(p[o], pf);
    if (dy_b != nullptr) {
      float gb[8];
      unpack8_bn(dy_b[o], gb);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] += gb[j];
    }
    const int wo = static_cast<int>(r % Wo);
    const long long t = r / Wo;
    const int ho = static_cast<int>(t % Ho);
    const long long n = t / Ho;
    const int hb = ho * stride - pad, wb = wo * stride - pad;
    float zf[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int tap = static_cast<int>(((j < 4 ? av.x : av.y) >> (8 * (j & 3))) & 0xffu);
      const int kh = tap / k, kw = tap - kh * k;
      zf[j] = 0.f;
      if (pf[j] > 0.f) zf[j] = __bfloat162float(z[((n * H + (hb + kh)) * W + (wb + kw)) * C + cg * 8 + j]);
      else g[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      a[j] += g[j];
      q[j] = fmaf(g[j], (zf[j] - m[j]) * rs[j], q[j]);
    }
  }
  colred_finish(a, q, sm, tpr, cg, rg, sums, C);
}

// dz = gamma * rstd * (g_dense - mean_g - xhat * mean_gx) with g_dense[n, h, w, c] = the pooled gradient of every window
// whose argmax is (h, w) (ReLU-masked through p > 0), gathered on the fly; block 0 accumulates dgamma / dbeta.
__global__ void __launch_bounds__(256)
bn_maxpool_bwd_apply_kernel(const uint4* __restrict__ z, const uint4* __restrict__ p, const uint2* __restrict__ arg,
                            const uint4* __restrict__ dy_a, const uint4* __restrict__ dy_b, uint4* __restrict__ dz,
                            const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                            const float* __restrict__ sums, float* __restrict__ dgamma, float* __restrict__ dbeta, int N,
                            int H, int W, int C, int k, int stride, int pad, int Ho, int Wo) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ float sm[];  // a[C], b[C], m[C], r[C], s[C]
  float* ka = sm;
  float* kb = sm + C;
  float* km = sm + 2 * C;
  float* kr = sm + 3 * C;
  float* ks = sm + 4 * C;
  const long long rows = static_cast<long long>(N) * H * W;
  const float inv_rows = 1.f / static_cast<float>(rows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float g = gamma != nullptr ? gamma[c] : 1.f;
    const float r = rstd[c];
    ka[c] = g * r;
    kb[c] = sums[c] * inv_rows;          // mean of the (dense) gradient
    km[c] = mean[c];
    kr[c] = r;
    ks[c] = sums[C + c] * inv_rows;      // mean of gradient * xhat
    if (blockIdx.x == 0) {
      if (dgamma != nullptr) dgamma[c] += sums[C + c];
      if (dbeta != nullptr) dbeta[c] += sums[c];
    }
  }
  __syncthreads();
  const int C8 = C >> 3;
  const long long total = rows * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % C8);
    long long t = i / C8;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    float xf[8];
    unpack8_bn(z[i], xf);
    float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int kh = 0; kh < k; ++kh) {
      const int hh = h + pad - kh;
      if (hh < 0 || hh % stride) continue;
      const int ho = hh / stride;
      if (ho >= Ho) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int ww = w + pad - kw;
        if (ww < 0 || ww % stride) continue;
        const int wo = ww / stride;
        if (wo >= Wo) continue;
        const long long o = ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * C8 + c8;
        const uint2 av = arg[o];
        float f[8], pf[8];
        unpack8_bn(dy_a[o], f);
        unpack8_bn(p[o], pf);
        if (dy_b != nullptr) {
          float fb[8];
          unpack8_bn(dy_b[o], fb);
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] += fb[j];
        }
        const uint32_t tap = static_cast<uint32_t>(kh * k + kw);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t aj = ((j < 4 ? av.x : av.y) >> (8 * (j & 3))) & 0xffu;
          if (aj == tap && pf[j] > 0.f) g[j] += f[j];
        }
      }
    }
    uint32_t o4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ca = c8 * 8 + 2 * j, cb = ca + 1;
      const float xh0 = (xf[2 * j] - km[ca]) * kr[ca], xh1 = (xf[2 * j + 1] - km[cb]) * kr[cb];
      o4[j] = pack_bf16x2(ka[ca] * (g[2 * j] - kb[ca] - xh0 * ks[ca]), ka[cb] * (g[2 * j + 1] - kb[cb] - xh1 * ks[cb]));
    }
    dz[i] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
  }
}

// Eval-mode BatchNorm folding: block b turns BatchNorm b into the per-channel scale / shift of bn_apply_kernel's eval
// branch (same expressions), read from the parameter arena.  table[b] = {gamma, beta, running_mean, running_var,
// output offset, C, eps bits}; the first four are element offsets into `arena`, gamma / beta may be -1 (affine=False).
// out[off .. off + C) = scale, out[off + C .. off + 2C) = shift.
__global__ void __launch_bounds__(256)
bn_fold_eval_kernel(const float* __restrict__ arena, const long long* __restrict__ table, float* __restrict__ out) {
  griddep_launch_dependents();
  griddep_wait();
  const long long* t = table + static_cast<size_t>(blockIdx.x) * 7;
  const long long go = t[0], bo = t[1], mo = t[2], vo = t[3], oo = t[4];
  const int C = static_cast<int>(t[5]);
  const float eps = __int_as_float(static_cast<int>(t[6]));
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float mean = arena[mo + c];
    const float var = arena[vo + c];
    const float rstd = rsqrtf(var + eps);
    const float g = go >= 0 ? arena[go + c] : 1.f;
    out[oo + c] = g * rstd;
    out[oo + C + c] = (bo >= 0 ? arena[bo + c] : 0.f) - mean * g * rstd;
  }
}

// ------------------------------------------------------------------ GroupNorm (+residual +ReLU)
// NHWC bf16 [N, HW, C] with G groups of Cg = C / G contiguous channels: group (n, g) is the HW x Cg block of sample n,
// M = HW * Cg elements.  One CTA per (n, g), blockIdx.x = n * G + g.  Statistics in fp32: the mean, then the biased
// variance from centred values (post-ReLU inputs have large means, so E[x^2] - E[x]^2 would cancel).
//   forward : y = relu?(gamma_c * (z - mean) * rstd + beta_c + residual?), saves mean / rstd [N, G]
//   backward: dy' = (dy_a + dy_b?) * (y > 0 if relu), dres = dy',
//             dz = rstd * (gamma_c dy' - mean(gamma dy') - xhat * mean(gamma dy' xhat)),
//             dgamma_c += sum_{n,hw} dy' xhat, dbeta_c += sum_{n,hw} dy'.
// CACHE: the (n, g) block is kept in shared memory (z as bf16, and dy' as fp32 in the backward), so global memory is read
// once and written once; otherwise (ResNet stems of large images) every pass re-reads global memory.  Every sum has a
// fixed order for a given shape: shuffle trees, warp partials in index order, and for the per-channel parameter
// gradients (which cross samples) per-CTA partials that the last CTA of each group adds in sample order -- the same bits
// on every launch, with no float atomics.  work: fp32 [G + 2 N C]; words [0, G) are per-group arrival counters that the
// forward zeroes and the backward leaves zero, then the [N][C][2] partials.
constexpr int GN_THREADS = 256;
constexpr long long GN_CACHE_ELEMS = 16384;      // one (n, g) block on chip: 32 KB forward, 96 KB backward

template <int W>
__device__ __forceinline__ void gn_ld(const __nv_bfloat16* p, float (&f)[W]) {
  if constexpr (W == 8) {
    unpack8_bn(*reinterpret_cast<const uint4*>(p), f);
  } else {
#pragma unroll
    for (int j = 0; j < W; ++j) f[j] = __bfloat162float(p[j]);
  }
}
template <int W>
__device__ __forceinline__ void gn_st(__nv_bfloat16* p, const float (&f)[W]) {
  if constexpr (W == 8) {
    *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                                              pack_bf16x2(f[6], f[7]));
  } else {
#pragma unroll
    for (int j = 0; j < W; ++j) p[j] = __float2bfloat16_rn(f[j]);
  }
}
// x and the masked gradient dy' of W consecutive channels at element offset o
template <int W>
__device__ __forceinline__ void gn_grad(long long o, const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ y,
                                        const __nv_bfloat16* __restrict__ dy_a, const __nv_bfloat16* __restrict__ dy_b,
                                        int relu, float (&xf)[W], float (&gf)[W]) {
  gn_ld<W>(z + o, xf);
  gn_ld<W>(dy_a + o, gf);
  if (dy_b != nullptr) {
    float t[W];
    gn_ld<W>(dy_b + o, t);
#pragma unroll
    for (int j = 0; j < W; ++j) gf[j] += t[j];
  }
  if (relu) {
    float yf[W];
    gn_ld<W>(y + o, yf);
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (!(yf[j] > 0.f)) gf[j] = 0.f;
  }
}
// CTA-wide sum in a fixed order; every thread receives it.  `red`: GN_THREADS / 32 floats of shared memory.
__device__ __forceinline__ float gn_cta_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                 // a previous call may still be reading red
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < GN_THREADS / 32; ++w) t += red[w];
  return t;
}

template <int VEC, bool CACHE>
__global__ void __launch_bounds__(GN_THREADS)
gn_fwd_kernel(const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ res, __nv_bfloat16* __restrict__ y,
              const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, unsigned* __restrict__ counters, long long HW, int C, int G, float eps,
              int relu) {
  griddep_launch_dependents();
  extern __shared__ __align__(16) unsigned char gn_smem[];
  __nv_bfloat16* zc = reinterpret_cast<__nv_bfloat16*>(gn_smem);    // [M] when CACHE
  __shared__ float red[GN_THREADS / 32];
  const int g = static_cast<int>(blockIdx.x % G);
  const long long n = blockIdx.x / G;
  const int Cg = C / G, CgV = Cg / VEC;
  const long long M = HW * Cg, MV = M / VEC;
  const long long base = n * HW * C + static_cast<long long>(g) * Cg;
  griddep_wait();
  float s = 0.f;
  for (long long v = threadIdx.x; v < MV; v += GN_THREADS) {
    float f[VEC];
    gn_ld<VEC>(z + base + (v / CgV) * C + (v % CgV) * VEC, f);
    if constexpr (CACHE) gn_st<VEC>(zc + v * VEC, f);
#pragma unroll
    for (int j = 0; j < VEC; ++j) s += f[j];
  }
  const float fm = static_cast<float>(M);
  const float mean = __fdiv_rn(gn_cta_sum(s, red), fm);
  float q = 0.f;
  for (long long v = threadIdx.x; v < MV; v += GN_THREADS) {
    float f[VEC];
    gn_ld<VEC>(CACHE ? zc + v * VEC : z + base + (v / CgV) * C + (v % CgV) * VEC, f);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d = f[j] - mean;
      q = fmaf(d, d, q);
    }
  }
  const float var = __fdiv_rn(gn_cta_sum(q, red), fm);
  const float rstd = rsqrtf(var + eps);
  if (threadIdx.x == 0) {
    mean_out[blockIdx.x] = mean;
    rstd_out[blockIdx.x] = rstd;
    if (counters != nullptr && n == 0) counters[g] = 0u;
  }
  for (long long v = threadIdx.x; v < MV; v += GN_THREADS) {
    const long long o = base + (v / CgV) * C + (v % CgV) * VEC;
    const int c0 = g * Cg + static_cast<int>(v % CgV) * VEC;
    float f[VEC], r[VEC];
    gn_ld<VEC>(CACHE ? zc + v * VEC : z + o, f);
    if (res != nullptr) {
      gn_ld<VEC>(res + o, r);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) r[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      float u = fmaf(gamma[c0 + j], (f[j] - mean) * rstd, beta[c0 + j]) + r[j];
      if (relu) u = fmaxf(u, 0.f);
      f[j] = u;
    }
    gn_st<VEC>(y + o, f);
  }
}

template <int VEC, bool CACHE>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_kernel(const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ y,
              const __nv_bfloat16* __restrict__ dy_a, const __nv_bfloat16* __restrict__ dy_b, __nv_bfloat16* __restrict__ dz,
              __nv_bfloat16* __restrict__ dres, const float* __restrict__ gamma, const float* __restrict__ mean_in,
              const float* __restrict__ rstd_in, float* __restrict__ dgamma, float* __restrict__ dbeta,
              float* __restrict__ work, long long HW, int C, int G, int relu) {
  griddep_launch_dependents();
  extern __shared__ __align__(16) unsigned char gn_smem[];
  const int g = static_cast<int>(blockIdx.x % G);
  const long long n = blockIdx.x / G;
  const int N = static_cast<int>(gridDim.x / G);
  const int Cg = C / G, CgV = Cg / VEC;
  const long long M = HW * Cg, MV = M / VEC;
  float* gc = reinterpret_cast<float*>(gn_smem);                               // [M] dy' when CACHE
  __nv_bfloat16* zc = reinterpret_cast<__nv_bfloat16*>(gn_smem + M * 4);     // [M] z when CACHE
  __shared__ float red[GN_THREADS / 32];
  __shared__ float part[2][GN_THREADS];
  __shared__ bool last;
  const long long base = n * HW * C + static_cast<long long>(g) * Cg;
  unsigned* counters = reinterpret_cast<unsigned*>(work);
  float* partials = work + G;                                                   // [N][C][2]: sum dy', sum dy' xhat
  griddep_wait();
  const float mean = mean_in[blockIdx.x], rstd = rstd_in[blockIdx.x];
  // pass 1: dy' -> dres, and the on-chip copy
  if (CACHE || dres != nullptr) {
    for (long long v = threadIdx.x; v < MV; v += GN_THREADS) {
      const long long o = base + (v / CgV) * C + (v % CgV) * VEC;
      float xf[VEC], gf[VEC];
      gn_grad<VEC>(o, z, y, dy_a, dy_b, relu, xf, gf);
      if (dres != nullptr) gn_st<VEC>(dres + o, gf);
      if constexpr (CACHE) {
        gn_st<VEC>(zc + v * VEC, xf);
#pragma unroll
        for (int j = 0; j < VEC; ++j) gc[v * VEC + j] = gf[j];
      }
    }
    if constexpr (CACHE) __syncthreads();
  }
  // per-channel sums over the HW positions of this sample: `span` channels at a time, each summed by `ns` threads over
  // interleaved positions, then the ns partials in slice order.  Their gamma-weighted totals are mean(gamma dy') etc.
  float ga = 0.f, gb = 0.f;
  for (int cb = 0; cb < Cg; cb += GN_THREADS) {
    const int span = min(Cg - cb, GN_THREADS), ns = GN_THREADS / span;
    const int cl = cb + static_cast<int>(threadIdx.x) % span, sl = static_cast<int>(threadIdx.x) / span;
    float sg = 0.f, sgx = 0.f;
    if (sl < ns) {
      for (long long p = sl; p < HW; p += ns) {
        float xf[1], gf[1];
        if constexpr (CACHE) {
          xf[0] = __bfloat162float(zc[p * Cg + cl]);
          gf[0] = gc[p * Cg + cl];
        } else {
          gn_grad<1>(base + p * C + cl, z, y, dy_a, dy_b, relu, xf, gf);
        }
        sg += gf[0];
        sgx = fmaf(gf[0], (xf[0] - mean) * rstd, sgx);
      }
    }
    __syncthreads();               // the previous block of channels may still be reading part
    part[0][threadIdx.x] = sg;
    part[1][threadIdx.x] = sgx;
    __syncthreads();
    if (static_cast<int>(threadIdx.x) < span) {
      float a = 0.f, b = 0.f;
      for (int k = 0; k < ns; ++k) {
        a += part[0][k * span + threadIdx.x];
        b += part[1][k * span + threadIdx.x];
      }
      const int c = g * Cg + cb + static_cast<int>(threadIdx.x);
      partials[(n * C + c) * 2] = a;
      partials[(n * C + c) * 2 + 1] = b;
      ga = fmaf(gamma[c], a, ga);
      gb = fmaf(gamma[c], b, gb);
    }
  }
  const float fm = static_cast<float>(M);
  const float ka = __fdiv_rn(gn_cta_sum(ga, red), fm), kb = __fdiv_rn(gn_cta_sum(gb, red), fm);
  // pass 2: dz
  for (long long v = threadIdx.x; v < MV; v += GN_THREADS) {
    const long long o = base + (v / CgV) * C + (v % CgV) * VEC;
    const int c0 = g * Cg + static_cast<int>(v % CgV) * VEC;
    float xf[VEC], gf[VEC];
    if constexpr (CACHE) {
      gn_ld<VEC>(zc + v * VEC, xf);
#pragma unroll
      for (int j = 0; j < VEC; ++j) gf[j] = gc[v * VEC + j];
    } else {
      gn_grad<VEC>(o, z, y, dy_a, dy_b, relu, xf, gf);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) xf[j] = rstd * (gamma[c0 + j] * gf[j] - ka - (xf[j] - mean) * rstd * kb);
    gn_st<VEC>(dz + o, xf);
  }
  // dgamma / dbeta: the last CTA of group g to arrive adds the N partials of each of its channels in sample order
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(counters + g, 1u) == static_cast<unsigned>(N - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int c = g * Cg + static_cast<int>(threadIdx.x); c < (g + 1) * Cg; c += GN_THREADS) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < N; ++k) {
      a += __ldcg(partials + (static_cast<long long>(k) * C + c) * 2);
      b += __ldcg(partials + (static_cast<long long>(k) * C + c) * 2 + 1);
    }
    if (dbeta != nullptr) dbeta[c] += a;
    if (dgamma != nullptr) dgamma[c] += b;
  }
  if (threadIdx.x == 0) counters[g] = 0u;
}

static inline int stream_grid(long long nvec) {
  long long g = (nvec + 255) / 256;
  if (g < 1) g = 1;
  if (g > device_sm_count() * 4) g = device_sm_count() * 4;
  return static_cast<int>(g);
}

}  // namespace b200

using namespace b200;
#define RET_LAST() return static_cast<int>(cudaGetLastError())

extern "C" int b200_bn_fold_eval(const float* arena, const long long* table, int n_bn, float* out, cudaStream_t stream) {
  if (n_bn <= 0) return 0;
  launch_pdl(bn_fold_eval_kernel, n_bn, 256, 0, stream, arena, table, out);
  RET_LAST();
}

extern "C" int b200_bn_stats(const void* x, float* sums, long long rows, int C, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C % 2) return -2;
  if (colred_vec_ok(C, x, nullptr, nullptr)) {
    const int rpc = colred_rows_per_cta(rows, C, 4);
    launch_pdl(bn_stats_vec_kernel, static_cast<unsigned>((rows + rpc - 1) / rpc), 256, 256 * 16 * sizeof(float), stream,
               reinterpret_cast<const uint4*>(x), sums, rows, C, rpc);
    RET_LAST();
  }
  launch_pdl(bn_stats_kernel, colred_grid(rows, C), 256, 0, stream, reinterpret_cast<const __nv_bfloat162*>(x), sums, rows, C);
  RET_LAST();
}
extern "C" int b200_bn_apply(const void* x, const void* residual, void* y, float* sums, const float* gamma,
                             const float* beta, float* running_mean, float* running_var, float* save_mean,
                             float* save_rstd, long long* nbt, long long rows, int C, float eps, float momentum,
                             int relu, int training, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C % 8) return -2;
  launch_pdl(bn_apply_kernel, stream_grid(rows * (C / 8)), 256, 2 * C * sizeof(float), stream, 
      reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(residual), reinterpret_cast<uint4*>(y), sums,
      gamma, beta, running_mean, running_var, save_mean, save_rstd, nbt, rows, C, eps, momentum, relu, training);
  RET_LAST();
}
extern "C" int b200_bn_bwd_reduce(const void* x, const void* y, const void* dy, const float* save_mean,
                                  const float* save_rstd, float* sums, long long rows, int C, int relu,
                                  cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C % 2) return -2;
  if (colred_vec_ok(C, x, relu ? y : nullptr, dy)) {
    const int rpc = colred_rows_per_cta(rows, C, 2);
    launch_pdl(bn_bwd_reduce_vec_kernel, static_cast<unsigned>((rows + rpc - 1) / rpc), 256, 256 * 16 * sizeof(float),
               stream, reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(y),
               reinterpret_cast<const uint4*>(dy), save_mean, save_rstd, sums, rows, C, relu, rpc);
    RET_LAST();
  }
  launch_pdl(bn_bwd_reduce_kernel, colred_grid(rows, C), 256, 0, stream, 
      reinterpret_cast<const __nv_bfloat162*>(x), reinterpret_cast<const __nv_bfloat162*>(y),
      reinterpret_cast<const __nv_bfloat162*>(dy), save_mean, save_rstd, sums, rows, C, relu);
  RET_LAST();
}
extern "C" int b200_bn_bwd_apply(const void* x, const void* y, const void* dy, void* dx, void* dres, const float* gamma,
                                 const float* save_mean, const float* save_rstd, float* sums, float* dgamma,
                                 float* dbeta, long long rows, int C, int relu, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C % 8) return -2;
  const size_t smem = 4 * C * sizeof(float);     // above the 48 KB default from C = 3080 (shapes the cluster kernel declines)
  if (smem > 48 * 1024) cudaFuncSetAttribute(bn_bwd_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  launch_pdl(bn_bwd_apply_kernel, stream_grid(rows * (C / 8)), 256, smem, stream,
      reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(y), reinterpret_cast<const uint4*>(dy),
      reinterpret_cast<uint4*>(dx), reinterpret_cast<uint4*>(dres), gamma, save_mean, save_rstd, sums, dgamma, dbeta,
      rows, C, relu);
  RET_LAST();
}
// one launch of the cluster BatchNorm backward with clusters of S CTAs along y; returns -2 when S > 8 and the device
// does not allow that non-portable cluster size (the caller then uses the two-kernel path).
template <int ITER>
static int launch_bn_bwd_cluster(dim3 grid, int S, cudaStream_t stream, const uint4* x, const uint4* y, const uint4* dy_a,
                                 const uint4* dy_b, uint4* dx, uint4* dres, const float* gamma, const float* mean,
                                 const float* rstd, float* dgamma, float* dbeta, int rows, int C, int relu, int rpc) {
  static int np16 = -1;      // may clusters of 16 CTAs be used?  (non-portable size: opt-in per function)
  if (np16 < 0) {
    np16 = cudaFuncSetAttribute(bn_bwd_cluster_kernel<ITER>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess;
    cudaGetLastError();
  }
  if (S > 8 && !np16) return -2;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (S > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = 1;
    attr[na].val.clusterDim.y = static_cast<unsigned>(S);
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, bn_bwd_cluster_kernel<ITER>, x, y, dy_a, dy_b, dx, dres, gamma, mean, rstd, dgamma,
                                     dbeta, rows, C, relu, rpc);
  if (e != cudaSuccess) return static_cast<int>(e);
  return static_cast<int>(cudaGetLastError());
}

// Single-kernel BatchNorm backward (cluster per 16-channel slice).  dy = dy_a (+ dy_b); dgamma / dbeta are
// ACCUMULATED.  Returns -2 when the shape does not fit (C % 16 != 0, misaligned pointers): use reduce + apply.
extern "C" int b200_bn_bwd_cluster(const void* x, const void* y, const void* dy_a, const void* dy_b, void* dx, void* dres,
                                   const float* gamma, const float* save_mean, const float* save_rstd, float* dgamma,
                                   float* dbeta, long long rows, int C, int relu, int max_cluster, cudaStream_t stream) {
  const bool allow_uncached = max_cluster < 0;       // negative cap: tests exercise the uncached variant explicitly
  if (max_cluster < 0) max_cluster = -max_cluster;
  if (rows <= 0) return 0;
  const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(relu ? y : x) |
                       reinterpret_cast<uintptr_t>(dy_a) | reinterpret_cast<uintptr_t>(dy_b) |
                       reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(dres);
  if (C % BNC_CW != 0 || (al & 15) || rows > (1ll << 30)) return -2;
  if (max_cluster <= 0 || max_cluster > 16) max_cluster = 16;
  const int slices = C / BNC_CW;
  int S = 1;
  while (S < max_cluster && (rows + S - 1) / S > BNC_LANES) S <<= 1;             // aim at one row per thread ...
  while (S > 1 && static_cast<long long>(slices) * S > 2 * device_sm_count()) S >>= 1;          // ... within two CTAs per SM
  const int rpc = static_cast<int>((rows + S - 1) / S);
  const int iters = (rpc + BNC_LANES - 1) / BNC_LANES;
  const dim3 grid(static_cast<unsigned>(slices), static_cast<unsigned>(S));
#define BNC_GO(I)                                                                                                        \
  return launch_bn_bwd_cluster<I>(grid, S, stream, reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(y), \
                                  reinterpret_cast<const uint4*>(dy_a), reinterpret_cast<const uint4*>(dy_b),            \
                                  reinterpret_cast<uint4*>(dx), reinterpret_cast<uint4*>(dres), gamma, save_mean,        \
                                  save_rstd, dgamma, dbeta, static_cast<int>(rows), C, relu, rpc)
  if (iters <= 1) BNC_GO(1);
  if (iters <= 2) BNC_GO(2);
  if (iters <= 4) BNC_GO(4);
  if (iters <= 8) BNC_GO(8);
  // More rows than the register cache holds (ResNet stem: 32768 rows x 64 channels): the uncached variant (ITER = 0,
  // second pass re-reads) is correct but a 16-trip latency-bound loop per thread, slower than the
  // grid-wide reduce + apply pair, so such shapes are handed back to the two-kernel path.
  if (!allow_uncached) return -2;
  BNC_GO(0);
#undef BNC_GO
}

extern "C" int b200_layernorm_fwd(const void* x, const void* residual, void* y, const float* gamma, const float* beta,
                                  float* mean, float* rstd, long long rows, int C, float eps, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(residual);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  if (row_vec_ok(C, x, residual, y) && ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define LN_FWD(LPR, VPL) launch_pdl(layernorm_fwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, xp, rp, yp, gamma, beta, mean, rstd, rows, C, eps)
    ROW_DISPATCH(C, LN_FWD);
#undef LN_FWD
    RET_LAST();
  }
  const int warps = 8;
  launch_pdl(layernorm_fwd_kernel, static_cast<unsigned>((rows + warps - 1) / warps), warps * 32, 0, stream, xp, rp, yp,
             gamma, beta, mean, rstd, rows, C, eps);
  RET_LAST();
}
extern "C" int b200_layernorm_bwd(const void* x, const void* dy, void* dx, const float* gamma, const float* mean,
                                  const float* rstd, float* dgamma, float* dbeta, long long rows, int C,
                                  cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(dx);
  if (row_vec_ok(C, x, dy, dx) && (reinterpret_cast<uintptr_t>(gamma) & 15) == 0) {
    const int rpb = rows_per_block(C);
    long long gv = (rows + rpb - 1) / rpb;
    if (gv > device_sm_count() * 2) gv = device_sm_count() * 2;
#define LN_BWD(LPR, VPL) launch_pdl(layernorm_bwd_vec_kernel<LPR, VPL>, static_cast<unsigned>(gv), 256, 2 * C * sizeof(float), stream, xp, gp, dp, gamma, mean, rstd, dgamma, dbeta, rows, C)
    ROW_DISPATCH(C, LN_BWD);
#undef LN_BWD
    RET_LAST();
  }
  long long g = (rows + 7) / 8;
  if (g > device_sm_count() * 2) g = device_sm_count() * 2;
  launch_pdl(layernorm_bwd_kernel, static_cast<unsigned>(g), 256, 2 * C * sizeof(float), stream, xp, gp, dp, gamma, mean,
             rstd, dgamma, dbeta, rows, C);
  RET_LAST();
}
extern "C" int b200_softmax_fwd(const void* x, void* y, long long rows, int C, float scale, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  if (row_vec_ok(C, x, y, nullptr)) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define SM_FWD(LPR, VPL) launch_pdl(softmax_fwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, xp, yp, rows, C, scale)
    ROW_DISPATCH(C, SM_FWD);
#undef SM_FWD
    RET_LAST();
  }
  launch_pdl(softmax_fwd_kernel, static_cast<unsigned>((rows + 7) / 8), 256, 0, stream, xp, yp, rows, C, scale);
  RET_LAST();
}
extern "C" int b200_softmax_bwd(const void* y, const void* dy, void* dx, long long rows, int C, float scale,
                                cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(y);
  const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(dx);
  if (row_vec_ok(C, y, dy, dx)) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define SM_BWD(LPR, VPL) launch_pdl(softmax_bwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, yp, gp, dp, rows, C, scale)
    ROW_DISPATCH(C, SM_BWD);
#undef SM_BWD
    RET_LAST();
  }
  launch_pdl(softmax_bwd_kernel, static_cast<unsigned>((rows + 7) / 8), 256, 0, stream, yp, gp, dp, rows, C, scale);
  RET_LAST();
}


// ---- ResNet stem: BatchNorm + ReLU + max-pool fused (forward) and its two-kernel backward.  Return -2 when the shape is
// not supported (C % 8, C/8 not a power of two <= 256 for the reduction, window > 255 taps): callers fall back.
extern "C" int b200_bn_relu_maxpool(const void* z, void* p, void* argmax, const float* sums, const float* gamma,
                                    const float* beta, float* running_mean, float* running_var, float* save_mean,
                                    float* save_rstd, long long* nbt, int N, int H, int W, int C, int k, int stride, int pad,
                                    int Ho, int Wo, float eps, float momentum, cudaStream_t stream) {
  if (C % 8 || k * k > 255) return -2;
  const long long total = static_cast<long long>(N) * Ho * Wo * (C / 8);
  if (total <= 0) return 0;
  launch_pdl(bn_relu_maxpool_kernel, stream_grid(total), 256, 2 * C * sizeof(float), stream,
             reinterpret_cast<const uint4*>(z), reinterpret_cast<uint4*>(p), reinterpret_cast<uint2*>(argmax), sums, gamma,
             beta, running_mean, running_var, save_mean, save_rstd, nbt, N, H, W, C, k, stride, pad, Ho, Wo, eps, momentum);
  RET_LAST();
}
extern "C" int b200_bn_maxpool_bwd(const void* z, const void* p, const void* argmax, const void* dy_a, const void* dy_b,
                                   void* dz, const float* gamma, const float* save_mean, const float* save_rstd, float* sums,
                                   float* dgamma, float* dbeta, int N, int H, int W, int C, int k, int stride, int pad, int Ho,
                                   int Wo, cudaStream_t stream) {
  if (k * k > 255 || !colred_vec_ok(C, z, p, dy_a) || (dy_b != nullptr && (reinterpret_cast<uintptr_t>(dy_b) & 15)))
    return -2;
  const long long prow = static_cast<long long>(N) * Ho * Wo;
  if (prow <= 0) return 0;
  int rpc = 2 * (256 / (C >> 3));       // two passes per CTA: 128 CTAs (and 128 atomics per channel) for the 32x32 stem
  if (rpc < colred_rows_per_cta(prow, C, 2)) rpc = colred_rows_per_cta(prow, C, 2);
  launch_pdl(bn_maxpool_bwd_reduce_kernel, static_cast<unsigned>((prow + rpc - 1) / rpc), 256, 256 * 16 * sizeof(float),
             stream, reinterpret_cast<const __nv_bfloat16*>(z), reinterpret_cast<const uint4*>(p),
             reinterpret_cast<const uint2*>(argmax), reinterpret_cast<const uint4*>(dy_a),
             reinterpret_cast<const uint4*>(dy_b), save_mean, save_rstd, sums, N, H, W, C, k, stride, pad, Ho, Wo, rpc);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long total = static_cast<long long>(N) * H * W * (C / 8);
  launch_pdl(bn_maxpool_bwd_apply_kernel, stream_grid(total), 256, 5 * C * sizeof(float), stream,
             reinterpret_cast<const uint4*>(z), reinterpret_cast<const uint4*>(p), reinterpret_cast<const uint2*>(argmax),
             reinterpret_cast<const uint4*>(dy_a), reinterpret_cast<const uint4*>(dy_b), reinterpret_cast<uint4*>(dz), gamma,
             save_mean, save_rstd, sums, dgamma, dbeta, N, H, W, C, k, stride, pad, Ho, Wo);
  RET_LAST();
}

// ---- GroupNorm.  Returns -2 for an unsupported shape (G not dividing C).  16-byte vectors when Cg % 8 == 0 and every
// tensor is 16-byte aligned; the (n, g) block stays on chip when it holds at most GN_CACHE_ELEMS elements.
// The cached backward keeps up to GN_CACHE_ELEMS * 6 bytes of dynamic shared memory, above the 48 KB default: opt each
// cached instantiation in to that maximum once per device (the same value from every thread, so concurrent first
// launches set the same attribute).  Returns the attribute's error code.
constexpr int GN_MAX_DEVICES = 64;
template <int V>
static int gn_bwd_cache_optin() {
  static std::atomic<int> done[GN_MAX_DEVICES] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  if (dev < GN_MAX_DEVICES && done[dev].load(std::memory_order_acquire)) return 0;
  e = cudaFuncSetAttribute(gn_bwd_kernel<V, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           static_cast<int>(GN_CACHE_ELEMS * 6));
  if (e != cudaSuccess) return static_cast<int>(e);
  if (dev < GN_MAX_DEVICES) done[dev].store(1, std::memory_order_release);
  return 0;
}
static inline bool gn_vec_ok(int C, int G, std::initializer_list<const void*> ptrs) {
  if ((C / G) % 8) return false;
  uintptr_t al = 0;
  for (const void* p : ptrs) al |= reinterpret_cast<uintptr_t>(p);
  return (al & 15) == 0;
}

extern "C" int b200_gn_fwd(const void* z, const void* residual, void* y, const float* gamma, const float* beta,
                           float* mean, float* rstd, float* work, long long N, long long HW, int C, int G, float eps,
                           int relu, cudaStream_t stream) {
  if (G <= 0 || C % G) return -2;
  if (N <= 0 || HW <= 0) return 0;
  const unsigned grid = static_cast<unsigned>(N * G);
  const long long M = HW * (C / G);
  const bool cache = M <= GN_CACHE_ELEMS;
  const size_t smem = cache ? static_cast<size_t>(M) * 2 : 0;
  unsigned* counters = reinterpret_cast<unsigned*>(work);
  const auto* zp = reinterpret_cast<const __nv_bfloat16*>(z);
  const auto* rp = reinterpret_cast<const __nv_bfloat16*>(residual);
  auto* yp = reinterpret_cast<__nv_bfloat16*>(y);
#define GN_FWD(V, CA) launch_pdl(gn_fwd_kernel<V, CA>, grid, GN_THREADS, smem, stream, zp, rp, yp, gamma, beta, mean, rstd, \
                                 counters, HW, C, G, eps, relu)
  if (gn_vec_ok(C, G, {z, residual, y})) {
    if (cache) GN_FWD(8, true); else GN_FWD(8, false);
  } else {
    if (cache) GN_FWD(1, true); else GN_FWD(1, false);
  }
#undef GN_FWD
  RET_LAST();
}

extern "C" int b200_gn_bwd(const void* z, const void* y, const void* dy_a, const void* dy_b, void* dz, void* dres,
                           const float* gamma, const float* mean, const float* rstd, float* dgamma, float* dbeta,
                           float* work, long long N, long long HW, int C, int G, int relu, cudaStream_t stream) {
  if (G <= 0 || C % G || work == nullptr) return -2;
  if (N <= 0 || HW <= 0) return 0;
  const unsigned grid = static_cast<unsigned>(N * G);
  const long long M = HW * (C / G);
  const bool cache = M <= GN_CACHE_ELEMS;
  const size_t smem = cache ? static_cast<size_t>(M) * 6 : 0;
  const auto* zp = reinterpret_cast<const __nv_bfloat16*>(z);
  const auto* yp = reinterpret_cast<const __nv_bfloat16*>(y);
  const auto* ap = reinterpret_cast<const __nv_bfloat16*>(dy_a);
  const auto* bp = reinterpret_cast<const __nv_bfloat16*>(dy_b);
  auto* dzp = reinterpret_cast<__nv_bfloat16*>(dz);
  auto* drp = reinterpret_cast<__nv_bfloat16*>(dres);
  const bool vec = gn_vec_ok(C, G, {z, relu ? y : z, dy_a, dy_b, dz, dres});
  if (cache) {
    const int rc = vec ? gn_bwd_cache_optin<8>() : gn_bwd_cache_optin<1>();
    if (rc != 0) return rc;
  }
#define GN_BWD(V, CA) launch_pdl(gn_bwd_kernel<V, CA>, grid, GN_THREADS, smem, stream, zp, yp, ap, bp, dzp, drp, gamma, \
                                 mean, rstd, dgamma, dbeta, work, HW, C, G, relu)
  if (vec) {
    if (cache) GN_BWD(8, true); else GN_BWD(8, false);
  } else {
    if (cache) GN_BWD(1, true); else GN_BWD(1, false);
  }
#undef GN_BWD
  RET_LAST();
}

B200_TRACE_REGISTER(norm)
