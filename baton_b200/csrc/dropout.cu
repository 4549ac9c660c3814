// Dropout forms of the LayerNorm and softmax row kernels (norm.cu) and an elementwise dropout, for BERT training.
// The masks are regenerated from the counter (dropout.cuh) wherever they are needed; no mask is stored.
//   LayerNorm, input dropout (MODE 1: attn_ln / ffn_ln):
//     forward : pre = drop(x) + residual?, y = LN(pre) * gamma + beta; writes y, pre (bf16), mean, rstd
//     backward: dpre = LN backward against pre; writes dpre (the residual's gradient) and dx = M s dpre
//   LayerNorm, output dropout (MODE 2: the embeddings):
//     forward : y = drop(LN(x + residual?) * gamma + beta)
//     backward: the LN backward of dy' = M s dy, masked as it is loaded (dgamma / dbeta included)
//   softmax (the multi-kernel attention path):
//     forward : P = softmax(scale x) (saved for backward) and Pd = drop(P) (the operand of the PV GEMM)
//     backward: g = M s dPd, dx = scale P (g - sum(P g))
//   dropout: y = drop(x) elementwise (forward and backward alike; the classifier input)
// Element i of a site is its flat row-major index row * C + col.  The vectorised kernels draw one Philox block per 4
// elements (two per 16-byte vector); the scalar kernels (C % 8 != 0 or misaligned rows) one per element.
#define B200_TU_TAG 13
#include "dropout.cuh"
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"
#include "rows.cuh"

namespace b200 {

constexpr int DROP_IN = 1, DROP_OUT = 2;

// ------------------------------------------------------------------ LayerNorm forward
template <int LPR, int VPL, int MODE>
__global__ void __launch_bounds__(256)
layernorm_drop_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                              __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ pre,
                              const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ mean,
                              float* __restrict__ rstd, long long rows, int C, float eps, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
  constexpr int RPW = 32 / LPR;
  const int gl = threadIdx.x & (LPR - 1);
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW +
                        ((threadIdx.x & 31) / LPR);
  const bool row_ok = row < rows;
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
      if (MODE == DROP_IN) {
        const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[k][j] = kept(bits, j, v[k][j], da.scale);
      }
      if (rr != nullptr) {
        float r8[8];
        unpack8(rr[idx], r8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[k][j] += r8[j];
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
      if (MODE == DROP_OUT) {
        const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = kept(bits, j, o[j], da.scale);
      } else {
        reinterpret_cast<uint4*>(pre + row * C)[idx] = pack8(v[k]);
      }
      yr[idx] = pack8(o);
    }
  }
  if (gl == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
}

template <int MODE>
__global__ void __launch_bounds__(256)
layernorm_drop_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                          __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ pre, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float* __restrict__ mean, float* __restrict__ rstd,
                          long long rows, int C, float eps, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __nv_bfloat16* xr = x + row * C;
  const __nv_bfloat16* rr = res != nullptr ? res + row * C : nullptr;
  const unsigned long long i0 = static_cast<unsigned long long>(row) * C;
  float v[LN_MAX_PER_LANE];
  float s = 0.f;
  int cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) {
    float t = __bfloat162float(xr[c]);
    if (MODE == DROP_IN) t = drop_keep1(dc, i0 + c) ? t * da.scale : 0.f;
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
  for (int c = lane; c < C; c += 32, ++cnt) {
    float o = fmaf((v[cnt] - mu) * rs, gamma[c], beta[c]);
    if (MODE == DROP_OUT) o = drop_keep1(dc, i0 + c) ? o * da.scale : 0.f;
    else pre[row * C + c] = __float2bfloat16_rn(v[cnt]);
    yr[c] = __float2bfloat16_rn(o);
  }
  if (lane == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
}

// ------------------------------------------------------------------ LayerNorm backward
// x: the pre-norm input (pre).  MODE 1: dx = dpre, dxd = M s dpre.  MODE 2: dy' = M s dy throughout; dxd unused.
template <int LPR, int VPL, int MODE>
__global__ void __launch_bounds__(256)
layernorm_drop_bwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                              __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dxd,
                              const float* __restrict__ gamma, const float* __restrict__ mean,
                              const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                              long long rows, int C, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
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
        if (MODE == DROP_OUT) {
          const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
          for (int j = 0; j < 8; ++j) g8[j] = kept(bits, j, g8[j], da.scale);
        }
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
          dr[idx] = pack8(o);
          if (MODE == DROP_IN) {
            const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = kept(bits, j, o[j], da.scale);
            reinterpret_cast<uint4*>(dxd + row * C)[idx] = pack8(o);
          }
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

template <int MODE>
__global__ void __launch_bounds__(256)
layernorm_drop_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                          __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dxd, const float* __restrict__ gamma,
                          const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ dgamma,
                          float* __restrict__ dbeta, long long rows, int C, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
  extern __shared__ float sm[];
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
    const unsigned long long i0 = static_cast<unsigned long long>(row) * C;
    const float mu = mean[row], rs = rstd[row];
    float xh[LN_MAX_PER_LANE], gg[LN_MAX_PER_LANE];
    float s1 = 0.f, s2 = 0.f;
    int cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) {
      const float h = (__bfloat162float(xr[c]) - mu) * rs;
      float g = __bfloat162float(gr[c]);
      if (MODE == DROP_OUT) g = drop_keep1(dc, i0 + c) ? g * da.scale : 0.f;
      atomicAdd(sg + c, g * h);
      atomicAdd(sb + c, g);
      const float gw = g * gamma[c];
      xh[cnt] = h; gg[cnt] = gw;
      s1 += gw; s2 = fmaf(gw, h, s2);
    }
    s1 = warp_sum(s1) / C;
    s2 = warp_sum(s2) / C;
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) {
      const float o = rs * (gg[cnt] - s1 - xh[cnt] * s2);
      dx[row * C + c] = __float2bfloat16_rn(o);
      if (MODE == DROP_IN) dxd[row * C + c] = __float2bfloat16_rn(drop_keep1(dc, i0 + c) ? o * da.scale : 0.f);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(dgamma + c, sg[c]);
    atomicAdd(dbeta + c, sb[c]);
  }
}

// ------------------------------------------------------------------ softmax
template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
softmax_drop_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                            __nv_bfloat16* __restrict__ yd, long long rows, int C, float scale, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
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
  uint4* ydr = reinterpret_cast<uint4*>(yd + row * C);
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int idx = gl + k * LPR;
    if (idx < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] *= inv;
      yr[idx] = pack8(v[k]);
      const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] = kept(bits, j, v[k][j], da.scale);
      ydr[idx] = pack8(v[k]);
    }
  }
}

__global__ void __launch_bounds__(256)
softmax_drop_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                        __nv_bfloat16* __restrict__ yd, long long rows, int C, float scale, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
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
  cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) {
    const float p = v[cnt] * inv;
    y[row * C + c] = __float2bfloat16_rn(p);
    yd[row * C + c] = __float2bfloat16_rn(drop_keep1(dc, static_cast<unsigned long long>(row) * C + c) ? p * da.scale : 0.f);
  }
}

// dx = scale * y * (g - sum(g * y)),  g = M s dy
template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
softmax_drop_bwd_vec_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                            __nv_bfloat16* __restrict__ dx, long long rows, int C, float scale, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
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
      const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(row) * C + idx * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        g[k][j] = kept(bits, j, g[k][j], da.scale);
        s = fmaf(p[k][j], g[k][j], s);
      }
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

__global__ void __launch_bounds__(256)
softmax_drop_bwd_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                        __nv_bfloat16* __restrict__ dx, long long rows, int C, float scale, const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
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
    const float t = __bfloat162float(gr[c]);
    g[cnt] = drop_keep1(dc, static_cast<unsigned long long>(row) * C + c) ? t * da.scale : 0.f;
    s = fmaf(p[cnt], g[cnt], s);
  }
  s = warp_sum(s);
  cnt = 0;
  for (int c = lane; c < C; c += 32, ++cnt) dx[row * C + c] = __float2bfloat16_rn(scale * p[cnt] * (g[cnt] - s));
}

// ------------------------------------------------------------------ elementwise: y = drop(x)
// thread t owns elements 8t .. 8t + 7 (16-byte vectors when x and y are aligned, else one element at a time)
__global__ void __launch_bounds__(256)
dropout_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n, int vec,
               const DropArgs da) {
  griddep_launch_dependents();
  griddep_wait();
  const DropCtr dc = drop_ctr(da);
  const long long i0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 8;
  if (i0 >= n) return;
  const uint32_t bits = drop_keep8(dc, static_cast<unsigned long long>(i0));
  if (vec && i0 + 8 <= n) {
    float v[8];
    unpack8(reinterpret_cast<const uint4*>(x)[i0 >> 3], v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = kept(bits, j, v[j], da.scale);
    reinterpret_cast<uint4*>(y)[i0 >> 3] = pack8(v);
    return;
  }
  for (int j = 0; j < 8 && i0 + j < n; ++j)
    y[i0 + j] = __float2bfloat16_rn(kept(bits, j, __bfloat162float(x[i0 + j]), da.scale));
}

}  // namespace b200

using namespace b200;

#define RET_LAST() return static_cast<int>(cudaGetLastError())

extern "C" int b200_layernorm_drop_fwd(const void* x, const void* residual, void* y, void* pre, const float* gamma,
                                       const float* beta, float* mean, float* rstd, long long rows, int C, float eps,
                                       int mode, const B200Dropout* drop, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE || (mode != DROP_IN && mode != DROP_OUT) || (mode == DROP_IN && pre == nullptr)) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(residual);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  __nv_bfloat16* pp = reinterpret_cast<__nv_bfloat16*>(pre);
  const DropArgs da = drop_args(drop);
  if (row_vec_ok(C, x, residual, y) && (reinterpret_cast<uintptr_t>(pre) & 15) == 0 &&
      ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define LN_FWD(LPR, VPL)                                                                                                 \
  (mode == DROP_IN ? launch_pdl(layernorm_drop_fwd_vec_kernel<LPR, VPL, DROP_IN>, grid, 256, 0, stream, xp, rp, yp, pp, \
                                gamma, beta, mean, rstd, rows, C, eps, da)                                               \
                   : launch_pdl(layernorm_drop_fwd_vec_kernel<LPR, VPL, DROP_OUT>, grid, 256, 0, stream, xp, rp, yp, pp, \
                                gamma, beta, mean, rstd, rows, C, eps, da))
    ROW_DISPATCH(C, LN_FWD);
#undef LN_FWD
    RET_LAST();
  }
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  if (mode == DROP_IN)
    launch_pdl(layernorm_drop_fwd_kernel<DROP_IN>, grid, 256, 0, stream, xp, rp, yp, pp, gamma, beta, mean, rstd, rows, C,
               eps, da);
  else
    launch_pdl(layernorm_drop_fwd_kernel<DROP_OUT>, grid, 256, 0, stream, xp, rp, yp, pp, gamma, beta, mean, rstd, rows, C,
               eps, da);
  RET_LAST();
}

extern "C" int b200_layernorm_drop_bwd(const void* x, const void* dy, void* dx, void* dxd, const float* gamma,
                                       const float* mean, const float* rstd, float* dgamma, float* dbeta, long long rows,
                                       int C, int mode, const B200Dropout* drop, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE || (mode != DROP_IN && mode != DROP_OUT) || (mode == DROP_IN && dxd == nullptr)) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(dx);
  __nv_bfloat16* ddp = reinterpret_cast<__nv_bfloat16*>(dxd);
  const DropArgs da = drop_args(drop);
  const size_t smem = 2 * C * sizeof(float);
  if (row_vec_ok(C, x, dy, dx) && ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(dxd)) & 15) == 0) {
    const int rpb = rows_per_block(C);
    long long gv = (rows + rpb - 1) / rpb;
    if (gv > device_sm_count() * 2) gv = device_sm_count() * 2;
    const unsigned grid = static_cast<unsigned>(gv);
#define LN_BWD(LPR, VPL)                                                                                                 \
  (mode == DROP_IN ? launch_pdl(layernorm_drop_bwd_vec_kernel<LPR, VPL, DROP_IN>, grid, 256, smem, stream, xp, gp, dp,  \
                                ddp, gamma, mean, rstd, dgamma, dbeta, rows, C, da)                                      \
                   : launch_pdl(layernorm_drop_bwd_vec_kernel<LPR, VPL, DROP_OUT>, grid, 256, smem, stream, xp, gp, dp, \
                                ddp, gamma, mean, rstd, dgamma, dbeta, rows, C, da))
    ROW_DISPATCH(C, LN_BWD);
#undef LN_BWD
    RET_LAST();
  }
  long long g = (rows + 7) / 8;
  if (g > device_sm_count() * 2) g = device_sm_count() * 2;
  if (mode == DROP_IN)
    launch_pdl(layernorm_drop_bwd_kernel<DROP_IN>, static_cast<unsigned>(g), 256, smem, stream, xp, gp, dp, ddp, gamma,
               mean, rstd, dgamma, dbeta, rows, C, da);
  else
    launch_pdl(layernorm_drop_bwd_kernel<DROP_OUT>, static_cast<unsigned>(g), 256, smem, stream, xp, gp, dp, ddp, gamma,
               mean, rstd, dgamma, dbeta, rows, C, da);
  RET_LAST();
}

extern "C" int b200_softmax_drop_fwd(const void* x, void* y, void* yd, long long rows, int C, float scale,
                                     const B200Dropout* drop, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  __nv_bfloat16* ydp = reinterpret_cast<__nv_bfloat16*>(yd);
  const DropArgs da = drop_args(drop);
  if (row_vec_ok(C, x, y, yd)) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define SM_FWD(LPR, VPL) launch_pdl(softmax_drop_fwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, xp, yp, ydp, rows, C, scale, da)
    ROW_DISPATCH(C, SM_FWD);
#undef SM_FWD
    RET_LAST();
  }
  launch_pdl(softmax_drop_fwd_kernel, static_cast<unsigned>((rows + 7) / 8), 256, 0, stream, xp, yp, ydp, rows, C, scale, da);
  RET_LAST();
}

extern "C" int b200_softmax_drop_bwd(const void* y, const void* dy, void* dx, long long rows, int C, float scale,
                                     const B200Dropout* drop, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (C > 32 * LN_MAX_PER_LANE) return -2;
  const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(y);
  const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(dx);
  const DropArgs da = drop_args(drop);
  if (row_vec_ok(C, y, dy, dx)) {
    const int rpb = rows_per_block(C);
    const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define SM_BWD(LPR, VPL) launch_pdl(softmax_drop_bwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, yp, gp, dp, rows, C, scale, da)
    ROW_DISPATCH(C, SM_BWD);
#undef SM_BWD
    RET_LAST();
  }
  launch_pdl(softmax_drop_bwd_kernel, static_cast<unsigned>((rows + 7) / 8), 256, 0, stream, yp, gp, dp, rows, C, scale, da);
  RET_LAST();
}

extern "C" int b200_dropout(const void* x, void* y, long long n, const B200Dropout* drop, cudaStream_t stream) {
  if (n <= 0) return 0;
  const int vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  const long long threads = (n + 7) / 8;
  launch_pdl(dropout_kernel, static_cast<unsigned>((threads + 255) / 256), 256, 0, stream,
             reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y), n, vec, drop_args(drop));
  RET_LAST();
}

B200_TRACE_REGISTER(dropout)
