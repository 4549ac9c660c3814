// Fused loss kernels (K7): forward + backward in one pass, with the batch-mean loss accumulated
// into a device scalar that the trainer reads ONCE per epoch (the reference does float(loss) -- a
// host sync -- on every batch: utils.py:88).
#define B200_TU_TAG 11
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <bool IN_FP32>
__device__ __forceinline__ float load_logit(const void* p, long long i) {
  if constexpr (IN_FP32)
    return reinterpret_cast<const float*>(p)[i];
  else
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}

// Soft targets (mixup / CutMix / label smoothing): the target of row r is
//   q = (1 - eps) (lam 1[a] + lam1 1[b]) + eps / C,   a = target[r], b = target[(r - 1 + rows) % rows]
// (the partner of the batch rolled by one, as the mixing gather pairs the images), lam / lam1 the fp32 bit patterns in
// words 0 / 1 of the step's mix row (data/mix.py); no mix row: lam = 1, lam1 = 0, b = a (plain label smoothing).
// loss_row = logsumexp(z) - sum_c q_c z_c, dz = (softmax(z) - q) * grad_scale, #correct += lam [argmax = a] + lam1
// [argmax = b].
struct SoftTarget {
  float wa, wb, u, lam, lam1;    // q = u + wa 1[a] + wb 1[b]
  int b;
};
__device__ __forceinline__ SoftTarget soft_target(const long long* target, long long row, long long rows, int a,
                                                  const int* mix_row, float eps, int C) {
  SoftTarget q{0.f, 0.f, eps / static_cast<float>(C), 1.f, 0.f, a};
  if (mix_row != nullptr) {
    q.lam = __int_as_float(mix_row[0]);
    q.lam1 = __int_as_float(mix_row[1]);
    q.b = static_cast<int>(target[row == 0 ? rows - 1 : row - 1]);
  }
  q.wa = (1.f - eps) * q.lam;
  q.wb = (1.f - eps) * q.lam1;
  return q;
}

// one warp per row: loss_row = logsumexp(z) - z[target]; dz = (softmax(z) - onehot) * grad_scale
// loss_acc[0] += sum(loss_row) * grad_scale ; loss_acc[1] += #correct (argmax == target)
// SOFT: the soft target above instead of the one-hot
template <bool IN_FP32, bool OUT_FP32, bool SOFT>
__device__ __forceinline__ void
softmax_xent_body(const void* __restrict__ logits, const long long* __restrict__ target, void* __restrict__ dlogits,
                  float* __restrict__ loss_acc, long long rows, int C, long long ld, float grad_scale,
                  const int* __restrict__ mix_row, float eps) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  float my_loss = 0.f, my_hit = 0.f;
  if (row < rows) {
    const long long base = row * ld;
    float m = -INFINITY;
    int am = 0;
    for (int c = lane; c < C; c += 32) {
      const float z = load_logit<IN_FP32>(logits, base + c);
      if (z > m) { m = z; am = c; }
    }
    // warp argmax (ties -> lowest index)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o);
      const int oa = __shfl_xor_sync(0xffffffffu, am, o);
      if (om > m || (om == m && oa < am)) { m = om; am = oa; }
    }
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += __expf(load_logit<IN_FP32>(logits, base + c) - m);
    s = wsum(s);
    const float lse = m + __logf(s);
    const int t = static_cast<int>(target[row]);
    const float inv = 1.f / s;
    SoftTarget q{};
    float zsum = 0.f;
    if constexpr (SOFT) q = soft_target(target, row, rows, t, mix_row, eps, C);
    for (int c = lane; c < C; c += 32) {
      const float z = load_logit<IN_FP32>(logits, base + c);
      float g;
      if constexpr (SOFT) {
        zsum += z;
        g = (__expf(z - m) * inv - (q.u + (c == t ? q.wa : 0.f) + (c == q.b ? q.wb : 0.f))) * grad_scale;
      } else {
        g = (__expf(z - m) * inv - (c == t ? 1.f : 0.f)) * grad_scale;
      }
      if (dlogits != nullptr) {
        if constexpr (OUT_FP32)
          reinterpret_cast<float*>(dlogits)[base + c] = g;
        else
          reinterpret_cast<__nv_bfloat16*>(dlogits)[base + c] = __float2bfloat16_rn(g);
      }
    }
    if constexpr (SOFT) {
      zsum = wsum(zsum);
      if (lane == 0) {
        const float zb = load_logit<IN_FP32>(logits, base + q.b);
        my_loss = (lse - q.wa * load_logit<IN_FP32>(logits, base + t) - q.wb * zb - q.u * zsum) * grad_scale;
        my_hit = (am == t ? q.lam : 0.f) + (am == q.b ? q.lam1 : 0.f);
      }
    } else if (lane == 0) {
      my_loss = (lse - load_logit<IN_FP32>(logits, base + t)) * grad_scale;
      my_hit = (am == t) ? 1.f : 0.f;
    }
  }
  // block-level combine -> one atomic pair per block
  __shared__ float sl[8], sh[8];
  if (lane == 0) { sl[threadIdx.x >> 5] = my_loss; sh[threadIdx.x >> 5] = my_hit; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) { a += sl[w]; b += sh[w]; }
    atomicAdd(loss_acc, a);
    atomicAdd(loss_acc + 1, b);
  }
}
template <bool IN_FP32, bool OUT_FP32>
__global__ void __launch_bounds__(256)
softmax_xent_kernel(const void* __restrict__ logits, const long long* __restrict__ target, void* __restrict__ dlogits,
                    float* __restrict__ loss_acc, long long rows, int C, long long ld, float grad_scale) {
  softmax_xent_body<IN_FP32, OUT_FP32, false>(logits, target, dlogits, loss_acc, rows, C, ld, grad_scale, nullptr, 0.f);
}
template <bool IN_FP32, bool OUT_FP32>
__global__ void __launch_bounds__(256)
softmax_xent_soft_kernel(const void* __restrict__ logits, const long long* __restrict__ target,
                         void* __restrict__ dlogits, float* __restrict__ loss_acc, long long rows, int C, long long ld,
                         float grad_scale, const int* __restrict__ mix_row, float eps) {
  softmax_xent_body<IN_FP32, OUT_FP32, true>(logits, target, dlogits, loss_acc, rows, C, ld, grad_scale, mix_row, eps);
}

// MSE: loss_acc[0] += sum((p - t)^2) * grad_scale ; dp = 2 * (p - t) * grad_scale   (grad_scale = 1/numel)
template <bool IN_FP32, bool OUT_FP32>
__global__ void __launch_bounds__(256)
mse_kernel(const void* __restrict__ pred, const float* __restrict__ target, void* __restrict__ dpred,
           float* __restrict__ loss_acc, long long n, float grad_scale) {
  griddep_launch_dependents();
  griddep_wait();
  float acc = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float d = load_logit<IN_FP32>(pred, i) - target[i];
    acc = fmaf(d, d, acc);
    if (dpred != nullptr) {
      const float g = 2.f * d * grad_scale;
      if constexpr (OUT_FP32)
        reinterpret_cast<float*>(dpred)[i] = g;
      else
        reinterpret_cast<__nv_bfloat16*>(dpred)[i] = __float2bfloat16_rn(g);
    }
  }
  acc = wsum(acc);
  __shared__ float s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) a += s[w];
    atomicAdd(loss_acc, a * grad_scale);
  }
}

// ------------------------------------------------------------------ classifier head in ONE launch
// logits = x W^T + b (classes <= 32), softmax cross-entropy, and the whole backward of the head:
//   dX[r, :] = dlogits[r, :] W          (bf16, feeds the backbone's backward)
//   dW      += dlogits^T X ,  db += colsum(dlogits)      (fp32 atomics straight into the gradient arena)
//   loss_acc[0] += mean loss, loss_acc[1] += #correct
// It replaces six launches (GEMM 128x10x512, loss, cast, colsum, two SIMT GEMMs) for ~4 MFLOP of work.  One CTA handles HEAD_ROWS rows: warp w owns row w for the logits, the
// 256 threads then share the dX / dW tiles.  x: bf16 [rows, K], W: bf16 [NC, K] (the arena's shadow), b: fp32.
// BACKWARD = false: the evaluation instantiation -- logits, loss and #correct only (no dX / dW / db; grid.y = 1).
// SOFT (training only): the soft target of softmax_xent_soft_kernel; z_b and sum(z) are one shuffle and one warp sum more.
constexpr int HEAD_ROWS = 8;
template <bool BACKWARD, bool SOFT>
__device__ __forceinline__ void
linear_xent_head_body(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                      const long long* __restrict__ target, __nv_bfloat16* __restrict__ dx, float* __restrict__ dw,
                      float* __restrict__ db, float* __restrict__ loss_acc, float* __restrict__ logits_out, int rows,
                      int K, int NC, float grad_scale, const int* __restrict__ mix_row, float eps) {
  griddep_launch_dependents();
  extern __shared__ __align__(16) unsigned char head_smem[];
  __nv_bfloat16* sw = reinterpret_cast<__nv_bfloat16*>(head_smem);                 // [NC][K]
  __nv_bfloat16* sx = sw + static_cast<size_t>(NC) * K;                           // [HEAD_ROWS][K]
  float* sdl = reinterpret_cast<float*>(sx + static_cast<size_t>(HEAD_ROWS) * K);  // [HEAD_ROWS][32]
  float* sred = sdl + HEAD_ROWS * 32;                                              // [HEAD_ROWS][2]
  griddep_wait();
  const int r0 = blockIdx.x * HEAD_ROWS;
  const int K8 = K >> 3;
  for (int i = threadIdx.x; i < NC * K8; i += 256) reinterpret_cast<uint4*>(sw)[i] = reinterpret_cast<const uint4*>(w)[i];
  for (int i = threadIdx.x; i < HEAD_ROWS * K8; i += 256) {
    const int r = i / K8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < rows) v = reinterpret_cast<const uint4*>(x + static_cast<size_t>(r0 + r) * K)[i - r * K8];
    reinterpret_cast<uint4*>(sx)[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {   // logits + loss of row `warp` (8 warps = HEAD_ROWS rows); lane c ends up holding logit c.  Four classes at a time:
      // independent accumulators and interleaved shuffle reductions (the one-class-at-a-time version was a 10-deep
      // dependent chain of reductions)
    const int row = r0 + warp;
    float mine = -INFINITY;
    for (int c0 = 0; c0 < NC; c0 += 4) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = lane * 2; k < K; k += 64) {
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sx + warp * K + k));
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (c0 + j < NC) {
            const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sw + (c0 + j) * K + k));
            acc[j] = fmaf(a.x, b.x, fmaf(a.y, b.y, acc[j]));
          }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (c0 + j < NC && lane == c0 + j) mine = acc[j] + (bias != nullptr ? bias[c0 + j] : 0.f);
    }
    float loss = 0.f, hit = 0.f, dl = 0.f;
    if (row < rows) {
      if (logits_out != nullptr && lane < NC && blockIdx.y == 0) logits_out[static_cast<size_t>(row) * NC + lane] = mine;
      float m = mine;
      int am = lane < NC ? lane : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        const int oa = __shfl_xor_sync(0xffffffffu, am, o);
        if (om > m || (om == m && oa < am)) { m = om; am = oa; }
      }
      const float e = lane < NC ? __expf(mine - m) : 0.f;
      const float ssum = wsum(e);
      const int t = static_cast<int>(target[row]);
      const float zt = __shfl_sync(0xffffffffu, mine, t & 31);
      if constexpr (SOFT) {
        const SoftTarget q = soft_target(target, row, rows, t, mix_row, eps, NC);
        const float zb = __shfl_sync(0xffffffffu, mine, q.b & 31);
        const float zsum = wsum(lane < NC ? mine : 0.f);
        loss = (m + __logf(ssum)) - q.wa * zt - q.wb * zb - q.u * zsum;
        hit = (am == t ? q.lam : 0.f) + (am == q.b ? q.lam1 : 0.f);
        dl = lane < NC ? (e / ssum - (q.u + (lane == t ? q.wa : 0.f) + (lane == q.b ? q.wb : 0.f))) * grad_scale : 0.f;
      } else {
        loss = (m + __logf(ssum)) - zt;
        hit = (am == t) ? 1.f : 0.f;
        dl = lane < NC ? (e / ssum - (lane == t ? 1.f : 0.f)) * grad_scale : 0.f;
      }
    }
    sdl[warp * 32 + lane] = dl;
    if (lane == 0) { sred[warp * 2] = loss; sred[warp * 2 + 1] = hit; }
  }
  __syncthreads();
  if (threadIdx.x == 0 && blockIdx.y == 0) {
    float l = 0.f, h = 0.f;
    for (int r = 0; r < HEAD_ROWS; ++r) { l += sred[r * 2]; h += sred[r * 2 + 1]; }
    atomicAdd(loss_acc, l * grad_scale);
    atomicAdd(loss_acc + 1, h);
  }
  if constexpr (!BACKWARD) return;
  // the backward outputs are split over blockIdx.y: slice s owns columns [k_lo, k_hi) of dX and dW (the logits above are
  // recomputed by every slice -- 8 x NC x K FMAs -- which is cheaper than the 16-CTA serial tail it replaces)
  const int kslice = K / static_cast<int>(gridDim.y);
  const int k_lo = static_cast<int>(blockIdx.y) * kslice;
  // dX[r, k] = sum_c dl[r, c] W[c, k]
  if (dx != nullptr) {
    const int half = kslice >> 1;
    for (int i = threadIdx.x; i < HEAD_ROWS * half; i += 256) {
      const int r = i / half, k = k_lo + (i - r * half) * 2;
      if (r0 + r >= rows) continue;
      float a0 = 0.f, a1 = 0.f;
      for (int c = 0; c < NC; ++c) {
        const float d = sdl[r * 32 + c];
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sw + c * K + k));
        a0 = fmaf(d, b.x, a0); a1 = fmaf(d, b.y, a1);
      }
      *reinterpret_cast<__nv_bfloat162*>(dx + static_cast<size_t>(r0 + r) * K + k) = __floats2bfloat162_rn(a0, a1);
    }
  }
  // dW[c, k] += sum_r dl[r, c] X[r, k]  (the bf16-rounded dl the GEMM path would have used is not reproduced: fp32 is closer)
  for (int i = threadIdx.x; i < NC * kslice; i += 256) {
    const int c = i / kslice, k = k_lo + (i - c * kslice);
    float a = 0.f;
#pragma unroll
    for (int r = 0; r < HEAD_ROWS; ++r) a = fmaf(sdl[r * 32 + c], __bfloat162float(sx[r * K + k]), a);
    atomicAdd(dw + c * K + k, a);
  }
  if (db != nullptr && blockIdx.y == 0 && threadIdx.x < NC) {
    float a = 0.f;
    for (int r = 0; r < HEAD_ROWS; ++r) a += sdl[r * 32 + threadIdx.x];
    atomicAdd(db + threadIdx.x, a);
  }
}
template <bool BACKWARD>
__global__ void __launch_bounds__(256)
linear_xent_head_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                        const long long* __restrict__ target, __nv_bfloat16* __restrict__ dx, float* __restrict__ dw,
                        float* __restrict__ db, float* __restrict__ loss_acc, float* __restrict__ logits_out, int rows,
                        int K, int NC, float grad_scale) {
  linear_xent_head_body<BACKWARD, false>(x, w, bias, target, dx, dw, db, loss_acc, logits_out, rows, K, NC, grad_scale,
                                         nullptr, 0.f);
}
__global__ void __launch_bounds__(256)
linear_xent_head_soft_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                             const float* __restrict__ bias, const long long* __restrict__ target,
                             __nv_bfloat16* __restrict__ dx, float* __restrict__ dw, float* __restrict__ db,
                             float* __restrict__ loss_acc, int rows, int K, int NC, float grad_scale,
                             const int* __restrict__ mix_row, float eps) {
  linear_xent_head_body<true, true>(x, w, bias, target, dx, dw, db, loss_acc, nullptr, rows, K, NC, grad_scale, mix_row,
                                    eps);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_softmax_xent(const void* logits, int logits_fp32, const long long* target, void* dlogits,
                                 int dl_fp32, float* loss_acc, long long rows, int C, long long ld, float grad_scale,
                                 cudaStream_t stream) {
  if (rows <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
#define XENT(A, B) launch_pdl(softmax_xent_kernel<A, B>, grid, 256, 0, stream, logits, target, dlogits, loss_acc, rows, C, ld, grad_scale)
  if (logits_fp32) { if (dl_fp32) XENT(true, true); else XENT(true, false); }
  else             { if (dl_fp32) XENT(false, true); else XENT(false, false); }
#undef XENT
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_softmax_xent_soft(const void* logits, int logits_fp32, const long long* target, void* dlogits,
                                      int dl_fp32, float* loss_acc, long long rows, int C, long long ld, float grad_scale,
                                      const int* mix_row, float eps, cudaStream_t stream) {
  if (rows <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
#define XENT(A, B)                                                                                                     \
  launch_pdl(softmax_xent_soft_kernel<A, B>, grid, 256, 0, stream, logits, target, dlogits, loss_acc, rows, C, ld,     \
             grad_scale, mix_row, eps)
  if (logits_fp32) { if (dl_fp32) XENT(true, true); else XENT(true, false); }
  else             { if (dl_fp32) XENT(false, true); else XENT(false, false); }
#undef XENT
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_mse(const void* pred, int pred_fp32, const float* target, void* dpred, int dp_fp32,
                        float* loss_acc, long long n, float grad_scale, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long g = (n + 255) / 256;
  if (g > device_sm_count() * 4) g = device_sm_count() * 4;
  const unsigned grid = static_cast<unsigned>(g);
#define MSE(A, B) launch_pdl(mse_kernel<A, B>, grid, 256, 0, stream, pred, target, dpred, loss_acc, n, grad_scale)
  if (pred_fp32) { if (dp_fp32) MSE(true, true); else MSE(true, false); }
  else           { if (dp_fp32) MSE(false, true); else MSE(false, false); }
#undef MSE
  return static_cast<int>(cudaGetLastError());
}

// classifier head: NC <= 32 classes, K % 8 == 0, K * (NC + HEAD_ROWS) * 2 bytes of shared memory.  Returns -2 otherwise.
extern "C" int b200_linear_xent_head(const void* x, const void* w, const float* bias, const long long* target, void* dx,
                                     float* dw, float* db, float* loss_acc, float* logits_out, int rows, int K, int NC,
                                     float grad_scale, cudaStream_t stream) {
  using namespace b200;
  if (rows <= 0) return 0;
  const size_t smem = static_cast<size_t>(K) * (NC + HEAD_ROWS) * 2 + HEAD_ROWS * 34 * 4;
  if (NC < 1 || NC > 32 || (K % 8) || smem > 200 * 1024 || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(dx) & 3))
    return -2;
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(linear_xent_head_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = smem;
  }
  int ks = 8;                                   // column slices of the backward outputs (grid.y); each a multiple of 8 columns
  while (ks > 1 && (K % (ks * 8))) ks >>= 1;
  cudaError_t le = launch_pdl(linear_xent_head_kernel<true>, dim3((rows + HEAD_ROWS - 1) / HEAD_ROWS, ks), dim3(256), smem, stream,
                              reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(w), bias,
                              target, reinterpret_cast<__nv_bfloat16*>(dx), dw, db, loss_acc, logits_out, rows, K, NC,
                              grad_scale);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

// classifier head with soft targets (training): b200_linear_xent_head's shape limits, no logits output
extern "C" int b200_linear_xent_head_soft(const void* x, const void* w, const float* bias, const long long* target,
                                          void* dx, float* dw, float* db, float* loss_acc, int rows, int K, int NC,
                                          float grad_scale, const int* mix_row, float eps, cudaStream_t stream) {
  using namespace b200;
  if (rows <= 0) return 0;
  const size_t smem = static_cast<size_t>(K) * (NC + HEAD_ROWS) * 2 + HEAD_ROWS * 34 * 4;
  if (NC < 1 || NC > 32 || (K % 8) || smem > 200 * 1024 || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(dx) & 3))
    return -2;
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(linear_xent_head_soft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = smem;
  }
  int ks = 8;
  while (ks > 1 && (K % (ks * 8))) ks >>= 1;
  cudaError_t le = launch_pdl(linear_xent_head_soft_kernel, dim3((rows + HEAD_ROWS - 1) / HEAD_ROWS, ks), dim3(256), smem,
                              stream, reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(w),
                              bias, target, reinterpret_cast<__nv_bfloat16*>(dx), dw, db, loss_acc, rows, K, NC,
                              grad_scale, mix_row, eps);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

// forward-only classifier head (evaluation): loss_acc[0] += sum of the row losses, loss_acc[1] += #correct, optional fp32
// logits.  Same shape limits as b200_linear_xent_head.
extern "C" int b200_linear_xent_eval(const void* x, const void* w, const float* bias, const long long* target,
                                     float* loss_acc, float* logits_out, int rows, int K, int NC, cudaStream_t stream) {
  using namespace b200;
  if (rows <= 0) return 0;
  const size_t smem = static_cast<size_t>(K) * (NC + HEAD_ROWS) * 2 + HEAD_ROWS * 34 * 4;
  if (NC < 1 || NC > 32 || (K % 8) || smem > 200 * 1024 || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15))
    return -2;
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(linear_xent_head_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = smem;
  }
  cudaError_t le = launch_pdl(linear_xent_head_kernel<false>, dim3((rows + HEAD_ROWS - 1) / HEAD_ROWS, 1), dim3(256), smem,
                              stream, reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(w),
                              bias, target, static_cast<__nv_bfloat16*>(nullptr), static_cast<float*>(nullptr),
                              static_cast<float*>(nullptr), loss_acc, logits_out, rows, K, NC, 1.0f);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

B200_TRACE_REGISTER(loss)
