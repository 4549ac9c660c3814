// NHWC convolution plumbing around the wgmma GEMM: im2col (forward / wgrad operand), col2im
// (dgrad scatter written as a gather so it needs no atomics), max / average pooling.
// A convolution is   Y[N*Ho*Wo, Cout] = col[N*Ho*Wo, KH*KW*Cin] * W[Cout, KH*KW*Cin]^T
// with K index = (kh*KW + kw)*Cin + c, i.e. weights stored [Cout, KH, KW, Cin] (channels_last).
#define B200_TU_TAG 9
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int CV_THREADS = 256;
static inline int cv_grid(long long n, int max_ctas = device_sm_count() * 8) {
  long long g = (n + CV_THREADS - 1) / CV_THREADS;
  if (g < 1) g = 1;
  if (g > max_ctas) g = max_ctas;
  return static_cast<int>(g);
}

// vector path: C % 8 == 0, one thread per 16-byte chunk of the col matrix
__global__ void __launch_bounds__(CV_THREADS)
im2col_vec_kernel(const uint4* __restrict__ x, uint4* __restrict__ col, int N, int H, int W, int C8, int KH, int KW,
                  int stride, int pad, int Ho, int Wo, int kp8) {
  griddep_launch_dependents();
  griddep_wait();
  const long long rows = static_cast<long long>(N) * Ho * Wo;
  const long long total = rows * kp8;
  const int k8 = KH * KW * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / kp8;
    const int kc = static_cast<int>(i - row * kp8);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (kc < k8) {
      const int tap = kc / C8, c8 = kc - tap * C8;
      const int kh = tap / KW, kw = tap - kh * KW;
      const int wo = static_cast<int>(row % Wo);
      const long long t = row / Wo;
      const int ho = static_cast<int>(t % Ho);
      const int n = static_cast<int>(t / Ho);
      const int h = ho * stride - pad + kh, w = wo * stride - pad + kw;
      if (h >= 0 && h < H && w >= 0 && w < W)
        v = __ldg(x + ((static_cast<long long>(n) * H + h) * W + w) * C8 + c8);
    }
    col[i] = v;
  }
}
// small-channel path (first layer, C = 3): one thread builds one 16-byte vector of `col` (8 consecutive k
// positions, walking (kh, kw, c) incrementally) from 2-byte gathers that hit L1 -- 8x fewer threads and
// stores than one element per thread
__global__ void __launch_bounds__(CV_THREADS)
im2col_scalar_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ col, int N, int H, int W, int C,
                     int KH, int KW, int stride, int pad, int Ho, int Wo, int kp) {
  griddep_launch_dependents();
  griddep_wait();
  const long long rows = static_cast<long long>(N) * Ho * Wo;
  const int kp8 = kp >> 3;
  const long long total = rows * kp8;
  const int K = KH * KW * C;
  const unsigned short* xs = reinterpret_cast<const unsigned short*>(x);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / kp8;
    const int kc0 = static_cast<int>(i - row * kp8) << 3;
    const int wo = static_cast<int>(row % Wo);
    const long long t = row / Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const int h0 = ho * stride - pad, w0 = wo * stride - pad;
    int tap = kc0 / C, c = kc0 - tap * C;
    int kh = tap / KW, kw = tap - kh * KW;
    const unsigned short* img = xs + static_cast<long long>(n) * H * W * C;
    unsigned short e[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      unsigned short v = 0;
      const int h = h0 + kh, w = w0 + kw;
      if (kc0 + j < K && h >= 0 && h < H && w >= 0 && w < W) v = __ldg(img + (h * W + w) * C + c);
      e[j] = v;
      if (++c == C) {
        c = 0;
        if (++kw == KW) { kw = 0; ++kh; }
      }
    }
    uint4 o;
    o.x = e[0] | (static_cast<uint32_t>(e[1]) << 16);
    o.y = e[2] | (static_cast<uint32_t>(e[3]) << 16);
    o.z = e[4] | (static_cast<uint32_t>(e[5]) << 16);
    o.w = e[6] | (static_cast<uint32_t>(e[7]) << 16);
    *reinterpret_cast<uint4*>(col + row * kp + kc0) = o;
  }
}

// small-channel path, shared-memory edition: one CTA builds the col rows of ONE output image row (n, ho).  The KH input
// rows it needs (KH x W x C elements, 1.3 KB for the 7x7x3 stem at 32x32) are fetched once with 16-byte loads, the
// 16-byte col vectors are then assembled from shared memory -- the scalar kernel above issued eight 2-byte global loads per
// vector.  Needs (W * C) % 8 == 0 (16-byte aligned image rows).
__global__ void __launch_bounds__(128)
im2col_smallc_smem_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ col, int N, int H, int W, int C,
                          int KH, int KW, int stride, int pad, int Ho, int Wo, int kp) {
  griddep_launch_dependents();
  griddep_wait();
  extern __shared__ __align__(16) unsigned short srow[];     // [KH][W * C]
  const int ho = blockIdx.x % Ho, n = blockIdx.x / Ho;
  const int wc = W * C, wc8 = wc >> 3;
  const int h0 = ho * stride - pad;
  for (int i = threadIdx.x; i < KH * wc8; i += blockDim.x) {
    const int kh = i / wc8, v = i - kh * wc8;
    const int h = h0 + kh;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (h >= 0 && h < H) val = __ldg(reinterpret_cast<const uint4*>(x + (static_cast<long long>(n) * H + h) * wc) + v);
    reinterpret_cast<uint4*>(srow)[i] = val;
  }
  __syncthreads();
  const int K = KH * KW * C, kp8 = kp >> 3;
  const long long row0 = (static_cast<long long>(n) * Ho + ho) * Wo;
  for (int i = threadIdx.x; i < Wo * kp8; i += blockDim.x) {
    const int wo = i / kp8, kc0 = (i - wo * kp8) << 3;
    const int w0 = wo * stride - pad;
    int tap = kc0 / C, c = kc0 - tap * C;
    int kh = tap / KW, kw = tap - kh * KW;
    unsigned short e[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int w = w0 + kw;
      e[j] = (kc0 + j < K && w >= 0 && w < W) ? srow[kh * wc + w * C + c] : static_cast<unsigned short>(0);
      if (++c == C) {
        c = 0;
        if (++kw == KW) { kw = 0; ++kh; }
      }
    }
    uint4 o;
    o.x = e[0] | (static_cast<uint32_t>(e[1]) << 16);
    o.y = e[2] | (static_cast<uint32_t>(e[3]) << 16);
    o.z = e[4] | (static_cast<uint32_t>(e[5]) << 16);
    o.w = e[6] | (static_cast<uint32_t>(e[7]) << 16);
    *reinterpret_cast<uint4*>(col + (row0 + wo) * kp + kc0) = o;
  }
}

// dX[n,h,w,c] = sum over taps (kh,kw) with ho = (h + pad - kh)/stride, wo = (w + pad - kw)/stride integral
// and in range of dcol[(n,ho,wo), (kh*KW+kw)*C + c].  One thread per 8 channels, fp32 accumulation.
__global__ void __launch_bounds__(CV_THREADS)
col2im_vec_kernel(const uint4* __restrict__ col, uint4* __restrict__ dx, int N, int H, int W, int C8, int KH, int KW,
                  int stride, int pad, int Ho, int Wo, int kp8) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * H * W * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % C8);
    long long t = i / C8;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int kh = 0; kh < KH; ++kh) {
      const int hh = h + pad - kh;
      if (hh < 0 || hh % stride) continue;
      const int ho = hh / stride;
      if (ho >= Ho) continue;
      for (int kw = 0; kw < KW; ++kw) {
        const int ww = w + pad - kw;
        if (ww < 0 || ww % stride) continue;
        const int wo = ww / stride;
        if (wo >= Wo) continue;
        const long long row = (static_cast<long long>(n) * Ho + ho) * Wo + wo;
        const uint4 v = __ldg(col + row * kp8 + (kh * KW + kw) * C8 + c8);
        const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      }
    }
    dx[i] = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                       pack_bf16x2(acc[6], acc[7]));
  }
}

// max pooling, NHWC, one thread per (n, ho, wo, channel pair); argmax = flat (h*W + w) of the winner
__global__ void __launch_bounds__(CV_THREADS)
maxpool_kernel(const __nv_bfloat162* __restrict__ x, __nv_bfloat162* __restrict__ y, int2* __restrict__ arg, int N,
               int H, int W, int C2, int k, int stride, int pad, int Ho, int Wo) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * Ho * Wo * C2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c2 = static_cast<int>(i % C2);
    long long t = i / C2;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    float m0 = -INFINITY, m1 = -INFINITY;
    int a0 = -1, a1 = -1;
    for (int kh = 0; kh < k; ++kh) {
      const int h = ho * stride - pad + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int w = wo * stride - pad + kw;
        if (w < 0 || w >= W) continue;
        const float2 v = __bfloat1622float2(x[((static_cast<long long>(n) * H + h) * W + w) * C2 + c2]);
        if (v.x > m0) { m0 = v.x; a0 = h * W + w; }
        if (v.y > m1) { m1 = v.y; a1 = h * W + w; }
      }
    }
    y[i] = __floats2bfloat162_rn(m0, m1);
    arg[i] = make_int2(a0, a1);
  }
}
// backward as a gather (no atomics): each input position scans the windows covering it
__global__ void __launch_bounds__(CV_THREADS)
maxpool_bwd_gather_kernel(const __nv_bfloat162* __restrict__ dy, const int2* __restrict__ arg,
                          __nv_bfloat162* __restrict__ dx, int N, int H, int W, int C2, int Ho, int Wo, int k,
                          int stride, int pad) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * H * W * C2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c2 = static_cast<int>(i % C2);
    long long t = i / C2;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    const int me = h * W + w;
    float g0 = 0.f, g1 = 0.f;
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
        const long long o = ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * C2 + c2;
        const int2 a = arg[o];
        const float2 g = __bfloat1622float2(dy[o]);
        if (a.x == me) g0 += g.x;
        if (a.y == me) g1 += g.y;
      }
    }
    dx[i] = __floats2bfloat162_rn(g0, g1);
  }
}

// ---- 16-byte variants (C % 8 == 0): one thread = 8 channels of one pixel; the winner is remembered as ONE BYTE (the tap
// index kh * k + kw inside the window) instead of a 4-byte flat position, and the backward optionally sums a two-piece
// gradient (dy_a + dy_b) while loading.  The scalar kernels above move 4 bytes per request.
__global__ void __launch_bounds__(CV_THREADS)
maxpool_vec_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, uint2* __restrict__ arg, int N, int H, int W, int C8,
                   int k, int stride, int pad, int Ho, int Wo) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * Ho * Wo * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % C8);
    long long t = i / C8;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    float m[8];
    uint32_t a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { m[j] = -INFINITY; a[j] = 255u; }
    for (int kh = 0; kh < k; ++kh) {
      const int h = ho * stride - pad + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int w = wo * stride - pad + kw;
        if (w < 0 || w >= W) continue;
        const uint4 v = x[((static_cast<long long>(n) * H + h) * W + w) * C8 + c8];
        const float2 p0 = unpack_bf16x2(v.x), p1 = unpack_bf16x2(v.y), p2 = unpack_bf16x2(v.z), p3 = unpack_bf16x2(v.w);
        const float f[8] = {p0.x, p0.y, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y};
        const uint32_t tap = static_cast<uint32_t>(kh * k + kw);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (f[j] > m[j]) { m[j] = f[j]; a[j] = tap; }
      }
    }
    y[i] = make_uint4(pack_bf16x2(m[0], m[1]), pack_bf16x2(m[2], m[3]), pack_bf16x2(m[4], m[5]), pack_bf16x2(m[6], m[7]));
    arg[i] = make_uint2(a[0] | (a[1] << 8) | (a[2] << 16) | (a[3] << 24), a[4] | (a[5] << 8) | (a[6] << 16) | (a[7] << 24));
  }
}

__global__ void __launch_bounds__(CV_THREADS)
maxpool_bwd_vec_kernel(const uint4* __restrict__ dy_a, const uint4* __restrict__ dy_b, const uint2* __restrict__ arg,
                       uint4* __restrict__ dx, int N, int H, int W, int C8, int Ho, int Wo, int k, int stride, int pad) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * H * W * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % C8);
    long long t = i / C8;
    const int w = static_cast<int>(t % W);
    t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
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
        const uint2 a = arg[o];
        uint4 v = dy_a[o];
        float2 p0 = unpack_bf16x2(v.x), p1 = unpack_bf16x2(v.y), p2 = unpack_bf16x2(v.z), p3 = unpack_bf16x2(v.w);
        float f[8] = {p0.x, p0.y, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y};
        if (dy_b != nullptr) {
          v = dy_b[o];
          p0 = unpack_bf16x2(v.x); p1 = unpack_bf16x2(v.y); p2 = unpack_bf16x2(v.z); p3 = unpack_bf16x2(v.w);
          f[0] += p0.x; f[1] += p0.y; f[2] += p1.x; f[3] += p1.y; f[4] += p2.x; f[5] += p2.y; f[6] += p3.x; f[7] += p3.y;
        }
        const uint32_t tap = static_cast<uint32_t>(kh * k + kw);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t aj = ((j < 4 ? a.x : a.y) >> (8 * (j & 3))) & 0xffu;
          if (aj == tap) g[j] += f[j];
        }
      }
    }
    dx[i] = make_uint4(pack_bf16x2(g[0], g[1]), pack_bf16x2(g[2], g[3]), pack_bf16x2(g[4], g[5]), pack_bf16x2(g[6], g[7]));
  }
}

// global average pool [N, HW, C] -> [N, C] and its backward
__global__ void __launch_bounds__(CV_THREADS)
avgpool_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int HW, int C) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * C;
  const float inv = 1.f / HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long n = i / C;
    float acc = 0.f;
    for (int p = 0; p < HW; ++p) acc += __bfloat162float(x[(n * HW + p) * C + c]);
    y[i] = __float2bfloat16_rn(acc * inv);
  }
}
__global__ void __launch_bounds__(CV_THREADS)
avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int N, int HW, int C) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = static_cast<long long>(N) * HW * C;
  const float inv = 1.f / HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long n = i / (static_cast<long long>(HW) * C);
    dx[i] = __float2bfloat16_rn(__bfloat162float(dy[n * C + c]) * inv);
  }
}

}  // namespace b200

using namespace b200;
#define RET_LAST() return static_cast<int>(cudaGetLastError())

extern "C" int b200_im2col_nhwc(const void* x, void* col, int N, int H, int W, int C, int KH, int KW, int stride,
                                int pad, int Ho, int Wo, int kp, cudaStream_t stream) {
  const long long rows = static_cast<long long>(N) * Ho * Wo;
  if (rows <= 0) return 0;
  if (C % 8 == 0 && kp % 8 == 0) {
    launch_pdl(im2col_vec_kernel, cv_grid(rows * (kp / 8)), CV_THREADS, 0, stream, 
        reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(col), N, H, W, C / 8, KH, KW, stride, pad, Ho, Wo,
        kp / 8);
  } else if (kp % 8 == 0 && (W * C) % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
             static_cast<size_t>(KH) * W * C * 2 <= 48 * 1024) {
    launch_pdl(im2col_smallc_smem_kernel, dim3(static_cast<unsigned>(N * Ho)), dim3(128),
               static_cast<size_t>(KH) * W * C * 2, stream, reinterpret_cast<const __nv_bfloat16*>(x),
               reinterpret_cast<__nv_bfloat16*>(col), N, H, W, C, KH, KW, stride, pad, Ho, Wo, kp);
  } else {
    if (kp % 8) return -2;
    launch_pdl(im2col_scalar_kernel, cv_grid(rows * (kp / 8)), CV_THREADS, 0, stream, 
        reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(col), N, H, W, C, KH, KW, stride,
        pad, Ho, Wo, kp);
  }
  RET_LAST();
}
extern "C" int b200_col2im_nhwc(const void* col, void* dx, int N, int H, int W, int C, int KH, int KW, int stride,
                                int pad, int Ho, int Wo, int kp, cudaStream_t stream) {
  if (C % 8 || kp % 8) return -2;
  const long long total = static_cast<long long>(N) * H * W * (C / 8);
  if (total <= 0) return 0;
  launch_pdl(col2im_vec_kernel, cv_grid(total), CV_THREADS, 0, stream, reinterpret_cast<const uint4*>(col),
                                                               reinterpret_cast<uint4*>(dx), N, H, W, C / 8, KH, KW,
                                                               stride, pad, Ho, Wo, kp / 8);
  RET_LAST();
}
// argmax: int32 flat positions (scalar path) or, when arg_u8 != 0 (C % 8 == 0, k * k <= 255), one byte per element
extern "C" int b200_maxpool_nhwc(const void* x, void* y, int* argmax, int N, int H, int W, int C, int k, int stride,
                                 int pad, int Ho, int Wo, int arg_u8, cudaStream_t stream) {
  if (arg_u8) {
    if (C % 8 || k * k > 255) return -2;
    const long long total8 = static_cast<long long>(N) * Ho * Wo * (C / 8);
    if (total8 <= 0) return 0;
    launch_pdl(maxpool_vec_kernel, cv_grid(total8), CV_THREADS, 0, stream, reinterpret_cast<const uint4*>(x),
               reinterpret_cast<uint4*>(y), reinterpret_cast<uint2*>(argmax), N, H, W, C / 8, k, stride, pad, Ho, Wo);
    RET_LAST();
  }
  if (C % 2) return -2;
  const long long total = static_cast<long long>(N) * Ho * Wo * (C / 2);
  if (total <= 0) return 0;
  launch_pdl(maxpool_kernel, cv_grid(total), CV_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat162*>(x),
                                                            reinterpret_cast<__nv_bfloat162*>(y),
                                                            reinterpret_cast<int2*>(argmax), N, H, W, C / 2, k, stride,
                                                            pad, Ho, Wo);
  RET_LAST();
}
extern "C" int b200_maxpool_bwd_nhwc(const void* dy, const void* dy_b, const int* argmax, void* dx, int N, int H, int W,
                                     int C, int Ho, int Wo, int k, int stride, int pad, int arg_u8, cudaStream_t stream) {
  if (arg_u8) {
    if (C % 8) return -2;
    const long long total8 = static_cast<long long>(N) * H * W * (C / 8);
    if (total8 <= 0) return 0;
    launch_pdl(maxpool_bwd_vec_kernel, cv_grid(total8), CV_THREADS, 0, stream, reinterpret_cast<const uint4*>(dy),
               reinterpret_cast<const uint4*>(dy_b), reinterpret_cast<const uint2*>(argmax), reinterpret_cast<uint4*>(dx), N,
               H, W, C / 8, Ho, Wo, k, stride, pad);
    RET_LAST();
  }
  if (dy_b != nullptr) return -2;
  if (C % 2) return -2;
  const long long total = static_cast<long long>(N) * H * W * (C / 2);
  if (total <= 0) return 0;
  launch_pdl(maxpool_bwd_gather_kernel, cv_grid(total), CV_THREADS, 0, stream, 
      reinterpret_cast<const __nv_bfloat162*>(dy), reinterpret_cast<const int2*>(argmax),
      reinterpret_cast<__nv_bfloat162*>(dx), N, H, W, C / 2, Ho, Wo, k, stride, pad);
  RET_LAST();
}
extern "C" int b200_avgpool_nhwc(const void* x, void* y, int N, int HW, int C, cudaStream_t stream) {
  const long long total = static_cast<long long>(N) * C;
  if (total <= 0) return 0;
  launch_pdl(avgpool_kernel, cv_grid(total), CV_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                                                            reinterpret_cast<__nv_bfloat16*>(y), N, HW, C);
  RET_LAST();
}
extern "C" int b200_avgpool_bwd_nhwc(const void* dy, void* dx, int N, int HW, int C, cudaStream_t stream) {
  const long long total = static_cast<long long>(N) * HW * C;
  if (total <= 0) return 0;
  launch_pdl(avgpool_bwd_kernel, cv_grid(total), CV_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(dy),
                                                                reinterpret_cast<__nv_bfloat16*>(dx), N, HW, C);
  RET_LAST();
}

B200_TRACE_REGISTER(conv)
