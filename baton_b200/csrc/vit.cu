// Vision Transformer pieces (models/vit.py): the token assembly forward and backward, and the pre-LN residual step
// s = x + r, y = LN(s) with both written, whose backward writes LN_bwd(dy) + ds once.  The add + LayerNorm kernels are
// the vectorised LayerNorm bodies of rows.cuh with SUM = true; the fused attention at S < 128 lives in attention.cu.
#define B200_TU_TAG 16
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"
#include "rows.cuh"

namespace b200 {

constexpr int EW_THREADS = 256;
static inline int ew_grid(long long n_vec, int max_ctas = device_sm_count() * 8) {
  long long g = (n_vec + EW_THREADS - 1) / EW_THREADS;
  if (g < 1) g = 1;
  if (g > max_ctas) g = max_ctas;
  return static_cast<int>(g);
}

// ---- ViT token assembly: [class token; patch embeddings] + position embedding, S = 1 + N tokens of D channels
// tok[b, 0] = bf16(cls + pos[0]); tok[b, 1 + n] = bf16((z[b, n] + bias) + pos[1 + n]), fp32 sums rounded once
__global__ void __launch_bounds__(EW_THREADS)
vit_tokens_fwd_kernel(const uint4* __restrict__ z, const float* __restrict__ cls, const float* __restrict__ bias,
                      const float* __restrict__ pos, uint4* __restrict__ tok, long long nv, int S, int D8) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d8 = static_cast<int>(i % D8);
    const long long bs = i / D8;
    const int s = static_cast<int>(bs % S);
    float o[8], a[8];
    load8f(pos + (static_cast<long long>(s) * D8 + d8) * 8, o);
    if (s == 0) {
      load8f(cls + d8 * 8, a);
    } else {
      float bb[8];
      unpack8(z[(bs / S * (S - 1) + s - 1) * D8 + d8], a);
      load8f(bias + d8 * 8, bb);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += bb[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = a[j] + o[j];
    tok[i] = pack8(o);
  }
}
// One launch: dz[b, n] = dtok[b, 1 + n]; dpos[s] += sum_b dtok[b, s]; dcls += sum_b dtok[b, 0];
// dbias += sum_{s >= 1} sum_b dtok[b, s].  CTA = one 8-channel group, thread (s, q) sums the images b = q (mod 4) in
// order; the four partials of a token, then the tokens 1..S-1 of dbias, are added in a fixed order, so the bits do not
// depend on the grid, the SM count or the run.  S <= 128.
constexpr int VT_Q = 4;
__global__ void __launch_bounds__(128 * VT_Q)
vit_tokens_bwd_kernel(const uint4* __restrict__ dtok, uint4* __restrict__ dz, float* __restrict__ dcls,
                      float* __restrict__ dbias, float* __restrict__ dpos, int B, int S, int D8) {
  __shared__ float part[VT_Q][128][9];
  griddep_launch_dependents();
  griddep_wait();
  const int d8 = blockIdx.x, s = threadIdx.x, q = threadIdx.y;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (s < S) {
#pragma unroll 4
    for (int b = q; b < B; b += VT_Q) {
      const uint4 u = __ldcs(dtok + (static_cast<long long>(b) * S + s) * D8 + d8);
      if (s > 0) dz[(static_cast<long long>(b) * (S - 1) + s - 1) * D8 + d8] = u;
      float f[8];
      unpack8(u, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[q][s][j] = acc[j];
  __syncthreads();
  if (q == 0 && s < S) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float t = part[0][s][j];
#pragma unroll
      for (int k = 1; k < VT_Q; ++k) t += part[k][s][j];
      part[0][s][j] = t;
      dpos[(static_cast<long long>(s) * D8 + d8) * 8 + j] += t;
      if (s == 0) dcls[d8 * 8 + j] += t;
    }
  }
  __syncthreads();
  if (q == 1 && s < 8) {
    float t = 0.f;
    for (int k = 1; k < S; ++k) t += part[0][k][s];
    dbias[d8 * 8 + s] += t;
  }
}

template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
layernorm_sum_fwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                             __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ sum, const float* __restrict__ gamma,
                             const float* __restrict__ beta, float* __restrict__ mean, float* __restrict__ rstd,
                             long long rows, int C, float eps) {
  layernorm_fwd_vec_body<LPR, VPL, true>(x, res, y, gamma, beta, mean, rstd, rows, C, eps, sum);
}
template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
layernorm_sum_bwd_vec_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                             const __nv_bfloat16* __restrict__ ds, __nv_bfloat16* __restrict__ dx,
                             const float* __restrict__ gamma, const float* __restrict__ mean,
                             const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                             long long rows, int C) {
  layernorm_bwd_vec_body<LPR, VPL, true>(x, dy, dx, gamma, mean, rstd, dgamma, dbeta, rows, C, ds);
}

}  // namespace b200

using namespace b200;

#define RET_LAST() return static_cast<int>(cudaGetLastError())

static inline bool vt_aligned(const void* a, const void* b, const void* c, const void* d, const void* e) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
           reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(e)) & 15) == 0;
}
// z [B, S-1, D] bf16, cls [D], bias [D], pos [S, D] fp32 -> tok [B, S, D] bf16; D % 8 == 0, 2 <= S <= 128
extern "C" int b200_vit_tokens_fwd(const void* z, const float* cls, const float* bias, const float* pos, void* tok, int B,
                                   int S, int D, cudaStream_t stream) {
  if (B <= 0) return 0;
  if (D % 8 || S < 2 || S > 128 || !vt_aligned(z, cls, bias, pos, tok)) return -2;
  const long long nv = static_cast<long long>(B) * S * (D / 8);
  launch_pdl(vit_tokens_fwd_kernel, ew_grid(nv), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(z), cls, bias,
             pos, reinterpret_cast<uint4*>(tok), nv, S, D / 8);
  RET_LAST();
}
// dtok [B, S, D] bf16 -> dz [B, S-1, D] bf16 (written), dcls [D], dbias [D], dpos [S, D] fp32 (accumulated)
extern "C" int b200_vit_tokens_bwd(const void* dtok, void* dz, float* dcls, float* dbias, float* dpos, int B, int S, int D,
                                   cudaStream_t stream) {
  if (B <= 0) return 0;
  if (D % 8 || S < 2 || S > 128 || !vt_aligned(dtok, dz, dcls, dbias, dpos)) return -2;
  launch_pdl(vit_tokens_bwd_kernel, dim3(D / 8), dim3(128, VT_Q), 0, stream, reinterpret_cast<const uint4*>(dtok),
             reinterpret_cast<uint4*>(dz), dcls, dbias, dpos, B, S, D / 8);
  RET_LAST();
}
// s = x + res, y = LN(s), both written (pre-LN blocks); vectorised rows only (-2 otherwise)
extern "C" int b200_layernorm_sum_fwd(const void* x, const void* residual, void* y, void* sum, const float* gamma,
                                      const float* beta, float* mean, float* rstd, long long rows, int C, float eps,
                                      cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (!row_vec_ok(C, x, residual, y) || ((reinterpret_cast<uintptr_t>(sum) | reinterpret_cast<uintptr_t>(gamma) |
                                          reinterpret_cast<uintptr_t>(beta)) & 15) != 0)
    return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(residual);
  __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(y);
  __nv_bfloat16* sp = reinterpret_cast<__nv_bfloat16*>(sum);
  const int rpb = rows_per_block(C);
  const unsigned grid = static_cast<unsigned>((rows + rpb - 1) / rpb);
#define LN_FWD(LPR, VPL) launch_pdl(layernorm_sum_fwd_vec_kernel<LPR, VPL>, grid, 256, 0, stream, xp, rp, yp, sp, gamma, beta, mean, rstd, rows, C, eps)
  ROW_DISPATCH(C, LN_FWD);
#undef LN_FWD
  RET_LAST();
}
// dsum = LN_bwd(dy) + ds (s: the saved sum); dgamma / dbeta accumulated as b200_layernorm_bwd does
extern "C" int b200_layernorm_sum_bwd(const void* s, const void* dy, const void* ds, void* dsum, const float* gamma,
                                      const float* mean, const float* rstd, float* dgamma, float* dbeta, long long rows,
                                      int C, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (!row_vec_ok(C, s, dy, dsum) || ((reinterpret_cast<uintptr_t>(ds) | reinterpret_cast<uintptr_t>(gamma)) & 15) != 0)
    return -2;
  const __nv_bfloat16* xp = reinterpret_cast<const __nv_bfloat16*>(s);
  const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(dy);
  const __nv_bfloat16* dsp = reinterpret_cast<const __nv_bfloat16*>(ds);
  __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(dsum);
  const int rpb = rows_per_block(C);
  long long gv = (rows + rpb - 1) / rpb;
  if (gv > device_sm_count() * 2) gv = device_sm_count() * 2;
#define LN_BWD(LPR, VPL) launch_pdl(layernorm_sum_bwd_vec_kernel<LPR, VPL>, static_cast<unsigned>(gv), 256, 2 * C * sizeof(float), stream, xp, gp, dsp, dp, gamma, mean, rstd, dgamma, dbeta, rows, C)
  ROW_DISPATCH(C, LN_BWD);
#undef LN_BWD
  RET_LAST();
}
#undef RET_LAST
