// LoRA adapter kernels: the down projection U = X A^T (and V = dY' B in the backward) and the adapter gradients
// dA = s V^T X, dB = s dY'^T U.  The rank-R term of the up projection runs in the epilogue of the base GEMM
// (b200_gemm_bf16_lora, csrc/gemm_wgmma.cu).  Shapes are tall and skinny: M = batch x sequence rows against at most
// B200_LORA_MAX_R ranks, so these are SIMT kernels over shared-memory tiles, not tensor-core GEMMs.
#include "ptx.cuh"
#include "launch.h"
#include "pdl.cuh"

namespace b200 {
namespace {

constexpr int DOWN_ROWS = 32;          // rows of X per CTA (one per lane)
constexpr int DOWN_K = 32;             // k per staged tile
constexpr int DOWN_PITCH = DOWN_K + 4; // floats: float4 rows 144 B apart, conflict-free across 8 lanes
constexpr int DOWN_THREADS = 256;      // 8 warps: warp w computes ranks w, w + 8, ... of its slice

struct DownArgs {
  const __nv_bfloat16* x;
  long long ldx;
  const __nv_bfloat16* w;
  long long w_ts, wsj, wsk;
  __nv_bfloat16* u;
  long long ldu;
  int M, T, rs, kt;
  long long xoff[3];
};

__global__ void __launch_bounds__(DOWN_THREADS) lora_down_kernel(const DownArgs a) {
  __shared__ __align__(16) float xs[DOWN_ROWS][DOWN_PITCH];
  __shared__ __align__(16) float ws[B200_LORA_MAX_R][DOWN_PITCH];
  griddep_launch_dependents();
  griddep_wait();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m0 = blockIdx.x * DOWN_ROWS, row = m0 + lane;
  const int nj = a.rs / 8;       // ranks per warp
  for (int t = 0; t < a.T; ++t) {
    const long long xoff = t == 0 ? a.xoff[0] : (t == 1 ? a.xoff[1] : a.xoff[2]);
    const __nv_bfloat16* w = a.w + t * a.w_ts;
    float acc[B200_LORA_MAX_R / 8];
#pragma unroll
    for (int i = 0; i < B200_LORA_MAX_R / 8; ++i) acc[i] = 0.f;
    for (int k0 = 0; k0 < a.kt; k0 += DOWN_K) {
      __syncthreads();        // the previous tile is consumed
      for (int i = tid; i < DOWN_ROWS * DOWN_K; i += DOWN_THREADS) {
        const int r = i / DOWN_K, k = i - r * DOWN_K;
        xs[r][k] = (m0 + r < a.M && k0 + k < a.kt)
                       ? __bfloat162float(a.x[static_cast<long long>(m0 + r) * a.ldx + xoff + k0 + k]) : 0.f;
      }
      for (int i = tid; i < a.rs * DOWN_K; i += DOWN_THREADS) {
        const int j = i / DOWN_K, k = i - j * DOWN_K;
        ws[j][k] = k0 + k < a.kt ? __bfloat162float(w[j * a.wsj + static_cast<long long>(k0 + k) * a.wsk]) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < DOWN_K; k += 4) {
        const float4 xv = *reinterpret_cast<const float4*>(&xs[lane][k]);
#pragma unroll
        for (int i = 0; i < B200_LORA_MAX_R / 8; ++i) {
          if (i < nj) {        // every lane of the warp reads the same rank row: one broadcast request
            const float4 wv = *reinterpret_cast<const float4*>(&ws[warp + 8 * i][k]);
            float s = acc[i];
            s = fmaf(xv.x, wv.x, s); s = fmaf(xv.y, wv.y, s); s = fmaf(xv.z, wv.z, s); s = fmaf(xv.w, wv.w, s);
            acc[i] = s;
          }
        }
      }
    }
    if (row < a.M) {
#pragma unroll
      for (int i = 0; i < B200_LORA_MAX_R / 8; ++i)
        if (i < nj) a.u[static_cast<long long>(row) * a.ldu + t * a.rs + warp + 8 * i] = __float2bfloat16_rn(acc[i]);
    }
  }
}

constexpr int GRAD_A = 128;            // a (the long axis) per CTA, one per thread of a half
constexpr int GRAD_B = 8;              // b (the rank axis) per CTA, four per thread
constexpr int GRAD_STEP = 32;          // rows per staged tile
constexpr int GRAD_THREADS = 256;

struct GradArgs {
  const __nv_bfloat16* l;
  long long ldl;
  const __nv_bfloat16* q;
  long long ldq;
  int M, NA, NB, S;
  long long lo[3], qo[3];
  float* work;       // [T][S][NB][NA]
};

// one partial per (slice, split, a tile, b tile): rows [split * B200_LORA_SPLIT_ROWS, +B200_LORA_SPLIT_ROWS) in order
__global__ void __launch_bounds__(GRAD_THREADS) lora_grad_partial_kernel(const GradArgs g) {
  __shared__ float ls[GRAD_STEP][GRAD_A];
  __shared__ float qs[GRAD_STEP][GRAD_B];
  griddep_launch_dependents();
  griddep_wait();
  const int tid = threadIdx.x;
  const int a0 = blockIdx.x * GRAD_A, b0 = blockIdx.y * GRAD_B;
  const int t = blockIdx.z / g.S, split = blockIdx.z - t * g.S;
  const long long lo = t == 0 ? g.lo[0] : (t == 1 ? g.lo[1] : g.lo[2]);
  const long long qo = t == 0 ? g.qo[0] : (t == 1 ? g.qo[1] : g.qo[2]);
  const int r0 = split * B200_LORA_SPLIT_ROWS;
  const int r1 = min(g.M, r0 + B200_LORA_SPLIT_ROWS);
  const int ai = tid % GRAD_A, bq = (tid / GRAD_A) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int m0 = r0; m0 < r1; m0 += GRAD_STEP) {
    __syncthreads();
    for (int i = tid; i < GRAD_STEP * GRAD_A; i += GRAD_THREADS) {
      const int r = i / GRAD_A, c = i - r * GRAD_A;
      ls[r][c] = (m0 + r < r1 && a0 + c < g.NA) ? __bfloat162float(g.l[static_cast<long long>(m0 + r) * g.ldl + lo + a0 + c])
                                                : 0.f;
    }
    for (int i = tid; i < GRAD_STEP * GRAD_B; i += GRAD_THREADS) {
      const int r = i / GRAD_B, c = i - r * GRAD_B;
      qs[r][c] = (m0 + r < r1 && b0 + c < g.NB) ? __bfloat162float(g.q[static_cast<long long>(m0 + r) * g.ldq + qo + b0 + c])
                                                : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < GRAD_STEP; ++r) {
      const float lv = ls[r][ai];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = fmaf(lv, qs[r][bq + i], acc[i]);
    }
  }
  float* w = g.work + static_cast<long long>(t * g.S + split) * g.NB * g.NA;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int b = b0 + bq + i, a = a0 + ai;
    if (b < g.NB && a < g.NA) w[static_cast<long long>(b) * g.NA + a] = acc[i];
  }
}

// out[t out_ts + a osa + b osb] += s * sum_split work[t][split][b][a], splits in order
__global__ void lora_grad_finish_kernel(const float* work, float* out, long long osa, long long osb, long long out_ts,
                                        int NA, int NB, int T, int S, float s) {
  griddep_launch_dependents();
  griddep_wait();
  const long long per = static_cast<long long>(NA) * NB;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < per * T;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i / per);
    const long long e = i - t * per;
    const int b = static_cast<int>(e / NA), a = static_cast<int>(e - static_cast<long long>(b) * NA);
    const float* w = work + static_cast<long long>(t) * S * per + e;
    float sum = 0.f;
    for (int k = 0; k < S; ++k) sum += w[k * per];
    float* o = out + t * out_ts + a * osa + b * osb;
    *o = fmaf(s, sum, *o);
  }
}

}  // namespace
}  // namespace b200

int b200_lora_down(const void* x, long long ldx, const void* w, long long w_ts, long long wsj, long long wsk, void* u,
                   long long ldu, int M, int T, int rs, int kt, const long long* xoff, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0) return 0;
  if (T < 1 || T > 3 || rs < 8 || rs % 8 || T * rs > B200_LORA_MAX_R || kt <= 0 || ldu < T * rs) return -3;
  DownArgs a;
  a.x = reinterpret_cast<const __nv_bfloat16*>(x); a.ldx = ldx;
  a.w = reinterpret_cast<const __nv_bfloat16*>(w); a.w_ts = w_ts; a.wsj = wsj; a.wsk = wsk;
  a.u = reinterpret_cast<__nv_bfloat16*>(u); a.ldu = ldu;
  a.M = M; a.T = T; a.rs = rs; a.kt = kt;
  for (int i = 0; i < 3; ++i) a.xoff[i] = i < T ? xoff[i] : 0;
  cudaError_t e = launch_pdl(lora_down_kernel, dim3((M + DOWN_ROWS - 1) / DOWN_ROWS), dim3(DOWN_THREADS), 0, stream, a);
  if (e != cudaSuccess) return static_cast<int>(e);
  return static_cast<int>(cudaGetLastError());
}

int b200_lora_grad(const void* l, long long ldl, const void* q, long long ldq, float* out, long long osa, long long osb,
                   long long out_ts, int M, int NA, int NB, int T, const long long* lo, const long long* qo, float s,
                   float* work, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0 || NA <= 0 || NB <= 0) return 0;
  if (T < 1 || T > 3) return -3;
  GradArgs g;
  g.l = reinterpret_cast<const __nv_bfloat16*>(l); g.ldl = ldl;
  g.q = reinterpret_cast<const __nv_bfloat16*>(q); g.ldq = ldq;
  g.M = M; g.NA = NA; g.NB = NB; g.S = (M + B200_LORA_SPLIT_ROWS - 1) / B200_LORA_SPLIT_ROWS;
  for (int i = 0; i < 3; ++i) { g.lo[i] = i < T ? lo[i] : 0; g.qo[i] = i < T ? qo[i] : 0; }
  g.work = work;
  const dim3 grid((NA + GRAD_A - 1) / GRAD_A, (NB + GRAD_B - 1) / GRAD_B, T * g.S);
  cudaError_t e = launch_pdl(lora_grad_partial_kernel, grid, dim3(GRAD_THREADS), 0, stream, g);
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long total = static_cast<long long>(NA) * NB * T;
  const int blocks = static_cast<int>(total < 256ll * 1024 ? (total + 255) / 256 : 1024);
  e = launch_pdl(lora_grad_finish_kernel, dim3(blocks), dim3(256), 0, stream, static_cast<const float*>(work), out, osa,
                 osb, out_ts, NA, NB, T, g.S, s);
  if (e != cudaSuccess) return static_cast<int>(e);
  return static_cast<int>(cudaGetLastError());
}
