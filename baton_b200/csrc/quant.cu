// MXFP8 quantisation for the block-scaled tensor-core path (OCP microscaling: e4m3 elements, one
// UE8M0 power-of-two scale per 32 consecutive elements ALONG THE REDUCTION DIMENSION of the GEMM
// that will consume the tensor).
//
//   quant_mx_rows : x[R, C] bf16  ->  q[R, Cp] e4m3, scales along C      (operand of a GEMM reducing over C)
//   quant_mx_cols : x[R, C] bf16  ->  q[C, Rp] e4m3 (TRANSPOSED), scales along R
//                                                       (operand of a GEMM reducing over R: dgrad / wgrad)
//
// Scales are written directly in the 512-byte atom layout gemm_fp8.cu reads:
//   atom(row_tile, k_tile)[ (row % 32) * 16 + ((row % 128) / 32) * 4 + (k % 128) / 32 ]
#define B200_TU_TAG 3
#include <cuda_fp8.h>

#include "launch.h"
#include "mx.cuh"
#include "pdl.cuh"
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ size_t sf_offset(long long row, long long k, long long k_tiles) {
  return (static_cast<size_t>(row >> 7) * k_tiles + (k >> 7)) * 512 + (row & 31) * 16 + ((row & 127) >> 5) * 4 +
         ((k & 127) >> 5);
}

// one thread = 8 consecutive elements of a row; 4 threads share a 32-element block
__global__ void __launch_bounds__(256)
quant_mx_rows_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf,
                     long long R, int C, long long ld_in, int Cp, long long Rpad, int Cpad) {
  griddep_launch_dependents();
  griddep_wait();
  const int vec_per_row = Cpad >> 3;
  const long long total = Rpad * vec_per_row;
  const long long k_tiles = Cpad >> 7;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vec_per_row;
    const int c0 = static_cast<int>(i - r * vec_per_row) << 3;
    float v[8];
    const bool in_row = r < R;
    if (in_row && c0 + 8 <= C && (ld_in & 7) == 0) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + r * ld_in + c0);
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (in_row && c0 + j < C) ? __bfloat162float(x[r * ld_in + c0 + j]) : 0.f;
    }
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
    // the 4 threads of a 32-element block are adjacent lanes (vec_per_row is a multiple of 16)
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const int e = mx_exponent(amax);
    const float inv = exp2_int(-e);
    if (in_row && c0 < Cp) {
      uint4 o;
      o.x = to_e4m3x2(v[0] * inv, v[1] * inv) | (static_cast<uint32_t>(to_e4m3x2(v[2] * inv, v[3] * inv)) << 16);
      o.y = to_e4m3x2(v[4] * inv, v[5] * inv) | (static_cast<uint32_t>(to_e4m3x2(v[6] * inv, v[7] * inv)) << 16);
      *reinterpret_cast<uint2*>(q + r * Cp + c0) = make_uint2(o.x, o.y);
    }
    if (((c0 >> 3) & 3) == 0) sf[sf_offset(r, c0, k_tiles)] = static_cast<uint8_t>(e + 127);
  }
}

// block = 128 threads, tile = 32 rows (R) x 128 columns (C); thread c owns one output row (= input column)
__global__ void __launch_bounds__(128)
quant_mx_cols_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf,
                     long long R, int C, long long ld_in, long long Rp, long long Rpad, int Cpad) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float tile[32][129];
  const long long r0 = static_cast<long long>(blockIdx.y) * 32;
  const int c0 = blockIdx.x * 128;
  // coalesced load: 128 threads sweep the 32 x 128 tile row by row
  for (int rr = 0; rr < 32; ++rr) {
    const long long r = r0 + rr;
    const int c = c0 + threadIdx.x;
    tile[rr][threadIdx.x] = (r < R && c < C) ? __bfloat162float(x[r * ld_in + c]) : 0.f;
  }
  __syncthreads();
  const int c = c0 + threadIdx.x;          // output row
  float amax = 0.f;
#pragma unroll
  for (int rr = 0; rr < 32; ++rr) amax = fmaxf(amax, fabsf(tile[rr][threadIdx.x]));
  const int e = mx_exponent(amax);
  const float inv = exp2_int(-e);
  const long long k_tiles = Rpad >> 7;
  if (c < Cpad) sf[sf_offset(c, r0, k_tiles)] = static_cast<uint8_t>(e + 127);
  if (c < C && r0 < Rp) {
    uint32_t w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      w[j] = to_e4m3x2(tile[4 * j][threadIdx.x] * inv, tile[4 * j + 1][threadIdx.x] * inv) |
             (static_cast<uint32_t>(to_e4m3x2(tile[4 * j + 2][threadIdx.x] * inv, tile[4 * j + 3][threadIdx.x] * inv)) << 16);
    uint8_t* dst = q + static_cast<long long>(c) * Rp + r0;
    if (r0 + 32 <= Rp) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
      *reinterpret_cast<uint4*>(dst + 16) = make_uint4(w[4], w[5], w[6], w[7]);
    } else {
      for (int j = 0; j < 32 && r0 + j < Rp; ++j) dst[j] = static_cast<uint8_t>((w[j >> 2] >> (8 * (j & 3))) & 0xFF);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_quant_mx_rows(const void* x, void* q, void* sf, long long R, int C, long long ld_in, int Cp,
                                  cudaStream_t stream) {
  if (R <= 0 || C <= 0) return 0;
  const long long Rpad = (R + 127) / 128 * 128;
  const int Cpad = (C + 127) / 128 * 128;
  long long blocks = (Rpad * (Cpad / 8) + 255) / 256;
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  launch_pdl(quant_mx_rows_kernel, static_cast<unsigned>(blocks), 256, 0, stream,
             reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<uint8_t*>(q), reinterpret_cast<uint8_t*>(sf), R, C,
             ld_in, Cp, Rpad, Cpad);
  return static_cast<int>(cudaGetLastError());
}
extern "C" int b200_quant_mx_cols(const void* x, void* q, void* sf, long long R, int C, long long ld_in, long long Rp,
                                  cudaStream_t stream) {
  if (R <= 0 || C <= 0) return 0;
  const long long Rpad = (R + 127) / 128 * 128;
  const int Cpad = (C + 127) / 128 * 128;
  dim3 grid(Cpad / 128, static_cast<unsigned>(Rpad / 32));
  launch_pdl(quant_mx_cols_kernel, grid, 128, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
             reinterpret_cast<uint8_t*>(q), reinterpret_cast<uint8_t*>(sf), R, C, ld_in, Rp, Rpad, Cpad);
  return static_cast<int>(cudaGetLastError());
}

B200_TRACE_REGISTER(quant)
