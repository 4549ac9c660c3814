// Ground work for implicit-GEMM convolution: TMA *im2col* tensor maps (cuTensorMapEncodeIm2col) let the A
// operand of the forward conv GEMM (and the MN-major B operand of the wgrad GEMM) be gathered straight from the
// NHWC activation -- one filter tap x 64 channels x 128 output pixels per k-tile -- so the explicit im2col kernel
// and its 9x copy of the activation disappear.
//
// Recipe (same as the CUTLASS sm90/sm100 conv collectives, cute/atom/copy_traits_sm90_im2col.hpp):
//   tensor dims (C, W, H, N); bounding box lower corner = -pad, upper corner = pad - (filter - 1);
//   traversal strides = conv stride; the instruction takes the base pixel of the 128-pixel column in INPUT
//   coordinates (w = q*stride - pad, h = p*stride - pad) and the filter tap as 16-bit offsets (s, r);
//   out-of-image taps are zero-filled.  The result lands as [pixels x 64 channels] rows of 128 B with the 128 B
//   swizzle, i.e. exactly the K-major A tile gemm_wgmma.cu already consumes.
//
// This file only contains the encoder, the PTX wrapper and a PROBE kernel that dumps such tiles back to global
// memory in the layout of the explicit im2col kernel, so the semantics can be pinned down against it
// (tests/test_gpu_kernels.py::test_tma_im2col_probe_matches_explicit_im2col).
// Semantics probe only (not on any model path): it pins down the im2col-mode coordinate convention the implicit-GEMM
// convolution modes of gemm_wgmma.cu rely on.
#define B200_TU_TAG 5
#include <cuda.h>

#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"

namespace b200 {

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

static EncodeIm2colFn get_im2col_encode_fn() {
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);   // driver entry points need a current context on this thread
    ctx_bound = true;
  }
  static EncodeIm2colFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeIm2colFn>(ptr);
  }
  return fn;
}

// NHWC bf16 activation [N, H, W, C] -> im2col map loading `pixels` output pixels x `channels` channels per call
static int make_map_im2col(CUtensorMap* map, const void* x, int N, int H, int W, int C, int KH, int KW, int stride,
                           int pad, int channels, int pixels) {
  EncodeIm2colFn fn = get_im2col_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t gstr[3] = {static_cast<cuuint64_t>(C) * 2, static_cast<cuuint64_t>(W) * C * 2,
                        static_cast<cuuint64_t>(H) * W * C * 2};
  int lower[2] = {-pad, -pad};                               // {W, H}
  int upper[2] = {pad - (KW - 1), pad - (KH - 1)};
  cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride), static_cast<cuuint32_t>(stride), 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), gdim, gstr, lower, upper,
                  static_cast<cuuint32_t>(channels), static_cast<cuuint32_t>(pixels), estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// probe: CTA (m_tile, k_tile) loads one [128 pixels x 64 channels] im2col tile and writes it, un-swizzled, to
// col[M, KH*KW*C] (the explicit kernel's layout)
__global__ void __launch_bounds__(128)
im2col_tma_probe_kernel(const __grid_constant__ CUtensorMap tm, __nv_bfloat16* __restrict__ col, int N, int C, int KW,
                        int stride, int pad, int Ho, int Wo, long long M, int kp) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* tile = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(tile + 128 * 128);
  const long long m0 = static_cast<long long>(blockIdx.x) * 128;
  const int cblocks = C / 64;
  const int tap = blockIdx.y / cblocks, c0 = (blockIdx.y % cblocks) * 64;
  const int r = tap / KW, s = tap % KW;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int q0 = static_cast<int>(m0 % Wo);
    const int p0 = static_cast<int>((m0 / Wo) % Ho);
    const int n0 = static_cast<int>(m0 / (static_cast<long long>(Wo) * Ho));
    mbar_expect_tx(bar, 128 * 128);
    tma_load_im2col_4d(tile, &tm, bar, c0, q0 * stride - pad, p0 * stride - pad, n0, s, r);
  }
  mbar_wait(bar, 0);
  // thread = pixel row; undo the 128 B swizzle (16-byte chunk index ^ row % 8)
  const int row = threadIdx.x;
  if (m0 + row < M) {
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      const uint4 v = *reinterpret_cast<const uint4*>(tile + row * 128 + ((ch ^ (row & 7)) << 4));
      *reinterpret_cast<uint4*>(col + (m0 + row) * kp + static_cast<long long>(tap) * C + c0 + ch * 8) = v;
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_encode_map_im2col_bf16(void* map, const void* x, int N, int H, int W, int C, int KH, int KW,
                                            int stride, int pad, int channels, int pixels) {
  return make_map_im2col(reinterpret_cast<CUtensorMap*>(map), x, N, H, W, C, KH, KW, stride, pad, channels, pixels);
}

// col[M = N*Ho*Wo, kp = KH*KW*C] via TMA im2col loads (C % 64 == 0).  Returns -2 for unsupported shapes.
extern "C" int b200_im2col_tma_probe(const void* x, void* col, int N, int H, int W, int C, int KH, int KW, int stride,
                                     int pad, int Ho, int Wo, cudaStream_t stream) {
  if (C % 64 != 0 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(col) & 15)) return -2;
  const long long M = static_cast<long long>(N) * Ho * Wo;
  if (M <= 0) return 0;
  CUtensorMap tm;
  int rc = make_map_im2col(&tm, x, N, H, W, C, KH, KW, stride, pad, 64, 128);
  if (rc) return rc;
  const int kp = KH * KW * C;
  dim3 grid(static_cast<unsigned>((M + 127) / 128), static_cast<unsigned>(KH * KW * (C / 64)));
  im2col_tma_probe_kernel<<<grid, 128, 128 * 128 + 64 + 1024, stream>>>(tm, reinterpret_cast<__nv_bfloat16*>(col), N, C, KW,
                                                                        stride, pad, Ho, Wo, M, kp);
  return static_cast<int>(cudaGetLastError());
}

B200_TRACE_REGISTER(im2col_tma)
