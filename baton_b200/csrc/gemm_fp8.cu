// Block-scaled FP8 (MXFP8) GEMM on the Hopper tensor cores.
//
//     D[M,N] = act( alpha * (A .* SFA)[M,K] * (B .* SFB)[N,K]^T + bias[N] )
//
// A, B: e4m3, both K-major (row-major [rows, K]); SFA / SFB: one UE8M0 scale per 32 consecutive K
// elements of every row (OCP MX format), accumulate fp32.  The transposed operands that dgrad / wgrad need are
// produced (already quantised along THEIR reduction dimension) by the fused quantise+transpose kernels in quant.cu,
// so one K-major kernel serves forward, dgrad and wgrad.
//
// Hopper's FP8 wgmma has no block scaling, so each 32-element K block is one m64 x BN x 32 wgmma into a scratch
// accumulator, folded into the running one as  acc += sfa[row] * sfb[col] * scratch  (a power-of-two scale per
// element, exact).  For a 128-row x 128-K tile the 128 x 4 scale bytes are stored in global memory as one contiguous
// 512-byte ATOM  [row % 32][row / 32][k-block]; per pipeline stage the producer fetches the A and B atoms with a
// plain bulk copy next to the TMA tiles and the consumer warpgroups read their rows' / columns' bytes from shared
// memory.
//
// `block_scaled = 0` runs the same pipeline with plain e4m3 wgmma accumulating across the whole k-tile (per-tensor
// scales folded into alpha).
#define B200_TU_TAG 2
#include "ptx.cuh"
#include "launch.h"
#include "pdl.cuh"

namespace b200 {

constexpr int F8_BM = 128;
constexpr int F8_BK = 128;      // 128 e4m3 = 128 B = one swizzle row
constexpr int F8_WG_K = 32;     // K per wgmma for 8-bit operands
constexpr int F8_THREADS = 384;    // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue
constexpr int F8_CONSUMER_WARPS = 8;
constexpr int SF_ATOM = 512;    // bytes: 128 rows x 4 k-blocks

struct Fp8Params {
  int M, N, K;
  void* D;
  long long ldd;
  const float* bias;
  int out_fp32, act, atomic_out, block_scaled;
  const uint8_t* sfa;   // [ceil(M/128)][k_tiles][512]
  const uint8_t* sfb;   // [ceil(N/128)][k_tiles][512]
  float alpha;
};

template <int BN>
struct F8Smem {
  static constexpr int A_BYTES = F8_BM * F8_BK;
  static constexpr int B_BYTES = BN * F8_BK;
  static constexpr int SFB_ATOMS = (BN + 127) / 128;
  static constexpr int SF_BYTES = SF_ATOM * (1 + SFB_ATOMS);
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES + 1024;   // + scale atoms (padded to keep 1024B alignment)
  static constexpr int TMA_BYTES = A_BYTES + B_BYTES;
};

__device__ __forceinline__ float f8_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    return 0.5f * v * (1.f + tanhf(k0 * (v + k1 * v * v * v)));
  }
  return v;
}

// 1-D bulk copy global -> shared, completing `bytes` on an mbarrier (scale-factor atoms)
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// position of the scale byte of (row, 32-element K block kb) inside a 512-byte atom [row % 32][row / 32][kb]
__device__ __forceinline__ int sf_index(int row, int kb) { return (row & 31) * 16 + (row >> 5) * 4 + kb; }
// UE8M0: a bare biased exponent, 2^(e - 127)
__device__ __forceinline__ float ue8m0(uint8_t e) { return __uint_as_float(static_cast<uint32_t>(e) << 23); }
template <int N>
__device__ __forceinline__ void wgmma_e4m3(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (N == 64) wgmma_e4m3_n64(d, da, db, scale_d);
  else wgmma_e4m3_n128(d, da, db, scale_d);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Fp8Params p) {
  using L = F8Smem<BN>;
  constexpr int PITCH = BN + 4;                      // fp32 pitch of the staged accumulator tile
  static_assert(STAGES * L::STAGE_BYTES >= F8_BM * PITCH * 4, "the drained ring must hold the fp32 accumulator tile");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int m0 = blockIdx.y * F8_BM;
  const int n0 = blockIdx.x * BN;
  const int k_tiles = (p.K + F8_BK - 1) / F8_BK;
  const int per = (k_tiles + gridDim.z - 1) / gridDim.z;
  const int kt_begin = blockIdx.z * per;
  int kt_end = kt_begin + per;
  if (kt_end > k_tiles) kt_end = k_tiles;
  const int num_kt = kt_end - kt_begin;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], F8_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();

  if (warp == 0) {
    if (elect_one()) {
      for (int i = 0; i < num_kt; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * L::STAGE_BYTES;
        uint8_t* sb = sa + L::A_BYTES;
        uint8_t* ssf = sb + L::B_BYTES;
        const int kt = kt_begin + i;
        mbar_expect_tx(&full_bar[s], L::TMA_BYTES + (p.block_scaled ? L::SF_BYTES : 0));
        tma_load_2d(sa, &tmA, &full_bar[s], kt * F8_BK, m0);
        tma_load_2d(sb, &tmB, &full_bar[s], kt * F8_BK, n0);
        if (p.block_scaled) {
          bulk_load(ssf, p.sfa + (static_cast<size_t>(blockIdx.y) * k_tiles + kt) * SF_ATOM, SF_ATOM, &full_bar[s]);
#pragma unroll
          for (int j = 0; j < L::SFB_ATOMS; ++j)
            bulk_load(ssf + SF_ATOM * (1 + j),
                      p.sfb + (static_cast<size_t>(n0 / 128 + j) * k_tiles + kt) * SF_ATOM, SF_ATOM, &full_bar[s]);
        }
      }
    }
  } else if (warp >= 4) {
    const int ew = warp - 4, g = ew >> 2;            // warpgroup g: rows 64 g .. 64 g + 63 of the tile
    const int lane = static_cast<int>(lane_id());
    const int fr0 = 64 * g + 16 * (ew & 3) + (lane >> 2);   // fragment rows fr0, fr0 + 8; columns 8 i + 2 (lane % 4) + e
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    for (int i = 0; i < num_kt; ++i) {
      const int s = i % STAGES;
      const uint32_t ph = (i / STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES) + g * 8192;   // 64 rows x 128 B
      const uint32_t sb = smem_u32(smem + s * L::STAGE_BYTES + L::A_BYTES);
      if (p.block_scaled) {
        // one K = 32 block at a time: tmp = A_kb B_kb^T, then acc += sfa[row, kb] * sfb[col, kb] * tmp
        const uint8_t* ssf = smem + s * L::STAGE_BYTES + L::A_BYTES + L::B_BYTES;
#pragma unroll 1
        for (int kb = 0; kb < F8_BK / F8_WG_K; ++kb) {
          float tmp[BN / 2];
          wgmma_fence();
          wgmma_e4m3<BN>(tmp, gmma_desc_sw128(sa + kb * 32, 16, 1024), gmma_desc_sw128(sb + kb * 32, 16, 1024), 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operands(tmp);
          const float sa0 = ue8m0(ssf[sf_index(fr0, kb)]), sa1 = ue8m0(ssf[sf_index(fr0 + 8, kb)]);
#pragma unroll
          for (int c8 = 0; c8 < BN / 8; ++c8) {
            const int col = 8 * c8 + 2 * (lane & 3);
            const float sb0 = ue8m0(ssf[SF_ATOM + sf_index(col, kb)]), sb1 = ue8m0(ssf[SF_ATOM + sf_index(col + 1, kb)]);
            acc[4 * c8] = fmaf(sa0 * sb0, tmp[4 * c8], acc[4 * c8]);
            acc[4 * c8 + 1] = fmaf(sa0 * sb1, tmp[4 * c8 + 1], acc[4 * c8 + 1]);
            acc[4 * c8 + 2] = fmaf(sa1 * sb0, tmp[4 * c8 + 2], acc[4 * c8 + 2]);
            acc[4 * c8 + 3] = fmaf(sa1 * sb1, tmp[4 * c8 + 3], acc[4 * c8 + 3]);
          }
        }
      } else {
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < F8_BK / F8_WG_K; ++kb)
          wgmma_e4m3<BN>(acc, gmma_desc_sw128(sa + kb * 32, 16, 1024), gmma_desc_sw128(sb + kb * 32, 16, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
      }
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }
    named_bar_sync(1, F8_CONSUMER_WARPS * 32);       // both warpgroups are done with the ring: stage the accumulator
    float* part = reinterpret_cast<float*>(smem);
    wg_store_acc<BN>(acc, part, PITCH, 64 * g);
    named_bar_sync(1, F8_CONSUMER_WARPS * 32);
    const int q = ew & 3;
    const int row = m0 + q * 32 + lane;
    const bool row_ok = row < p.M;
    const size_t elt = p.out_fp32 ? 4 : 2;
    uint8_t* drow = reinterpret_cast<uint8_t*>(p.D) + static_cast<size_t>(row) * p.ldd * elt;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && ((p.ldd * elt) % 16 == 0);
#pragma unroll 1
    for (int c = g * 32; c < BN; c += 64) {          // the two warps of a row quarter take alternate 32-column chunks
      uint32_t r[32];
      acc_ld_row32(part + (q * 32 + lane) * PITCH + c, r);
      const int col0 = n0 + c;
      if (!row_ok || col0 >= p.N) continue;
      float v[32];
      // (bias, activation) resolved once per chunk by warp-uniform branches, then straight-line code
      if (p.bias != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          v[j] = fmaf(__uint_as_float(r[j]), p.alpha, (col0 + j) < p.N ? __ldg(p.bias + col0 + j) : 0.f);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]) * p.alpha;
      }
      if (p.act == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
      } else if (p.act != 0) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = f8_act(v[j], p.act);
      }
      const bool full = (col0 + 32 <= p.N);
      if (p.out_fp32) {
        float* d = reinterpret_cast<float*>(drow) + col0;
        if (p.atomic_out) {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) atomicAdd(d + j, v[j]);
        } else if (full && vec_ok) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(d + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
        } else {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) d[j] = v[j];
        }
      } else {
        __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(drow) + col0;
        if (full && vec_ok) {
#pragma unroll
          for (int j = 0; j < 32; j += 8)
            *reinterpret_cast<uint4*>(d + j) = make_uint4(pack_bf16x2(v[j], v[j + 1]), pack_bf16x2(v[j + 2], v[j + 3]),
                                                          pack_bf16x2(v[j + 4], v[j + 5]), pack_bf16x2(v[j + 6], v[j + 7]));
        } else {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) d[j] = __float2bfloat16_rn(v[j]);
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn8)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn8 encode8() {
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  static EncodeTiledFn8 fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn8>(ptr);
  }
  return fn;
}
static int make_map8(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, int box_rows) {
  EncodeTiledFn8 fn = encode8();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(F8_BK), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

template <int BN, int STAGES>
static int launch8(const CUtensorMap& ta, const CUtensorMap& tb, const Fp8Params& p, dim3 grid, cudaStream_t stream) {
  constexpr int smem = STAGES * F8Smem<BN>::STAGE_BYTES + (2 * STAGES + 1) * 8 + 16 + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_fp8_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  cudaError_t le = launch_pdl(gemm_fp8_kernel<BN, STAGES>, grid, F8_THREADS, smem, stream, ta, tb, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace b200

// a: e4m3 [M, K] pitch lda (bytes == elements), b: e4m3 [N, K] pitch ldb; sfa/sfb: scale atoms (see above) or
// nullptr for the unscaled kind::f8f6f4 path.  Pitches must be multiples of 16.
extern "C" int b200_gemm_fp8(const void* a, const void* b, void* d, const float* bias, const void* sfa, const void* sfb,
                             int M, int N, int K, long long lda, long long ldb, long long ldd, int out_fp32, int act,
                             int split_k, int accumulate, float alpha, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 16) || (ldb % 16) || (reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15))
    return -2;
  // the 128-row scale atoms fix the N tile of the block-scaled path at 128
  const int bn = (N > 64 || (sfa != nullptr && sfb != nullptr)) ? 128 : 64;
  CUtensorMap ta, tb;
  int rc = make_map8(&ta, a, M, K, lda, F8_BM);
  if (rc) return rc;
  rc = make_map8(&tb, b, N, K, ldb, bn);
  if (rc) return rc;
  Fp8Params p;
  p.M = M; p.N = N; p.K = K; p.D = d; p.ldd = ldd; p.bias = bias; p.out_fp32 = out_fp32; p.act = act;
  p.block_scaled = (sfa != nullptr && sfb != nullptr) ? 1 : 0;
  p.sfa = reinterpret_cast<const uint8_t*>(sfa);
  p.sfb = reinterpret_cast<const uint8_t*>(sfb);
  p.alpha = alpha;
  const int k_tiles = (K + F8_BK - 1) / F8_BK;
  if (split_k < 1) split_k = 1;
  if (split_k > k_tiles) split_k = k_tiles;
  const int per = (k_tiles + split_k - 1) / split_k;
  split_k = (k_tiles + per - 1) / per;
  p.atomic_out = (accumulate || split_k > 1) ? 1 : 0;
  if (p.atomic_out && (!out_fp32 || bias != nullptr || act != 0)) return -3;
  dim3 grid((N + bn - 1) / bn, (M + F8_BM - 1) / F8_BM, split_k);
  if (bn == 128) return launch8<128, 5>(ta, tb, p, grid, stream);
  return launch8<64, 6>(ta, tb, p, grid, stream);
}

B200_TRACE_REGISTER(gemm_fp8)
