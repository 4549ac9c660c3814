// Halo-tiled implicit GEMM for 3x3, pad-1 convolutions (ResNet layer1 and layer2), forward and input gradient.
//
// The im2col-mode kernels (gemm_wgmma.cu CONV 1 / 3) issue one TMA im2col load per filter tap, so every input pixel
// crosses L2 -> SM nine times, and every CTA loads all the weight k-tiles for itself.  Here a CTA owns BM = 64 output
// pixels = 64 / (Ho Wo) whole images and a 64-column block of the output (blockIdx.x), and loads
//   * the halo of those images ONCE: one tiled 4-D TMA box {64 ch, STRIDE (Wo - 1) + 3, STRIDE (Ho - 1) + 3, images}
//     per 64-channel block of the gathered tensor, starting at (64 cb, -1, -1, n0); the out-of-bounds zero fill is the
//     padding;
//   * the 9 CB [64 x 64] weight k-tiles of its column block, each into its own slot with its own mbarrier (no ring, no
//     slot reuse), split by rows over a cluster of `mc` CTAs along M: each CTA multicasts its slice into every member.
// The A fragments of each k-tile are gathered from the halo with ldmatrix (lane -> halo pixel
// (img, STRIDE i + r, STRIDE j + s)) and feed wgmma with A in registers; the ldmatrix of k-tile kt + 1 overlaps the
// MMAs of k-tile kt.  The k order -- tap-major, then channel block, then 4 x k16, kt = tap * CB + cb -- is that of the
// im2col-mode kernels, so the accumulator equals theirs with cluster split-K 1 bit for bit.
//
// Template parameters:
//   DGRAD   false: y [N Ho Wo, Cout] = conv(x, w); B = w [Cout, 9 C] K-major, k-tile kt = columns [64 kt, 64 kt + 64)
//           true:  dx [N H W, Cin] = conv(dy, flipped w), stride 1 only; B = the [64 cout] x [64 cin] slab of tap
//                  8 - tap and cout block cb, MN-major
//   CB      64-channel blocks of the gathered tensor (x forward, dy dgrad): CB halo boxes, 9 CB k-tiles
//   STRIDE  1 or 2 (forward only)
//
// Warp roles (256 threads): warp 0 = loads (one elected lane), warpgroup 1 = the m64 x 64 MMAs, then the row-per-lane
// epilogue of the fixed-depth GEMM with the fused BatchNorm column statistics.  A 64-row tile (rather than the GEMM
// kernels' 128) gives a layer1 GEMM 128 CTAs instead of 64: the tensor-core time of a CTA is about a microsecond at
// 128 rows, and half the SMs would sit idle.
#define B200_TU_TAG 12
#include "ptx.cuh"
#include "epilogue.cuh"
#include "launch.h"
#include "pdl.cuh"

namespace b200 {

constexpr int HALO_BM = 64;
constexpr int HALO_BN = 64;
constexpr int HALO_TAPS = 9;
constexpr int HALO_THREADS = 256;
constexpr int HALO_CONSUMERS = 128;
constexpr int HALO_SLOT_BYTES = 64 * 64 * 2;        // one weight k-tile
constexpr int HALO_PART_PITCH = HALO_BN + 4;        // floats; +4 keeps float4 alignment, skews banks
constexpr int HALO_MAX_SMEM = 227 * 1024;

struct HaloParams {
  int M, N;              // GEMM rows (output pixels) and columns (output channels)
  int Ho, Wo;            // output image size
  __nv_bfloat16* D;      // [M, N] bf16
  float* col_stats;      // optional [2N]: += column sums / sums of squares of the bf16 output (BatchNorm)
  int ncol;              // dgrad: Cin, the column pitch of one tap inside a weight row
  int mc;                // CTAs of a cluster along M sharing the weight k-tiles (1, 2, 4, 8)
  int halo_bytes;        // one channel block's halo box bytes rounded up to 1024 (the boxes and B slots stay aligned)
};

// mbarriers: [0] halo, [1 + kt] slot of k-tile kt, padded to a multiple of 16 (128 B at 9 k-tiles, 256 B at 18)
__host__ __device__ constexpr int halo_barriers(int k_tiles) { return (1 + k_tiles + 15) / 16 * 16; }

__host__ __device__ constexpr int halo_fixed_bytes(int k_tiles) {
  // slots, barriers, statistics, realignment
  return k_tiles * HALO_SLOT_BYTES + halo_barriers(k_tiles) * 8 + 4 * HALO_BN * 4 + 1024;
}

template <bool DGRAD, int CB, int STRIDE>
__global__ void __launch_bounds__(HALO_THREADS, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const HaloParams p) {
  constexpr int KT = HALO_TAPS * CB;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* halo = smem;                                                                 // [CB][halo_bytes]
  uint8_t* bslot = smem + CB * p.halo_bytes;
  uint64_t* bar = reinterpret_cast<uint64_t*>(bslot + KT * HALO_SLOT_BYTES);   // [0] halo, [1 + kt] slot of k-tile kt
  float* cstat = reinterpret_cast<float*>(bar + halo_barriers(KT));              // [2 row halves][2 * BN]

  griddep_launch_dependents();  // PDL: the next kernel may start its prologue now
  const int warp = threadIdx.x >> 5;
  const int m0 = blockIdx.y * HALO_BM;
  const int n0 = blockIdx.x * HALO_BN;
  const int hw = p.Ho * p.Wo;
  const int hp = STRIDE * (p.Ho - 1) + 3, wp = STRIDE * (p.Wo - 1) + 3;   // halo box of one image

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < 1 + KT; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (p.mc > 1) cluster_sync_all();   // no peer multicasts into a barrier before it is initialised
  griddep_wait();  // PDL: everything above overlapped the previous kernel; its results are visible from here

  if (warp == 0) {
    if (elect_one()) {
      // ---- all loads up front: the CB halo boxes, then the weight k-tiles (this CTA's rows of each, multicast) ----
      const int imgs = HALO_BM / hw;
      mbar_expect_tx(&bar[0], CB * imgs * hp * wp * 128);
#pragma unroll
      for (int cb = 0; cb < CB; ++cb) tma_load_4d(halo + cb * p.halo_bytes, &tmX, &bar[0], 64 * cb, -1, -1, m0 / hw);
      const int rows = 64 / p.mc;
      const int rank = p.mc > 1 ? static_cast<int>(cluster_ctarank()) : 0;
      const uint16_t mask = static_cast<uint16_t>((1u << p.mc) - 1);
      // every member's slot barrier expects the whole k-tile; a CTA whose rows all lie past M still issues its slice
#pragma unroll 1
      for (int kt = 0; kt < KT; ++kt) {
        const int tap = kt / CB, cb = kt - tap * CB;
        mbar_expect_tx(&bar[1 + kt], HALO_SLOT_BYTES);
        uint8_t* dst = bslot + kt * HALO_SLOT_BYTES + rank * rows * 128;
        const int c0 = DGRAD ? (HALO_TAPS - 1 - tap) * p.ncol + n0 : kt * 64;
        const int c1 = DGRAD ? cb * 64 + rank * rows : n0 + rank * rows;
        if (p.mc > 1)
          tma_load_2d_mc(dst, &tmW, &bar[1 + kt], c0, c1, mask);
        else
          tma_load_2d(dst, &tmW, &bar[1 + kt], c0, c1);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers =====================
    const int ew = warp - 4;                   // 0..3: rows [16 ew, 16 ew + 16) of the MMA fragment
    const int lane = static_cast<int>(lane_id());
    // ldmatrix.x4 address of this lane: row (lane & 15) of the warp's 16, channel half (lane >> 4) of each k16 step
    const int m = 16 * ew + (lane & 15);
    const int img = m / hw, rem = m - img * hw;
    const int oi = rem / p.Wo, oj = rem - oi * p.Wo;
    const int hrow0 = (img * hp + STRIDE * oi) * wp + STRIDE * oj;   // halo pixel of tap (0, 0)
    const uint32_t halo_a = smem_u32(halo);
    const int half = lane >> 4;
    // 128B swizzle of each halo box (1024-aligned): 16-byte chunk c of halo pixel (= box row) r sits at chunk
    // c ^ (r & 7); eight consecutive output columns hit eight different chunks (conflict-free at stride 1)
    auto load_a = [&](uint32_t (&a)[4][4], int kt) {
      const int tap = kt / CB, cb = kt - tap * CB;
      const int r = tap / 3, s = tap - 3 * r;
      const int hrow = hrow0 + r * wp + s;
      const uint32_t row_addr = halo_a + static_cast<uint32_t>(cb * p.halo_bytes + hrow * 128);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) ldmatrix_x4(a[kk], row_addr + ((((2 * kk + half) ^ hrow) & 7) << 4));
    };

    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    uint32_t a[2][4][4];
    mbar_wait(&bar[0], 0);
    load_a(a[0], 0);
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
      mbar_wait(&bar[1 + kt], 0);
      const uint32_t sb = smem_u32(bslot + kt * HALO_SLOT_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        // K-major B: K advance = 32 B inside the swizzle row; MN-major B: 16 k rows = 2048 B
        const uint64_t bd = DGRAD ? gmma_desc_sw128(sb + kk * 2048, 8192, 1024) : gmma_desc_sw128(sb + kk * 32, 16, 1024);
        wgmma_bf16_n64_rs<DGRAD ? 1 : 0>(acc, a[kt & 1][kk], bd, 1u);
      }
      wgmma_commit();
      if (kt + 1 < KT) {
        wgmma_wait<1>();                       // the MMAs of k-tile kt - 1 have read a[(kt + 1) & 1]
        load_a(a[(kt + 1) & 1], kt + 1);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (threadIdx.x == 128) TRACE_POINT();  // halo: accumulator complete (epilogue starts)

    // ---- epilogue: park the tile over the idle halo / B area, then one row per lane ----
    named_bar_sync(1, HALO_CONSUMERS);         // every warp's MMAs retired: the halo / B area may be overwritten
    float* part = reinterpret_cast<float*>(smem);
    wg_store_acc<HALO_BN>(acc, part, HALO_PART_PITCH, 0);
    named_bar_sync(1, HALO_CONSUMERS);
    const int q = ew & 1;                      // row half
    const int c = (ew >> 1) * 32;              // the two warps of a half take one 32-column chunk each
    const int lrow = q * 32 + lane;
    const int row = m0 + lrow;
    const int col0 = n0 + c;
    float* sstat = cstat + q * 2 * HALO_BN;
    const bool want_stats = p.col_stats != nullptr;
    if (col0 >= p.N) {                         // warp-uniform
      if (want_stats) { sstat[c + lane] = 0.f; sstat[HALO_BN + c + lane] = 0.f; }
    } else {
      uint32_t r[32];
      acc_ld_row32(part + lrow * HALO_PART_PITCH + c, r);
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
      // rows past M hold exact zeros (the halo of images past N is zero-filled): they add nothing to the sums
      if (want_stats) stage_col_stats(sstat, HALO_BN, c, v);
      if (row < p.M) {
        __nv_bfloat16* d = p.D + static_cast<size_t>(row) * p.N + col0;
        if (col0 + 32 <= p.N && (p.N % 8) == 0) {
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            uint4 o;
            o.x = pack_bf16x2(v[j], v[j + 1]);
            o.y = pack_bf16x2(v[j + 2], v[j + 3]);
            o.z = pack_bf16x2(v[j + 4], v[j + 5]);
            o.w = pack_bf16x2(v[j + 6], v[j + 7]);
            *reinterpret_cast<uint4*>(d + j) = o;
          }
        } else {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) d[j] = __float2bfloat16_rn(v[j]);
        }
      }
    }
    if (want_stats) {
      named_bar_sync(1, HALO_CONSUMERS);       // all four warps staged their column sums
      for (int i = threadIdx.x - 128; i < 2 * HALO_BN; i += HALO_CONSUMERS) {
        const int col = i < HALO_BN ? i : i - HALO_BN;
        if (n0 + col < p.N)
          atomicAdd(p.col_stats + (i < HALO_BN ? 0 : p.N) + n0 + col,
                    cstat[i] + cstat[2 * HALO_BN + i]);
      }
    }
  }
  // No cluster barrier before exit: peers only write into this CTA's slots, and it has waited for every byte of them.
}

// launch of one instantiation: PDL, and a cluster of p.mc CTAs along M
template <auto KERNEL>
static int launch_halo(const CUtensorMap& tx, const CUtensorMap& tw, const HaloParams& p, dim3 grid, int smem,
                       cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         HALO_MAX_SMEM);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(HALO_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (p.mc > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = 1;
    attr[na].val.clusterDim.y = p.mc;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t le = cudaLaunchKernelEx(&cfg, KERNEL, tx, tw, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace b200

extern "C" int b200_encode_map2_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     int box_cols, int box_rows);
extern "C" int b200_encode_map4_box_bf16(void* map, const void* base, const long long* dims,
                                         const long long* stride_bytes, const int* box);

// src [N, H, W, C] NHWC bf16 (x forward, dy dgrad); w [Cout, 9 * Cin] channels_last; out [N Ho Wo, Nout] bf16 with
// Nout = Cout forward, Cin dgrad.  Instantiated (stride, C): (1, 64) and (1, 128) forward and dgrad, (2, 64) forward.
// mc: cluster size along M (1, 2, 4, 8; must divide the number of 64-row tiles).  col_stats (forward only): optional
// [2 Nout] fp32.  Returns 0, a CUDA / driver error code, or -2 when the shape is not one the kernel takes.
extern "C" int b200_conv_halo(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout,
                              int stride, int dgrad, int mc, float* col_stats, cudaStream_t stream) {
  using namespace b200;
  const bool s1c64 = stride == 1 && C == 64, s1c128 = stride == 1 && C == 128, s2c64 = stride == 2 && C == 64 && !dgrad;
  if (!s1c64 && !s1c128 && !s2c64) return -2;
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;      // 3x3, pad 1
  const long long M = static_cast<long long>(N) * Ho * Wo;
  if (M <= 0 || Nout <= 0) return 0;
  const int hw = Ho * Wo;
  const long long m_tiles = (M + HALO_BM - 1) / HALO_BM;
  const int hp = stride * (Ho - 1) + 3, wp = stride * (Wo - 1) + 3;
  if (H <= 0 || W <= 0 || HALO_BM % hw != 0 || hp > 256 || wp > 256 || M > (1ll << 30) || Nout % 8 != 0 ||
      (dgrad && Nout % 64 != 0) || (mc != 1 && mc != 2 && mc != 4 && mc != 8) || m_tiles % mc != 0 ||
      (reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(w) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return -2;
  const int imgs = HALO_BM / hw;
  const int cb = C / 64;
  const int halo_bytes = (imgs * hp * wp * 128 + 1023) / 1024 * 1024;
  const int smem = cb * halo_bytes + halo_fixed_bytes(HALO_TAPS * cb);
  if (smem > HALO_MAX_SMEM) return -2;
  CUtensorMap tx, tw;
  const long long dims[4] = {C, W, H, N};
  const long long strides[3] = {static_cast<long long>(C) * 2, static_cast<long long>(W) * C * 2,
                                static_cast<long long>(H) * W * C * 2};
  const int box[4] = {64, wp, hp, imgs};
  int rc = b200_encode_map4_box_bf16(&tx, src, dims, strides, box);
  if (rc) return rc;
  // weight slices: 64 / mc rows of a 64-column box (forward: Cout rows of 9 C columns; dgrad: C = Cout rows of 9 Cin)
  const long long wrows = dgrad ? C : Nout, wcols = dgrad ? 9ll * Nout : 9ll * C;
  rc = b200_encode_map2_bf16(&tw, w, wrows, wcols, wcols, 64, 64 / mc);
  if (rc) return rc;
  HaloParams p;
  p.M = static_cast<int>(M); p.N = Nout; p.Ho = Ho; p.Wo = Wo; p.D = reinterpret_cast<__nv_bfloat16*>(out);
  p.col_stats = col_stats; p.ncol = Nout; p.mc = mc; p.halo_bytes = halo_bytes;
  dim3 grid((Nout + HALO_BN - 1) / HALO_BN, static_cast<unsigned>(m_tiles), 1);
  if (s2c64) return launch_halo<conv_halo_kernel<false, 1, 2>>(tx, tw, p, grid, smem, stream);
  if (s1c64)
    return dgrad ? launch_halo<conv_halo_kernel<true, 1, 1>>(tx, tw, p, grid, smem, stream)
                 : launch_halo<conv_halo_kernel<false, 1, 1>>(tx, tw, p, grid, smem, stream);
  return dgrad ? launch_halo<conv_halo_kernel<true, 2, 1>>(tx, tw, p, grid, smem, stream)
               : launch_halo<conv_halo_kernel<false, 2, 1>>(tx, tw, p, grid, smem, stream);
}

B200_TRACE_REGISTER(conv_halo)
