// Halo-tiled implicit GEMM for 3x3, pad-1 convolutions (ResNet layer1 and layer2; layer3 in image mode, below), forward
// and input gradient.
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
//   BN      output columns of a CTA: 64, or 32 (the layer3 forms, whose 36 weight k-tiles fit only at 32 columns)
//   IMG     false: halo mode (above).  true: image mode, for small maps whose halo would be several times the image
//           (a 2x2 map's is 4x4): the box is the images alone, {64, W, H, images} at (64 cb, 0, 0, n0), and a lane
//           whose tap falls outside its image points its ldmatrix at a 16-byte zero line.  All nine taps stay in the
//           k loop, so the k order, and the result, are those of the halo mode and of the im2col-mode kernels.
//
// Warp roles (256 threads): warp 0 = loads (one elected lane), warpgroup 1 = the m64 x BN MMAs, then the row-per-lane
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
constexpr int HALO_MAX_SMEM = 227 * 1024;
constexpr int HALO_ZERO_BYTES = 128;                // image mode: the zero line of out-of-image taps

struct HaloParams {
  int M, N;              // GEMM rows (output pixels) and columns (output channels)
  int Ho, Wo;            // output image size
  __nv_bfloat16* D;      // [M, N] bf16
  float* col_stats;      // optional [2N]: += column sums / sums of squares of the bf16 output (BatchNorm)
  int ncol;              // dgrad: Cin, the column pitch of one tap inside a weight row
  int mc;                // CTAs of a cluster along M sharing the weight k-tiles (1, 2, 4, 8)
  int halo_bytes;        // one channel block's box bytes rounded up to 1024 (the boxes and B slots stay aligned)
  int bh, bw;            // box height and width of one image: the halo (STRIDE (Ho - 1) + 3) or the image (H, W)
};

// mbarriers: [0] halo, [1 + kt] slot of k-tile kt, padded to a multiple of 16 (128 B at 9 k-tiles, 256 B at 18)
__host__ __device__ constexpr int halo_barriers(int k_tiles) { return (1 + k_tiles + 15) / 16 * 16; }

// one weight k-tile: [BN cout] x [64 k] K-major (forward) or [64 cout] x [BN cin] MN-major (dgrad)
__host__ __device__ constexpr int halo_slot_bytes(int bn) { return bn * 64 * 2; }

__host__ __device__ constexpr int halo_fixed_bytes(int k_tiles, int bn = HALO_BN, bool img = false) {
  // slots, barriers, statistics, zero line, realignment
  return k_tiles * halo_slot_bytes(bn) + halo_barriers(k_tiles) * 8 + 4 * bn * 4 + (img ? HALO_ZERO_BYTES : 0) + 1024;
}

template <bool DGRAD, int CB, int STRIDE, int BN = HALO_BN, bool IMG = false>
__global__ void __launch_bounds__(HALO_THREADS, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const HaloParams p) {
  static_assert(BN == 32 || BN == 64, "conv_halo_kernel: 32 or 64 columns");
  constexpr int KT = HALO_TAPS * CB;
  constexpr int SLOT = halo_slot_bytes(BN);
  constexpr int PITCH = BN + 4;                 // epilogue tile, floats; +4 keeps float4 alignment, skews banks
  constexpr int ORIGIN = IMG ? 0 : -1;          // box coordinate of image pixel (0, 0) is -ORIGIN
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* halo = smem;                                                                 // [CB][halo_bytes]
  uint8_t* bslot = smem + CB * p.halo_bytes;
  uint64_t* bar = reinterpret_cast<uint64_t*>(bslot + KT * SLOT);               // [0] halo, [1 + kt] slot of k-tile kt
  float* cstat = reinterpret_cast<float*>(bar + halo_barriers(KT));              // [2 row halves][2 * BN]
  uint8_t* zline = reinterpret_cast<uint8_t*>(cstat + 4 * BN);                   // image mode: HALO_ZERO_BYTES of 0

  griddep_launch_dependents();  // PDL: the next kernel may start its prologue now
  const int warp = threadIdx.x >> 5;
  const int m0 = blockIdx.y * HALO_BM;
  const int n0 = blockIdx.x * BN;
  const int hw = p.Ho * p.Wo;
  const int hp = p.bh, wp = p.bw;               // box of one image

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
      for (int cb = 0; cb < CB; ++cb)
        tma_load_4d(halo + cb * p.halo_bytes, &tmX, &bar[0], 64 * cb, ORIGIN, ORIGIN, m0 / hw);
      // A slot is SROWS rows of RB bytes; each member loads `rows` of them.  A slice starts on a whole swizzle atom
      // (8 rows: 1024 B at 128 B rows, 512 B at 64 B rows), so a 32-row forward slot takes at most 4 slices and the
      // members of a cluster of 8 past the fourth load nothing.
      constexpr int SROWS = DGRAD ? 64 : BN;
      constexpr int RB = SLOT / SROWS;
      const int rows = max(SROWS / p.mc, 8);
      const int rank = p.mc > 1 ? static_cast<int>(cluster_ctarank()) : 0;
      const uint16_t mask = static_cast<uint16_t>((1u << p.mc) - 1);
      // every member's slot barrier expects the whole k-tile; a CTA whose rows all lie past M still issues its slice
#pragma unroll 1
      for (int kt = 0; kt < KT; ++kt) {
        const int tap = kt / CB, cb = kt - tap * CB;
        mbar_expect_tx(&bar[1 + kt], SLOT);
        if (rank * rows >= SROWS) continue;
        uint8_t* dst = bslot + kt * SLOT + rank * rows * RB;
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
    const int y0 = STRIDE * oi - 1 - ORIGIN, x0 = STRIDE * oj - 1 - ORIGIN;   // box row / column of tap (0, 0)
    const int hrow0 = (img * hp + y0) * wp + x0;                              // box pixel of tap (0, 0)
    const uint32_t halo_a = smem_u32(halo);
    const int half = lane >> 4;
    // 128B swizzle of each box (1024-aligned): 16-byte chunk c of box pixel (= box row) r sits at chunk
    // c ^ (r & 7); eight consecutive output columns hit eight different chunks (conflict-free at stride 1)
    auto load_a = [&](uint32_t (&a)[4][4], int kt) {
      const int tap = kt / CB, cb = kt - tap * CB;
      const int r = tap / 3, s = tap - 3 * r;
      const int hrow = hrow0 + r * wp + s;
      uint32_t row_addr = halo_a + static_cast<uint32_t>(cb * p.halo_bytes + hrow * 128);
      if constexpr (IMG) {
        const int y = y0 + r, x = x0 + s;
        if (y < 0 || y >= hp || x < 0 || x >= wp) row_addr = smem_u32(zline);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) ldmatrix_x4(a[kk], row_addr + ((((2 * kk + half) ^ hrow) & 7) << 4));
    };

    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    uint32_t a[2][4][4];
    if constexpr (IMG) {
      if (threadIdx.x < 128 + HALO_ZERO_BYTES / 16) reinterpret_cast<uint4*>(zline)[threadIdx.x - 128] = make_uint4(0, 0, 0, 0);
      named_bar_sync(1, HALO_CONSUMERS);
    }
    mbar_wait(&bar[0], 0);
    if (threadIdx.x == 128) TRACE_POINT();  // halo: activations landed
    load_a(a[0], 0);
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
      mbar_wait(&bar[1 + kt], 0);
      if (threadIdx.x == 128 && (kt == 0 || kt == KT - 1)) TRACE_POINT();  // halo: weight k-tile 0 / last landed
      const uint32_t sb = smem_u32(bslot + kt * SLOT);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        // K-major B: K advance = 32 B inside the swizzle row; MN-major B: 16 k rows of 2 BN bytes (128B swizzle at
        // 64 columns, 64B swizzle at 32)
        uint64_t bd;
        if constexpr (!DGRAD)
          bd = gmma_desc_sw128(sb + kk * 32, 16, 1024);
        else if constexpr (BN == 64)
          bd = gmma_desc_sw128(sb + kk * 2048, 8192, 1024);
        else
          bd = gmma_desc_sw64(sb + kk * 1024, 4096, 512);
        if constexpr (BN == 64)
          wgmma_bf16_n64_rs<DGRAD ? 1 : 0>(acc, a[kt & 1][kk], bd, 1u);
        else
          wgmma_bf16_n32_rs<DGRAD ? 1 : 0>(acc, a[kt & 1][kk], bd, 1u);
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
    wg_store_acc<BN>(acc, part, PITCH, 0);
    named_bar_sync(1, HALO_CONSUMERS);
    const int q = ew & 1;                      // row half
    const int c = (ew >> 1) * 32;              // the two warps of a half take one 32-column chunk each (at BN 32,
                                               // warps 2 and 3 have none)
    const int lrow = q * 32 + lane;
    const int row = m0 + lrow;
    const int col0 = n0 + c;
    float* sstat = cstat + q * 2 * BN;
    const bool want_stats = p.col_stats != nullptr;
    if (c >= BN) {                             // warp-uniform
    } else if (col0 >= p.N) {                  // warp-uniform
      if (want_stats) { sstat[c + lane] = 0.f; sstat[BN + c + lane] = 0.f; }
    } else {
      uint32_t r[32];
      acc_ld_row32(part + lrow * PITCH + c, r);
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
      // rows past M hold exact zeros (the halo of images past N is zero-filled): they add nothing to the sums
      if (want_stats) stage_col_stats(sstat, BN, c, v);
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
      for (int i = threadIdx.x - 128; i < 2 * BN; i += HALO_CONSUMERS) {
        const int col = i < BN ? i : i - BN;
        if (n0 + col < p.N)
          atomicAdd(p.col_stats + (i < BN ? 0 : p.N) + n0 + col,
                    cstat[i] + cstat[2 * BN + i]);
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

// Shape checks, tensor maps and parameters of one launch (halo mode: img false, bn 64).  src [N, H, W, C] NHWC bf16
// (x forward, dy dgrad); w [Cout, 9 * Cin] channels_last; out [N Ho Wo, Nout] bf16 with Nout = Cout forward, Cin
// dgrad.  mc: cluster size along M (1, 2, 4, 8; must divide the number of 64-row tiles).  Returns 0, 1 when there is
// nothing to compute, a CUDA / driver error code, or -2 when the shape is not one the kernel takes.
static int conv_tiled_setup(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout, int stride,
                            int dgrad, int mc, int bn, bool img, float* col_stats, CUtensorMap* tx, CUtensorMap* tw,
                            HaloParams* p, dim3* grid, int* smem);

}  // namespace b200

extern "C" int b200_encode_map2_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     int box_cols, int box_rows);
extern "C" int b200_encode_map2_sw64_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                          int box_cols, int box_rows);
extern "C" int b200_encode_map4_box_bf16(void* map, const void* base, const long long* dims,
                                         const long long* stride_bytes, const int* box);

namespace b200 {

static int conv_tiled_setup(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout, int stride,
                            int dgrad, int mc, int bn, bool img, float* col_stats, CUtensorMap* tx, CUtensorMap* tw,
                            HaloParams* p, dim3* grid, int* smem) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;      // 3x3, pad 1
  const long long M = static_cast<long long>(N) * Ho * Wo;
  if (M <= 0 || Nout <= 0) return 1;                                  // nothing to compute
  const int hw = Ho * Wo;
  const long long m_tiles = (M + HALO_BM - 1) / HALO_BM;
  const int bh = img ? H : stride * (Ho - 1) + 3, bw = img ? W : stride * (Wo - 1) + 3;
  if (H <= 0 || W <= 0 || HALO_BM % hw != 0 || bh > 256 || bw > 256 || M > (1ll << 30) || Nout % 8 != 0 ||
      ((dgrad || img) && Nout % bn != 0) || (mc != 1 && mc != 2 && mc != 4 && mc != 8) || m_tiles % mc != 0 ||
      (reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(w) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return -2;
  const int imgs = HALO_BM / hw;
  const int cb = C / 64;
  const int box_bytes = (imgs * bh * bw * 128 + 1023) / 1024 * 1024;
  *smem = cb * box_bytes + halo_fixed_bytes(HALO_TAPS * cb, bn, img);
  if (*smem > HALO_MAX_SMEM) return -2;
  const long long dims[4] = {C, W, H, N};
  const long long strides[3] = {static_cast<long long>(C) * 2, static_cast<long long>(W) * C * 2,
                                static_cast<long long>(H) * W * C * 2};
  const int box[4] = {64, bw, bh, imgs};
  int rc = b200_encode_map4_box_bf16(tx, src, dims, strides, box);
  if (rc) return rc;
  // weight slices of the kernel's `rows` (forward: a 64-column box of Cout rows of 9 C columns; dgrad: a bn-column box
  // of C = Cout rows of 9 Cin, MN-major in shared memory, whose 64 B rows at bn 32 take the 64B swizzle)
  const long long wrows = dgrad ? C : Nout, wcols = dgrad ? 9ll * Nout : 9ll * C;
  const int srows = dgrad ? 64 : bn;
  const int rows = srows / mc > 8 ? srows / mc : 8;
  rc = dgrad && bn == 32 ? b200_encode_map2_sw64_bf16(tw, w, wrows, wcols, wcols, bn, rows)
                         : b200_encode_map2_bf16(tw, w, wrows, wcols, wcols, dgrad ? bn : 64, rows);
  if (rc) return rc;
  p->M = static_cast<int>(M); p->N = Nout; p->Ho = Ho; p->Wo = Wo; p->D = reinterpret_cast<__nv_bfloat16*>(out);
  p->col_stats = col_stats; p->ncol = Nout; p->mc = mc; p->halo_bytes = box_bytes; p->bh = bh; p->bw = bw;
  *grid = dim3((Nout + bn - 1) / bn, static_cast<unsigned>(m_tiles), 1);
  return 0;
}

}  // namespace b200

// Instantiated (stride, C): (1, 64) and (1, 128) forward and dgrad, (2, 64) forward.  col_stats (forward only):
// optional [2 Nout] fp32.
extern "C" int b200_conv_halo(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout,
                              int stride, int dgrad, int mc, float* col_stats, cudaStream_t stream) {
  using namespace b200;
  const bool s1c64 = stride == 1 && C == 64, s1c128 = stride == 1 && C == 128, s2c64 = stride == 2 && C == 64 && !dgrad;
  if (!s1c64 && !s1c128 && !s2c64) return -2;
  CUtensorMap tx, tw;
  HaloParams p;
  dim3 grid;
  int smem = 0;
  const int rc = conv_tiled_setup(src, w, out, N, H, W, C, Nout, stride, dgrad, mc, HALO_BN, false, col_stats, &tx, &tw,
                                  &p, &grid, &smem);
  if (rc) return rc == 1 ? 0 : rc;
  if (s2c64) return launch_halo<conv_halo_kernel<false, 1, 2>>(tx, tw, p, grid, smem, stream);
  if (s1c64)
    return dgrad ? launch_halo<conv_halo_kernel<true, 1, 1>>(tx, tw, p, grid, smem, stream)
                 : launch_halo<conv_halo_kernel<false, 1, 1>>(tx, tw, p, grid, smem, stream);
  return dgrad ? launch_halo<conv_halo_kernel<true, 2, 1>>(tx, tw, p, grid, smem, stream)
               : launch_halo<conv_halo_kernel<false, 2, 1>>(tx, tw, p, grid, smem, stream);
}

// Image mode (layer3 of ResNet-18 on 32x32 inputs: 2x2 output maps).  Instantiated (stride, C, bn): (1, 256, 32)
// forward and dgrad, (2, 128, 32) and (2, 128, 64) forward.  Arguments and return as b200_conv_halo.
extern "C" int b200_conv_smallmap(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout,
                                  int stride, int dgrad, int mc, int bn, float* col_stats, cudaStream_t stream) {
  using namespace b200;
  const bool s1c256 = stride == 1 && C == 256 && bn == 32;
  const bool s2c128 = stride == 2 && C == 128 && !dgrad && (bn == 32 || bn == 64);
  if (!s1c256 && !s2c128) return -2;
  CUtensorMap tx, tw;
  HaloParams p;
  dim3 grid;
  int smem = 0;
  const int rc = conv_tiled_setup(src, w, out, N, H, W, C, Nout, stride, dgrad, mc, bn, true, col_stats, &tx, &tw, &p,
                                  &grid, &smem);
  if (rc) return rc == 1 ? 0 : rc;
  if (s2c128)
    return bn == 32 ? launch_halo<conv_halo_kernel<false, 2, 2, 32, true>>(tx, tw, p, grid, smem, stream)
                    : launch_halo<conv_halo_kernel<false, 2, 2, 64, true>>(tx, tw, p, grid, smem, stream);
  return dgrad ? launch_halo<conv_halo_kernel<true, 4, 1, 32, true>>(tx, tw, p, grid, smem, stream)
               : launch_halo<conv_halo_kernel<false, 4, 1, 32, true>>(tx, tw, p, grid, smem, stream);
}

B200_TRACE_REGISTER(conv_halo)
