// bf16 GEMM on the Hopper tensor cores: TMA -> 128B-swizzled smem ring -> wgmma (two consumer warpgroups,
// accumulator in registers) -> fp32 tile in shared memory -> row-per-lane epilogue with fused bias / activation / cast.
//
//     D[M,N] = act( alpha * A[M,K] * B[N,K]^T + bias[N] )          (A, B bf16; accumulate fp32)
//
// Each operand may be K-major (row-major [rows, K]) or MN-major (row-major [K, rows]), so the
// three training GEMMs need no transposes:
//     fwd    Y  = X  W^T      A = X   (K-major)   B = W  (K-major)
//     dgrad  dX = dY W        A = dY  (K-major)   B = W  (MN-major)
//     wgrad  dW = dY^T X      A = dY  (MN-major)  B = X  (MN-major)
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected lane of warp 0), warpgroups 1 and 2 = consumers:
// each issues m64 x BN x 16 wgmma for its 64 rows of the 128-row tile, parks the accumulator in shared memory and
// runs the epilogue over it.  BN is 64 or 128: a 64 x 256 fp32 accumulator would take 128 registers per thread.
//
// Split-K, two flavours:
//   * atomic   (fp32 output, gradient accumulation): gridDim.z slices red.global.add into D;
//   * cluster  (any output): the z-slices of one output tile form a thread-block CLUSTER; each CTA
//     parks its fp32 partial tile in its own shared memory, and after a cluster barrier CTA r
//     reduces rows [r*128/S, (r+1)*128/S) of all S partials through distributed shared memory
//     (ld.shared::cluster), applies the epilogue and stores -- no workspace, no second kernel.
//     This is what makes the deep layers of a ResNet (M = 128, K = 4608) use more than 8 SMs.
//
// Flag-gated variant ("bcast_gemm", K3 in SURVEY.md 2.6): the producer acquires per-arena-tile
// arrival flags (published by the FedAvg kernel with st.release) before issuing the TMA loads of
// a weight tile, so the first GEMM of a round consumes the new global weights tile by tile while
// the rest of the model is still landing over NVLink.
#define B200_TU_TAG 1
#include "ptx.cuh"
#include "epilogue.cuh"
#include "launch.h"
#include "pdl.cuh"
#include "sgd.cuh"

namespace b200 {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int WG_K = 16;               // K per wgmma for 16-bit operands
constexpr int GEMM_THREADS = 384;
constexpr int CONSUMER_WARPS = 8;      // warpgroups 1 and 2
constexpr int CONSUMER_THREADS = 32 * CONSUMER_WARPS;
constexpr int MAX_STAGES = 8;
constexpr int S2_MAX_TAPS = 4;         // taps of one parity class of a stride-2 dgrad (3x3: at most 2 x 2)

struct GemmParams {
  int M, N, K;
  void* D;
  long long ldd;          // leading dimension of D in elements
  const float* bias;      // [N] or nullptr
  int out_fp32;           // 1: D is fp32, 0: D is bf16
  int act;                // 0 none, 1 relu, 2 gelu(tanh)
  float* col_stats;       // optional [2N]: += column sums / sums of squares of the (bf16-rounded) output (BatchNorm)
  int a_mn, b_mn;         // operand majors
  int k_tiles_per_split;  // split-K: k tiles handled by one z-slice
  int atomic_out;         // 1: red.add fp32 into D
  int cluster_k;          // > 1: z-slices form a cluster of this size and reduce through DSMEM
  int stages;             // pipeline depth (1..MAX_STAGES)
  const uint32_t* tile_flags;  // optional arrival flags, one per arena tile (bcast_gemm)
  uint32_t flag_epoch;         // value a flag must reach before the data under it may be loaded
  long long flag_elem_off;     // arena element offset of B[0,0]
  int flag_tile_elems;         // arena elements covered by one flag
  long long flag_bias_off;     // arena element offset of bias[0], or -1
  long long ldb;               // row pitch of B (elements)
  float alpha;
  // strided-batched mode (attention): blockIdx.z = outer * batch_inner + inner; operands come from
  // 4-D tensor maps (col, row, inner, outer); D is offset by outer * d_outer + inner * d_inner elements
  int batched, batch_inner;
  int batch_count;         // persistent batched mode: number of z slices
  long long d_outer, d_inner;
  // implicit-GEMM convolution (CONV template modes; appended last so existing field offsets do not move)
  int conv_ho, conv_wo;    // output image size
  int conv_stride, conv_pad;
  int conv_kw;             // filter width (tap = r * kw + s)
  int conv_cin;            // channels of the im2col-gathered tensor (multiple of 64): Cin forward, Cout for dgrad
  int conv_taps;           // dgrad: KH * KW
  int conv_ncol;           // dgrad: Cin of the convolution (column pitch of one tap inside a weight row)
  const uint32_t* flag_epoch_ptr;   // bcast_gemm inside a captured graph: the required flag value lives in device memory
  // optimizer epilogue (the SGD instantiation of the fixed-depth kernel, single K pass): SGD on theta instead of
  // red.add into D; the pointers address the element D[0, 0] would and are indexed like D
  const float* sgd_hyper = nullptr;
  float* sgd_theta = nullptr;
  __nv_bfloat16* sgd_wb = nullptr;
  float* sgd_mom = nullptr;
  int sgd_nesterov = 0;
  // stride-2 implicit dgrad (CONV == 4): dx pixel (2i + a, 2j + b) of parity class c = 2a + b sums s2_ntaps[c] taps,
  // each packed as filter tap | dy row offset << 16 | dy column offset << 24: dy pixel (i + dp, j + dq)
  int conv_h = 0, conv_w = 0;  // dx image size
  int s2_ntaps[4] = {0, 0, 0, 0};
  int s2_tap[4][S2_MAX_TAPS] = {};
  // eval-mode BatchNorm epilogue (the AFFINE instantiations): D = act(acc * bn_scale[c] + bn_shift[c] + residual[r, c]),
  // bf16 out; act is 0 or 1 (ReLU)
  const float* bn_scale = nullptr;
  const float* bn_shift = nullptr;
  const __nv_bfloat16* residual = nullptr;   // optional, [M, ldr]
  long long ldr = 0;
  // FedProx anchor of the optimizer epilogue, indexed like sgd_theta; nullptr: no proximal term (sgd_hyper has 4 floats)
  const float* sgd_anchor = nullptr;
  // SCAFFOLD correction c - c_i of the optimizer epilogue, indexed like sgd_theta; nullptr: no correction term
  const float* sgd_corr = nullptr;
  // AdamW second moment of the optimizer epilogue, indexed like sgd_theta (sgd_mom is then the first moment and
  // sgd_hyper the step's AdamW row); nullptr: SGD
  float* sgd_v = nullptr;
  // rank-R LoRA term of the LORA instantiation (see lora_chunk), added to the fp32 accumulator before alpha / bias / act
  const __nv_bfloat16* lora_u = nullptr;     // [M, lora_ldu]: the down projection, ranks [0, lora_R)
  const __nv_bfloat16* lora_f = nullptr;     // the up factor, element (row, j) at row * lora_fs_n + j * lora_fs_j
  long long lora_ldu = 0, lora_fs_n = 0, lora_fs_j = 0;
  int lora_R = 0;                            // ranks of U (multiple of 8, <= B200_LORA_MAX_R)
  int lora_rs = 0;                           // ranks per slice (multiple of 8)
  int lora_ds = 0;                           // columns per slice (multiple of 32)
  int lora_slot[3] = {-1, -1, -1};           // slice -> its rank block t (U columns [t rs, t rs + rs)), -1: no term
  float lora_s = 0.f;
};

// Wait until every arrival flag covering arena elements [e0, e1] has reached `need` (published by the FedAvg kernel with
// st.release.sys).  Bounded: a collective that died must not hang the consumer (it then reads what is there).
__device__ __forceinline__ void wait_arrival_flags(const uint32_t* flags, long long e0, long long e1, int granule,
                                                   uint32_t need) {
  for (long long t = e0 / granule; t <= e1 / granule; ++t) {
    unsigned long long spins = 0;
    while (static_cast<int32_t>(ld_acquire_sys(flags + t) - need) < 0) {
      if (++spins > (1ull << 26)) break;
    }
  }
}

template <int BN>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int PART_PITCH = BN + 4;                  // floats; +4 keeps float4 alignment, skews banks
  static constexpr int PART_BYTES = BM * PART_PITCH * 4;     // fp32 partial tile for the cluster reduce
};

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    float t = tanhf(k0 * (v + k1 * v * v * v));
    return 0.5f * v * (1.f + t);
  }
  return v;
}

__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_smem_addr), "r"(cta_rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(remote)
               : "memory");
  return v;
}

// BatchNorm batch statistics fused into the producing GEMM: every lane of the warp must call this.  Rows
// beyond M hold exact zeros (TMA zero-fills out-of-range operand rows; no bias / activation in this mode).
__device__ __forceinline__ void accumulate_col_stats(const GemmParams& p, int col0, const float (&v)[32]) {
  float s[32], q[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float r = __bfloat162float(__float2bfloat16_rn(v[j]));   // what the consumer will read back
    s[j] = r;
    q[j] = r * r;
  }
  const float cs = warp_colsum32(s), cq = warp_colsum32(q);
  const int col = col0 + static_cast<int>(lane_id());
  if (col < p.N) {
    atomicAdd(p.col_stats + col, cs);
    atomicAdd(p.col_stats + p.N + col, cq);
  }
}

// alpha / bias / activation of one row chunk.  The (activation, bias) combination is resolved ONCE per chunk
// with warp-uniform branches into fully unrolled straight-line code; the per-element runtime switch this
// replaces expands to hundreds of instructions per 32-column chunk.
template <int NV, int ACT, bool BIAS>
__device__ __forceinline__ void transform_chunk_t(const GemmParams& p, int col0, float (&v)[NV]) {
  float b[NV];
  if (BIAS) {
    if (col0 + NV <= p.N && ((reinterpret_cast<uintptr_t>(p.bias + col0) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < NV; j += 4) {      // every lane reads the same addresses: one broadcast request each
        const float4 t = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + j));
        b[j] = t.x; b[j + 1] = t.y; b[j + 2] = t.z; b[j + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < NV; ++j) b[j] = (col0 + j) < p.N ? __ldg(p.bias + col0 + j) : 0.f;
    }
  }
  const float alpha = p.alpha;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    float x = v[j] * alpha;
    if (BIAS) x += b[j];
    if (ACT == 1) x = fmaxf(x, 0.f);
    if (ACT == 2) {
      const float k0 = 0.7978845608028654f, k1 = 0.044715f;
      x = 0.5f * x * (1.f + tanhf(k0 * (x + k1 * x * x * x)));
    }
    v[j] = x;
  }
}
template <int NV>
__device__ __forceinline__ void transform_chunk(const GemmParams& p, int col0, float (&v)[NV]) {
  if (p.bias == nullptr) {
    if (p.act == 0) transform_chunk_t<NV, 0, false>(p, col0, v);
    else if (p.act == 1) transform_chunk_t<NV, 1, false>(p, col0, v);
    else transform_chunk_t<NV, 2, false>(p, col0, v);
  } else {
    if (p.act == 0) transform_chunk_t<NV, 0, true>(p, col0, v);
    else if (p.act == 1) transform_chunk_t<NV, 1, true>(p, col0, v);
    else transform_chunk_t<NV, 2, true>(p, col0, v);
  }
}

// Eval-mode BatchNorm of one row chunk (columns [col0, col0 + NV) of `row` < M): bn_apply's eval arithmetic,
// fmaf(z, scale, shift) + residual, then ReLU, on the fp32 accumulator instead of a bf16-rounded z.  The host
// guarantees N % 8 == 0, 16-byte aligned scale / shift / residual rows and ldr % 8 == 0, so every group of 8 columns
// is either wholly inside N or wholly past it and loads as vectors.
template <int NV>
__device__ __forceinline__ void affine_chunk(const GemmParams& p, int row, int col0, float (&v)[NV]) {
  static_assert(NV % 8 == 0, "affine epilogue works on groups of 8 columns");
  const bool relu = p.act == 1;
  const __nv_bfloat16* res = p.residual != nullptr ? p.residual + static_cast<size_t>(row) * p.ldr + col0 : nullptr;
#pragma unroll
  for (int j = 0; j < NV; j += 8) {
    if (col0 + j >= p.N) break;
    // every lane of a warp reads the same scale / shift addresses: one broadcast request each
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(p.bn_scale + col0 + j));
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(p.bn_scale + col0 + j + 4));
    const float4 h0 = __ldg(reinterpret_cast<const float4*>(p.bn_shift + col0 + j));
    const float4 h1 = __ldg(reinterpret_cast<const float4*>(p.bn_shift + col0 + j + 4));
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    float r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (res != nullptr) {
      const uint4 rv = *reinterpret_cast<const uint4*>(res + j);
      const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(rw[i]);
        r[2 * i] = f.x;
        r[2 * i + 1] = f.y;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = fmaf(v[j + i], sc[i], sh[i]) + r[i];
      v[j + i] = relu ? fmaxf(x, 0.f) : x;
    }
  }
}

template <int NV, bool AFFINE = false>
__device__ __forceinline__ void store_row_chunk(const GemmParams& p, int row, int col0, float (&v)[NV], bool vec_ok,
                                                size_t d_off = 0) {
  if constexpr (AFFINE)
    affine_chunk<NV>(p, row, col0, v);
  else
    transform_chunk<NV>(p, col0, v);
  const bool full = (col0 + NV <= p.N);
  if (p.out_fp32) {
    float* d = reinterpret_cast<float*>(p.D) + d_off + static_cast<size_t>(row) * p.ldd + col0;
    if (p.atomic_out) {
      if (full && vec_ok) {
#pragma unroll
        for (int j = 0; j < NV; j += 4)
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + j), "f"(v[j]), "f"(v[j + 1]),
                       "f"(v[j + 2]), "f"(v[j + 3])
                       : "memory");
      } else {
        _Pragma("unroll") for (int j = 0; j < NV; ++j) if (col0 + j < p.N) atomicAdd(d + j, v[j]);
      }
    } else if (full && vec_ok) {
#pragma unroll
      for (int j = 0; j < NV; j += 4) *reinterpret_cast<float4*>(d + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
      _Pragma("unroll") for (int j = 0; j < NV; ++j) if (col0 + j < p.N) d[j] = v[j];
    }
  } else {
    __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(p.D) + d_off + static_cast<size_t>(row) * p.ldd + col0;
    if (full && vec_ok) {
#pragma unroll
      for (int j = 0; j < NV; j += 8) {
        uint4 o;
        o.x = pack_bf16x2(v[j], v[j + 1]);
        o.y = pack_bf16x2(v[j + 2], v[j + 3]);
        o.z = pack_bf16x2(v[j + 4], v[j + 5]);
        o.w = pack_bf16x2(v[j + 6], v[j + 7]);
        *reinterpret_cast<uint4*>(d + j) = o;
      }
    } else {
      _Pragma("unroll") for (int j = 0; j < NV; ++j) if (col0 + j < p.N) d[j] = __float2bfloat16_rn(v[j]);
    }
  }
}

// Optimizer epilogue of one 32-column row chunk (columns [col0, col0 + 32) of `row`, `e` = its element offset from D[0,0]).
// The tile holds the complete gradient of these weights (single K pass), so the SGD step runs here and the gradient
// buffer is never touched.  0 + v is the value a red.add into the zeroed gradient would have left (-0 becomes +0), and
// sgd_update is the arena optimizer's arithmetic: the result matches accumulate-then-fused_sgd bit for bit.
// PROX: FedProx step, the anchor (sgd_anchor) is read beside theta.  SCAF: SCAFFOLD step, the correction (sgd_corr)
// is read beside theta instead.
template <bool PROX, bool SCAF = false>
__device__ __forceinline__ void sgd_epilogue_chunk(const GemmParams& p, size_t e, int col0, const float (&v)[32],
                                                   bool vec);

// The AdamW form (adamw_update of sgd.cuh, the arithmetic of the arena kernels' AdamW instantiations): m is sgd_mom,
// v is sgd_v, the coefficients are the step row at sgd_hyper.
__device__ __forceinline__ void adamw_epilogue_chunk(const GemmParams& p, size_t e, int col0, const float (&v)[32],
                                                     bool vec) {
  const AdamHyper h = load_adam_hyper(p.sgd_hyper);
  float* w = p.sgd_theta + e;
  float* m = p.sgd_mom + e;
  float* sq = p.sgd_v + e;
  __nv_bfloat16* wb = p.sgd_wb != nullptr ? p.sgd_wb + e : nullptr;
  if (vec && col0 + 32 <= p.N) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      float4 mv = *reinterpret_cast<const float4*>(m + j), vv = *reinterpret_cast<const float4*>(sq + j);
      const float4 gv = make_float4(__fadd_rn(0.f, v[j]), __fadd_rn(0.f, v[j + 1]), __fadd_rn(0.f, v[j + 2]),
                                    __fadd_rn(0.f, v[j + 3]));
      const float4 wv = adamw_update4(h, *reinterpret_cast<const float4*>(w + j), gv, mv, vv);
      *reinterpret_cast<float4*>(w + j) = wv;
      *reinterpret_cast<float4*>(m + j) = mv;
      *reinterpret_cast<float4*>(sq + j) = vv;
      if (wb != nullptr) *reinterpret_cast<uint2*>(wb + j) = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (col0 + j < p.N) {
        const float wv = adamw_update(h, w[j], __fadd_rn(0.f, v[j]), m[j], sq[j]);
        w[j] = wv;
        if (wb != nullptr) wb[j] = __float2bfloat16_rn(wv);
      }
    }
  }
}

template <bool PROX, bool SCAF>
__device__ __forceinline__ void sgd_epilogue_chunk(const GemmParams& p, size_t e, int col0, const float (&v)[32],
                                                   bool vec) {
  const float* a = PROX ? p.sgd_anchor + e : SCAF ? p.sgd_corr + e : nullptr;
  const SgdHyper h = PROX ? load_sgd_hyper_prox(p.sgd_hyper) : load_sgd_hyper(p.sgd_hyper);
  float* w = p.sgd_theta + e;
  float* m = p.sgd_mom != nullptr ? p.sgd_mom + e : nullptr;
  __nv_bfloat16* wb = p.sgd_wb != nullptr ? p.sgd_wb + e : nullptr;
  const bool nest = p.sgd_nesterov != 0;
  if (vec && col0 + 32 <= p.N) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      float4 mv = m != nullptr ? *reinterpret_cast<const float4*>(m + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 gv = make_float4(__fadd_rn(0.f, v[j]), __fadd_rn(0.f, v[j + 1]), __fadd_rn(0.f, v[j + 2]),
                                    __fadd_rn(0.f, v[j + 3]));
      const float4 w0 = *reinterpret_cast<const float4*>(w + j);
      const float4 wv = PROX ? sgd_update4_prox(h, w0, gv, *reinterpret_cast<const float4*>(a + j), mv, m != nullptr,
                                                nest)
                        : SCAF ? sgd_update4_scaf(h, w0, gv, *reinterpret_cast<const float4*>(a + j), mv, m != nullptr,
                                                  nest)
                               : sgd_update4(h, w0, gv, mv, m != nullptr, nest);
      *reinterpret_cast<float4*>(w + j) = wv;
      if (m != nullptr) *reinterpret_cast<float4*>(m + j) = mv;
      if (wb != nullptr) *reinterpret_cast<uint2*>(wb + j) = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (col0 + j < p.N) {
        float mv = m != nullptr ? m[j] : 0.f;
        const float gj = __fadd_rn(0.f, v[j]);
        const float wv = PROX ? sgd_update_prox(h, w[j], gj, a[j], mv, m != nullptr, nest)
                         : SCAF ? sgd_update_scaf(h, w[j], gj, a[j], mv, m != nullptr, nest)
                                : sgd_update(h, w[j], gj, mv, m != nullptr, nest);
        w[j] = wv;
        if (m != nullptr) m[j] = mv;
        if (wb != nullptr) wb[j] = __float2bfloat16_rn(wv);
      }
    }
  }
}

// Consumer main loop, shared by every kernel below: warpgroup g (0 or 1) accumulates rows [64 g, 64 g + 64) of the
// 128 x BN tile in registers over `num_kt` k-tiles of the ring.  A stage is handed back to the producer (one arrival
// per consumer warp) as soon as the wgmma that read it have retired -- one k-tile of MMAs stays in flight.
template <int BN>
__device__ __forceinline__ void consume_ktiles(float (&acc)[BN / 2], uint8_t* smem, int stages, uint64_t* full_bar,
                                               uint64_t* empty_bar, int& s, uint32_t& ph, int num_kt, int a_mn,
                                               int b_mn, int g) {
  using L = SmemLayout<BN>;
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
  int prev = -1;
  for (int i = 0; i < num_kt; ++i) {
    mbar_wait(&full_bar[s], ph);
    // K-major A: 64 rows x 128 B = 8192 B per warpgroup; MN-major A: the warpgroup's 64-wide atom is 8192 B
    const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES) + g * 8192;
    const uint32_t sb = smem_u32(smem + s * L::STAGE_BYTES + L::A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k) {
      // K-major: 8-row groups are 1024 B apart (SBO), K advance = 32 B inside the swizzle row.
      // MN-major: 64-wide MN atoms are 8192 B apart (LBO), 8-row K groups 1024 B apart (SBO),
      //           K advance of 16 rows = 2048 B.
      const uint64_t ad = a_mn ? gmma_desc_sw128(sa + k * 2048, 8192, 1024) : gmma_desc_sw128(sa + k * 32, 16, 1024);
      const uint64_t bd = b_mn ? gmma_desc_sw128(sb + k * 2048, 8192, 1024) : gmma_desc_sw128(sb + k * 32, 16, 1024);
      wgmma_bf16<BN>(acc, ad, bd, 1u, a_mn, b_mn);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == stages) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_operands(acc);
  if (prev >= 0 && lane_id() == 0) mbar_arrive(&empty_bar[prev]);
}

// ---- stride-2 implicit dgrad (CONV == 4): sub-pixel decomposition ----
// The dx pixels of parity class c = 2a + b, (2i + a, 2j + b), form a stride-1 correlation of dy with the taps that land
// on them.  Every class enumerates the same N x Ho x Wo grid of (n, i, j) as GEMM rows; blockIdx.y = c * m_tiles + m
// tile.  A class without taps runs no k tile and stores zeros; rows outside dx (odd H or W) are not stored.
__device__ __forceinline__ int s2_class(const GemmParams& p, int& m0) {
  const int tiles_m = (p.M + BM - 1) / BM;
  const int cls = static_cast<int>(blockIdx.y) / tiles_m;
  m0 = (static_cast<int>(blockIdx.y) - cls * tiles_m) * BM;
  return cls;
}
// selects instead of a dynamic index: a runtime-indexed kernel parameter array would be copied to local memory
__device__ __forceinline__ int s2_ntaps(const GemmParams& p, int cls) {
  int n = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) n = c == cls ? p.s2_ntaps[c] : n;
  return n;
}
__device__ __forceinline__ int s2_tap(const GemmParams& p, int cls, int slot) {
  int w = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int t = 0; t < S2_MAX_TAPS; ++t) w = (c == cls && t == slot) ? p.s2_tap[c][t] : w;
  return w;
}
// dx row of GEMM row m of class cls, or -1 (m >= M, or the pixel lies past the last row / column of an odd-sized dx)
__device__ __forceinline__ int s2_dx_row(const GemmParams& p, int cls, int m) {
  if (m >= p.M) return -1;
  const int hw = p.conv_ho * p.conv_wo;
  const int n = m / hw, r = m - n * hw;
  const int i = r / p.conv_wo, j = r - i * p.conv_wo;
  const int h = 2 * i + (cls >> 1), w = 2 * j + (cls & 1);
  return (h < p.conv_h && w < p.conv_w) ? (n * p.conv_h + h) * p.conv_w + w : -1;
}
// TMA loads of k tile kt of class cls: A = 128 dy pixels (i + dp, j + dq) x 64 output channels (zero outside dy),
// B = the [64 cout] x [BN cin] slab of the tap inside the channels_last weight matrix, MN-major
template <int BN>
__device__ __forceinline__ void s2_load_ktile(const CUtensorMap* tmA, const CUtensorMap* tmB, const GemmParams& p,
                                              uint8_t* sa, uint8_t* sb, uint64_t* bar, int cls, int kt, int m0, int n0) {
  const int cblocks = p.conv_cin >> 6;
  const int slot = kt / cblocks, cb = kt - slot * cblocks;
  const int tw = s2_tap(p, cls, slot);
  const int q0 = m0 % p.conv_wo, t0 = m0 / p.conv_wo;
  tma_load_im2col_4d(sa, tmA, bar, cb * 64, q0, t0 % p.conv_ho, t0 / p.conv_ho, (tw >> 24) & 0xff, (tw >> 16) & 0xff);
  const int wcol = (tw & 0xffff) * p.conv_ncol + n0;
#pragma unroll
  for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, tmB, bar, wcol + j * 64, cb * 64);
}

// ---- LoRA epilogue (the LORA instantiation of the fixed-depth kernel) ----
// Column n of slice sl = n / lora_ds with rank block t = lora_slot[sl] >= 0 receives
//     lora_s * sum_{j < rs} U[m, t rs + j] * F(t ds + n - sl ds, j)
// in fp32, j ascending, added to the accumulator (one fmaf) before alpha, bias and activation; the output is then
// rounded once.  The CTA stages its 128 U rows ([128][R + 8] bf16) and the factor rows of its BN columns ([BN][rs + 8]
// bf16, zero for columns of an untargeted slice or past N) behind the column-statistics area.
__device__ __forceinline__ int lora_slot(const GemmParams& p, int sl) {
  return sl == 0 ? p.lora_slot[0] : (sl == 1 ? p.lora_slot[1] : (sl == 2 ? p.lora_slot[2] : -1));
}

template <int BN>
__device__ __forceinline__ void lora_stage(const GemmParams& p, __nv_bfloat16* us, __nv_bfloat16* fs, int m0, int n0) {
  const int tid = static_cast<int>(threadIdx.x) - 128;
  const int R = p.lora_R, up = R + 8, rs = p.lora_rs, fp = rs + 8;
  const int vr = R / 8;      // 16-byte vectors per U row (host: R % 8 == 0, ldu % 8 == 0, 16-byte aligned U)
  for (int i = tid; i < BM * vr; i += CONSUMER_THREADS) {
    const int r = i / vr, c = (i - r * vr) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (m0 + r < p.M) v = __ldg(reinterpret_cast<const uint4*>(p.lora_u + static_cast<size_t>(m0 + r) * p.lora_ldu + c));
    *reinterpret_cast<uint4*>(us + r * up + c) = v;
  }
  for (int i = tid; i < BN * rs; i += CONSUMER_THREADS) {
    const int j = i / BN, c = i - j * BN, n = n0 + c;
    __nv_bfloat16 v = __float2bfloat16_rn(0.f);
    if (n < p.N) {
      const int sl = n / p.lora_ds, t = lora_slot(p, sl);
      if (t >= 0)
        v = p.lora_f[static_cast<long long>(t * p.lora_ds + n - sl * p.lora_ds) * p.lora_fs_n +
                     static_cast<long long>(j) * p.lora_fs_j];
    }
    fs[c * fp + j] = v;
  }
}

// the rank term of one 32-column row chunk: local row lrow, local columns [c, c + 32); lora_ds % 32 == 0, so the chunk
// lies in one slice
__device__ __forceinline__ void lora_chunk(const GemmParams& p, const __nv_bfloat16* us, const __nv_bfloat16* fs,
                                           int lrow, int c, int col0, float (&v)[32]) {
  const int t = lora_slot(p, col0 / p.lora_ds);      // warp-uniform
  if (t < 0) return;
  const int rs = p.lora_rs, fp = rs + 8;
  const __nv_bfloat16* urow = us + lrow * (p.lora_R + 8) + t * rs;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll 1
  for (int j = 0; j < rs; j += 8) {
    const uint4 uv = *reinterpret_cast<const uint4*>(urow + j);
    const float2 u0 = unpack_bf16x2(uv.x), u1 = unpack_bf16x2(uv.y), u2 = unpack_bf16x2(uv.z), u3 = unpack_bf16x2(uv.w);
    const float u[8] = {u0.x, u0.y, u1.x, u1.y, u2.x, u2.y, u3.x, u3.y};
#pragma unroll
    for (int i = 0; i < 32; ++i) {       // every lane reads the same factor row: one broadcast request
      const uint4 fv = *reinterpret_cast<const uint4*>(fs + (c + i) * fp + j);
      const float2 f0 = unpack_bf16x2(fv.x), f1 = unpack_bf16x2(fv.y), f2 = unpack_bf16x2(fv.z), f3 = unpack_bf16x2(fv.w);
      float a = acc[i];
      a = fmaf(u[0], f0.x, a); a = fmaf(u[1], f0.y, a); a = fmaf(u[2], f1.x, a); a = fmaf(u[3], f1.y, a);
      a = fmaf(u[4], f2.x, a); a = fmaf(u[5], f2.y, a); a = fmaf(u[6], f3.x, a); a = fmaf(u[7], f3.y, a);
      acc[i] = a;
    }
  }
  const float s = p.lora_s;
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = fmaf(s, acc[i], v[i]);
}

// ---- fixed-depth pipeline: the default path ----
// CONV: 0 = plain GEMM; 1 = implicit-GEMM conv forward (A = im2col(x) gathered by TMA im2col, k-tile = one filter
// tap x 64 input channels); 2 = implicit wgrad (B = im2col(x) MN-major, k-tile = 64 output pixels, every 64-wide
// N atom = one tap x 64 channels); 3 = implicit dgrad of a stride-1 convolution: dx = conv(dy, flipped w) -- A =
// im2col(dy) gathered by TMA im2col with pad' = k - 1 - pad (k-tile = one flipped tap x 64 OUTPUT channels), B = the
// [64 cout] x [BN cin] slab of that tap inside the channels_last weight matrix, loaded MN-major (no weight transpose,
// no col2im); 4 = implicit dgrad of a stride-2 convolution, one parity class of dx pixels per group of M tiles (see
// s2_class).  See csrc/im2col_tma.cu for the tensor maps.
// SGD: optimizer epilogue instantiation (weight gradients only) -- every other GEMM keeps the plain epilogue.
// PROX (with SGD): the FedProx form of that epilogue.  SCAF (with SGD): its SCAFFOLD form.  ADAM (with SGD): its
// AdamW form (adamw_epilogue_chunk).
// AFFINE: eval-mode BatchNorm epilogue instantiation (affine_chunk, forward convolutions in evaluation).
// LORA: the rank-R LoRA term in the epilogue (lora_chunk; plain GEMM, single K pass).
template <int BN, int STAGES, int CONV = 0, bool SGD = false, bool AFFINE = false, bool PROX = false, bool SCAF = false,
          bool ADAM = false, bool LORA = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_fixed_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                         const GemmParams p) {
  using L = SmemLayout<BN>;
  static_assert(STAGES * L::STAGE_BYTES >= L::PART_BYTES, "the drained ring must hold the fp32 accumulator tile");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem is only guaranteed 16B aligned: realign to the 1024B the 128B swizzle needs
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* cstat = reinterpret_cast<float*>(empty_bar + STAGES);   // [4 row quarters][2 * BN] column statistics

  griddep_launch_dependents();  // PDL: the next kernel may start its prologue now
  const int warp = threadIdx.x >> 5;
  int m0 = blockIdx.y * BM;
  const int cls = CONV == 4 ? s2_class(p, m0) : 0;
  const int n0 = blockIdx.x * BN;
  const int k_tiles_total = CONV == 4 ? s2_ntaps(p, cls) * (p.conv_cin >> 6) : (p.K + BK - 1) / BK;
  const int bz_outer = p.batched ? static_cast<int>(blockIdx.z) / p.batch_inner : 0;
  const int bz_inner = p.batched ? static_cast<int>(blockIdx.z) % p.batch_inner : 0;
  const int kt_begin = p.batched ? 0 : blockIdx.z * p.k_tiles_per_split;
  int kt_end = kt_begin + p.k_tiles_per_split;
  if (kt_end > k_tiles_total) kt_end = k_tiles_total;
  // host guarantees >= 1 for every launched z, except CONV == 4: a class without taps runs none
  const int num_kt = kt_end - kt_begin;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();  // PDL: everything above overlapped the previous kernel; its results are visible from here

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      if (p.tile_flags != nullptr) {
        // bcast_gemm: wait until the FedAvg kernel has published every arena tile under the rows
        // [n0, n0+BN) of the (K-major) weight matrix this CTA is about to TMA-load
        const int rows_here = (p.N - n0) < BN ? (p.N - n0) : BN;
        const uint32_t need = p.flag_epoch_ptr != nullptr ? *reinterpret_cast<const volatile uint32_t*>(p.flag_epoch_ptr)
                                                          : p.flag_epoch;
        wait_arrival_flags(p.tile_flags, p.flag_elem_off + static_cast<long long>(n0) * p.ldb,
                           p.flag_elem_off + static_cast<long long>(n0 + rows_here) * p.ldb - 1, p.flag_tile_elems, need);
        if (p.flag_bias_off >= 0)  // the bias slice the epilogue of this CTA will add
          wait_arrival_flags(p.tile_flags, p.flag_bias_off + n0, p.flag_bias_off + n0 + rows_here - 1,
                             p.flag_tile_elems, need);
        fence_proxy_async_all();  // order the acquires before the async-proxy (TMA) reads of global memory
      }
      TRACE_POINT();  // fixed: producer starts issuing TMA
      for (int i = 0; i < num_kt; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * L::STAGE_BYTES;
        uint8_t* sb = sa + L::A_BYTES;
        const int k0 = (kt_begin + i) * BK;
        if constexpr (CONV == 2) {
          const int live = (p.N - n0 + 63) / 64 < BN / 64 ? (p.N - n0 + 63) / 64 : BN / 64;
          mbar_expect_tx(&full_bar[s], L::A_BYTES + live * 8192);
        } else {
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
        }
        if (p.batched) {
          if (!p.a_mn) {
            tma_load_4d(sa, &tmA, &full_bar[s], k0, m0, bz_inner, bz_outer);
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j)
              tma_load_4d(sa + j * 8192, &tmA, &full_bar[s], m0 + j * 64, k0, bz_inner, bz_outer);
          }
          if (!p.b_mn) {
            tma_load_4d(sb, &tmB, &full_bar[s], k0, n0, bz_inner, bz_outer);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_4d(sb + j * 8192, &tmB, &full_bar[s], n0 + j * 64, k0, bz_inner, bz_outer);
          }
        } else if constexpr (CONV == 4) {
          s2_load_ktile<BN>(&tmA, &tmB, p, sa, sb, &full_bar[s], cls, kt_begin + i, m0, n0);
        } else {
        if constexpr (CONV == 1 || CONV == 3) {
          // k-tile -> (filter tap, 64-channel block); base pixel of this CTA's 128 output pixels in input coords
          const int kt = kt_begin + i;
          const int cblocks = p.conv_cin >> 6;
          const int tap = kt / cblocks, cb = kt - tap * cblocks;
          const int fr = tap / p.conv_kw, fs = tap - fr * p.conv_kw;
          const int q0 = m0 % p.conv_wo, t0 = m0 / p.conv_wo;
          tma_load_im2col_4d(sa, &tmA, &full_bar[s], cb * 64, q0 * p.conv_stride - p.conv_pad,
                             (t0 % p.conv_ho) * p.conv_stride - p.conv_pad, t0 / p.conv_ho, fs, fr);
        } else if (!p.a_mn) {
          tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);  // box [64 k][128 rows]
        } else {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j)  // box [64 m][64 k rows] per MN atom
            tma_load_2d(sa + j * 8192, &tmA, &full_bar[s], m0 + j * 64, k0);
        }
        if constexpr (CONV == 2) {
          // k-tile = 64 output pixels starting at k0; N atom j = (tap, channel block) of column n0 + 64 j
          const int q0 = k0 % p.conv_wo, t0 = k0 / p.conv_wo;
          const int w0 = q0 * p.conv_stride - p.conv_pad, h0 = (t0 % p.conv_ho) * p.conv_stride - p.conv_pad;
          const int img = t0 / p.conv_ho;
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) {
            const int col = n0 + j * 64;
            if (col < p.N) {          // atoms past the last tap are never stored: leave them (expect_tx below)
              const int tap = col / p.conv_cin, c = col - tap * p.conv_cin;
              const int fr = tap / p.conv_kw, fs = tap - fr * p.conv_kw;
              tma_load_im2col_4d(sb + j * 8192, &tmB, &full_bar[s], c, w0, h0, img, fs, fr);
            }
          }
        } else if constexpr (CONV == 3) {
          const int kt = kt_begin + i;
          const int cblocks = p.conv_cin >> 6;
          const int tap = kt / cblocks, cb = kt - tap * cblocks;
          const int wcol = (p.conv_taps - 1 - tap) * p.conv_ncol + n0;      // flipped tap, cin block of this CTA
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[s], wcol + j * 64, cb * 64);
        } else if (!p.b_mn) {
          tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);  // box [64 k][BN rows]
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[s], n0 + j * 64, k0);
        }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: two warpgroups of wgmma, then the epilogue =====================
    const int ew = warp - 4;                    // 0..7
    __nv_bfloat16* lora_us = reinterpret_cast<__nv_bfloat16*>(cstat + 8 * BN);
    __nv_bfloat16* lora_fs = lora_us + BM * (p.lora_R + 8);
    if constexpr (LORA) lora_stage<BN>(p, lora_us, lora_fs, m0, n0);   // read after the barriers below
    float acc[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    consume_ktiles<BN>(acc, smem, STAGES, full_bar, empty_bar, s, ph, num_kt, p.a_mn, p.b_mn, ew >> 2);
    if (threadIdx.x == 128) TRACE_POINT();  // fixed: accumulator complete (epilogue starts)
    named_bar_sync(1, CONSUMER_THREADS);        // both warpgroups' MMAs retired: the ring may be overwritten
    float* part = reinterpret_cast<float*>(smem);
    wg_store_acc<BN>(acc, part, L::PART_PITCH, 64 * (ew >> 2));
    named_bar_sync(1, CONSUMER_THREADS);
    // Row-per-lane epilogue over the staged tile: warp ew reads rows 32 (ew % 4) .. + 31, the two warps sharing a row
    // quarter split the 32-column chunks between them.
    const int q = ew & 3;
    constexpr int NCHUNK = BN / 32;
    const int c_begin = (ew < 4 ? 0 : (NCHUNK + 1) / 2) * 32, c_end = (ew < 4 ? (NCHUNK + 1) / 2 : NCHUNK) * 32;
    const int lrow = q * 32 + static_cast<int>(lane_id());
    const int row = m0 + lrow;
    const int orow = CONV == 4 ? s2_dx_row(p, cls, row) : row;   // output row (CONV == 4: -1 = not stored)
    const bool row_ok = CONV == 4 ? orow >= 0 : row < p.M;
    const size_t elt = p.out_fp32 ? 4 : 2;
    uint8_t* drow = reinterpret_cast<uint8_t*>(p.D) +
                    (static_cast<size_t>(CONV == 4 && orow < 0 ? 0 : orow) * p.ldd + static_cast<size_t>(bz_outer) * p.d_outer +
                     static_cast<size_t>(bz_inner) * p.d_inner) * elt;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && ((p.ldd * elt) % 16 == 0);
    const bool sgd_vec = SGD && (p.ldd % 4 == 0) &&
                         ((reinterpret_cast<uintptr_t>(p.sgd_theta) | reinterpret_cast<uintptr_t>(p.sgd_mom) |
                           (PROX ? reinterpret_cast<uintptr_t>(p.sgd_anchor) : 0) |
                           (SCAF ? reinterpret_cast<uintptr_t>(p.sgd_corr) : 0) |
                           (ADAM ? reinterpret_cast<uintptr_t>(p.sgd_v) : 0)) & 15) == 0 &&
                         (reinterpret_cast<uintptr_t>(p.sgd_wb) & 7) == 0;
    // fused BatchNorm statistics: per row quarter column sums, [4 quarters][2 * BN] floats
    float* sstat = cstat + q * 2 * BN;
    const bool want_stats = p.col_stats != nullptr;
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 32) {
      uint32_t r[32];
      acc_ld_row32(part + lrow * L::PART_PITCH + c, r);
      const int col0 = n0 + c;
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
      if (col0 >= p.N) {                          // warp-uniform
        if (want_stats) { sstat[c + lane_id()] = 0.f; sstat[BN + c + lane_id()] = 0.f; }
        continue;
      }
      if constexpr (LORA) lora_chunk(p, lora_us, lora_fs, lrow, c, col0, v);
      if constexpr (AFFINE) {
        if (!row_ok) continue;
        affine_chunk<32>(p, row, col0, v);
      } else {
        transform_chunk<32>(p, col0, v);
        if (want_stats) stage_col_stats(sstat, BN, c, v);
        if (!row_ok) continue;
      }
      const bool full = (col0 + 32 <= p.N);
      if constexpr (SGD) {
        if constexpr (ADAM) adamw_epilogue_chunk(p, static_cast<size_t>(row) * p.ldd + col0, col0, v, sgd_vec);
        else sgd_epilogue_chunk<PROX, SCAF>(p, static_cast<size_t>(row) * p.ldd + col0, col0, v, sgd_vec);
        continue;
      }
      if (p.atomic_out) {
        float* d = reinterpret_cast<float*>(drow) + col0;
        if (full && vec_ok) {
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + j), "f"(v[j]), "f"(v[j + 1]),
                         "f"(v[j + 2]), "f"(v[j + 3])
                         : "memory");
        } else {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) atomicAdd(d + j, v[j]);
        }
      } else if (p.out_fp32) {
        float* d = reinterpret_cast<float*>(drow) + col0;
        if (full && vec_ok) {
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            *reinterpret_cast<float4*>(d + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
        } else {
          _Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) d[j] = v[j];
        }
      } else {
        __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(drow) + col0;
        if (full && vec_ok) {
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
    if (threadIdx.x == 128) TRACE_POINT();  // fixed: epilogue stores issued
    if (want_stats) {
      named_bar_sync(1, CONSUMER_THREADS);                 // all eight warps staged their column sums
      for (int i = threadIdx.x - 128; i < 2 * BN; i += CONSUMER_THREADS) {
        const int col = i < BN ? i : i - BN;
        if (n0 + col < p.N)
          atomicAdd(p.col_stats + (i < BN ? 0 : p.N) + n0 + col,
                    cstat[i] + cstat[2 * BN + i] + cstat[4 * BN + i] + cstat[6 * BN + i]);
      }
    }
  }
}


// Epilogue of one 128 x BN accumulator tile for the persistent kernel, read back from the staged fp32 tile one
// row per lane.  Direct stores would scatter 16 B pieces over 32 different output rows per instruction; instead each
// warp stages 32 rows x 128 B in shared memory (pitch 144 B: conflict-free 16 B accesses) and writes them back with
// lanes running along the row -- every store instruction covers four complete 128 B row segments.  The two warps of
// a row quarter (`half` 0 / 1) take alternate 128-byte column passes.
constexpr int EPI_PITCH = 144;
constexpr int EPI_WARP_BYTES = 32 * EPI_PITCH;

template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float* acc_tile, int q, int half, int m0,
                                              int n0, uint8_t* stage, bool vec_ok, size_t d_off = 0) {
  using L = SmemLayout<BN>;
  const int lane = static_cast<int>(lane_id());
  const int row = m0 + q * 32 + lane;
  const float* arow = acc_tile + (q * 32 + lane) * L::PART_PITCH;
  const int elt = p.out_fp32 ? 4 : 2;
  const bool fast = vec_ok && !p.atomic_out && (p.N % 8 == 0);
  if (!fast) {
#pragma unroll 1
    for (int c = half * 32; c < BN; c += 64) {
      uint32_t r[32];
      acc_ld_row32(arow + c, r);
      const int col0 = n0 + c;
      if (col0 >= p.N) continue;                  // warp-uniform
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
      if (p.col_stats != nullptr) accumulate_col_stats(p, col0, v);   // alpha == 1, no bias / act in this mode
      if (row >= p.M) continue;
      store_row_chunk<32>(p, row, col0, v, vec_ok, d_off);
    }
    return;
  }
  const int W = 128 / elt;                          // output columns per 128-byte pass
  uint8_t* srow = stage + lane * EPI_PITCH;
#pragma unroll 1
  for (int c0 = half * W; c0 < BN; c0 += 2 * W) {
    if (n0 + c0 >= p.N) break;                      // warp-uniform
    for (int cc = 0; cc < W; cc += 32) {
      uint32_t r[32];
      acc_ld_row32(arow + c0 + cc, r);
      const int col0 = n0 + c0 + cc;
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
      transform_chunk<32>(p, col0, v);
      if (p.col_stats != nullptr) accumulate_col_stats(p, col0, v);
      if (p.out_fp32) {
#pragma unroll
        for (int j = 0; j < 32; j += 4)
          *reinterpret_cast<float4*>(srow + (cc + j) * 4) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 32; j += 8)
          *reinterpret_cast<uint4*>(srow + (cc + j) * 2) =
              make_uint4(pack_bf16x2(v[j], v[j + 1]), pack_bf16x2(v[j + 2], v[j + 3]), pack_bf16x2(v[j + 4], v[j + 5]),
                         pack_bf16x2(v[j + 6], v[j + 7]));
      }
    }
    __syncwarp();
    const int per16 = 16 / elt;                     // columns per 16-byte chunk
#pragma unroll
    for (int it = 0; it < 8; ++it) {                // 32 rows x 8 chunks = 256 chunks, 32 per instruction
      const int idx = it * 32 + lane;
      const int r = idx >> 3, ch = idx & 7;
      const int grow = m0 + q * 32 + r;
      const int col = n0 + c0 + ch * per16;
      if (grow < p.M && col < p.N) {
        const uint4 val = *reinterpret_cast<const uint4*>(stage + r * EPI_PITCH + ch * 16);
        *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(p.D) +
                                  (d_off + static_cast<size_t>(grow) * p.ldd + col) * elt) = val;
      }
    }
    __syncwarp();
  }
}

// ---- persistent kernel: one CTA per SM walks the tile list; the TMA producer runs ahead across tile
// ---- boundaries, so the loads of tile i+1 overlap the epilogue of tile i (large problems: >= one wave of tiles) ----
template <int BN, int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                            const GemmParams p) {
  using L = SmemLayout<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* acc_tile = reinterpret_cast<float*>(smem + STAGES * L::STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES + L::PART_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint8_t* epi_stage = reinterpret_cast<uint8_t*>(empty_bar + STAGES);   // 8 warps x 32 rows x 144 B

  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int tiles_per_z = tiles_m * tiles_n;
  const int num_tiles = tiles_per_z * (p.batched ? p.batch_count : 1);   // batched: z-major tile list
  const int num_kt = (p.K + BK - 1) / BK;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();

  if (warp == 0) {
    // ===================== TMA producer: runs ahead across tile boundaries =====================
    if (elect_one()) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        // consecutive CTAs share the same N block (the B tile stays hot in L2) and walk M
        const int z = tile / tiles_per_z, rem = tile - z * tiles_per_z;
        const int m0 = (rem % tiles_m) * BM, n0 = (rem / tiles_m) * BN;
        const int zo = p.batched ? z / p.batch_inner : 0, zi = p.batched ? z % p.batch_inner : 0;
        for (int kt = 0; kt < num_kt; ++kt) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          const int k0 = kt * BK;
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
          if (p.batched) {
            if (!p.a_mn) {
              tma_load_4d(sa, &tmA, &full_bar[s], k0, m0, zi, zo);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_4d(sa + j * 8192, &tmA, &full_bar[s], m0 + j * 64, k0, zi, zo);
            }
            if (!p.b_mn) {
              tma_load_4d(sb, &tmB, &full_bar[s], k0, n0, zi, zo);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_4d(sb + j * 8192, &tmB, &full_bar[s], n0 + j * 64, k0, zi, zo);
            }
          } else {
            if (!p.a_mn) {
              tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * 8192, &tmA, &full_bar[s], m0 + j * 64, k0);
            }
            if (!p.b_mn) {
              tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[s], n0 + j * 64, k0);
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: main loop, stage the accumulator, epilogue =====================
    const int ew = warp - 4;
    const size_t elt = p.out_fp32 ? 4 : 2;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && ((p.ldd * elt) % 16 == 0);
    int s = 0;
    uint32_t ph = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int z = tile / tiles_per_z, rem = tile - z * tiles_per_z;
      const int m0 = (rem % tiles_m) * BM, n0 = (rem / tiles_m) * BN;
      size_t d_off = 0;
      if (p.batched)
        d_off = static_cast<size_t>(z / p.batch_inner) * p.d_outer + static_cast<size_t>(z % p.batch_inner) * p.d_inner;
      consume_ktiles<BN>(acc, smem, STAGES, full_bar, empty_bar, s, ph, num_kt, p.a_mn, p.b_mn, ew >> 2);
      named_bar_sync(1, CONSUMER_THREADS);          // the previous tile's epilogue is done with the staged tile
      wg_store_acc<BN>(acc, acc_tile, L::PART_PITCH, 64 * (ew >> 2));
      named_bar_sync(1, CONSUMER_THREADS);
      epilogue_tile<BN>(p, acc_tile, ew & 3, ew >> 2, m0, n0, epi_stage + ew * EPI_WARP_BYTES,
                        vec_ok && ((d_off * elt) & 15) == 0, d_off);
    }
  }
}


// ---- runtime-depth pipeline + cluster split-K (DSMEM reduce) ----
// AFFINE: eval-mode BatchNorm epilogue (affine_chunk), applied by the CTA that stores the reduced rows
template <int BN, bool CLUSTER, int CONV = 0, bool AFFINE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_splitk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const GemmParams p) {
  using L = SmemLayout<BN>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem is only guaranteed 16B aligned: realign to the 1024B the 128B swizzle needs
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int STAGES = p.stages;
  const int ring_bytes = STAGES * L::STAGE_BYTES;
  const int data_bytes = L::PART_BYTES > ring_bytes ? L::PART_BYTES : ring_bytes;   // the drained ring holds the fp32 tile
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + data_bytes);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  float* cstat = reinterpret_cast<float*>(empty_bar + MAX_STAGES);   // [4 warps][2 * BN] column statistics of this CTA's rows

  griddep_launch_dependents();  // PDL: the next kernel may start its prologue now
  const int warp = threadIdx.x >> 5;
  const int m0 = blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int k_tiles_total = (p.K + BK - 1) / BK;
  const int kt_begin = blockIdx.z * p.k_tiles_per_split;
  int kt_end = kt_begin + p.k_tiles_per_split;
  if (kt_end > k_tiles_total) kt_end = k_tiles_total;
  const int num_kt = kt_end - kt_begin;  // host guarantees >= 1 for every launched z

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();  // PDL: everything above overlapped the previous kernel; its results are visible from here

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      if (p.tile_flags != nullptr) {
        // bcast_gemm: wait until the FedAvg kernel has published every arena tile under the rows
        // [n0, n0+BN) of the (K-major) weight matrix this CTA is about to TMA-load
        const int rows_here = (p.N - n0) < BN ? (p.N - n0) : BN;
        const uint32_t need = p.flag_epoch_ptr != nullptr ? *reinterpret_cast<const volatile uint32_t*>(p.flag_epoch_ptr)
                                                          : p.flag_epoch;
        wait_arrival_flags(p.tile_flags, p.flag_elem_off + static_cast<long long>(n0) * p.ldb,
                           p.flag_elem_off + static_cast<long long>(n0 + rows_here) * p.ldb - 1, p.flag_tile_elems, need);
        if (p.flag_bias_off >= 0)  // the bias slice the epilogue of this CTA will add
          wait_arrival_flags(p.tile_flags, p.flag_bias_off + n0, p.flag_bias_off + n0 + rows_here - 1,
                             p.flag_tile_elems, need);
        fence_proxy_async_all();  // order the acquires before the async-proxy (TMA) reads of global memory
      }
      int s = 0;
      uint32_t ph = 0;
      for (int i = 0; i < num_kt; ++i) {
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * L::STAGE_BYTES;
        uint8_t* sb = sa + L::A_BYTES;
        const int k0 = (kt_begin + i) * BK;
        mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
        if constexpr (CONV == 1 || CONV == 3) {
          const int kt = kt_begin + i;
          const int cblocks = p.conv_cin >> 6;
          const int tap = kt / cblocks, cb = kt - tap * cblocks;
          const int fr = tap / p.conv_kw, fs = tap - fr * p.conv_kw;
          const int q0 = m0 % p.conv_wo, t0 = m0 / p.conv_wo;
          tma_load_im2col_4d(sa, &tmA, &full_bar[s], cb * 64, q0 * p.conv_stride - p.conv_pad,
                             (t0 % p.conv_ho) * p.conv_stride - p.conv_pad, t0 / p.conv_ho, fs, fr);
        } else if (!p.a_mn) {
          tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);  // box [64 k][128 rows]
        } else {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j)  // box [64 m][64 k rows] per MN atom
            tma_load_2d(sa + j * 8192, &tmA, &full_bar[s], m0 + j * 64, k0);
        }
        if constexpr (CONV == 3) {
          const int kt = kt_begin + i;
          const int cblocks = p.conv_cin >> 6;
          const int tap = kt / cblocks, cb = kt - tap * cblocks;
          const int wcol = (p.conv_taps - 1 - tap) * p.conv_ncol + n0;
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[s], wcol + j * 64, cb * 64);
        } else if (!p.b_mn) {
          tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);  // box [64 k][BN rows]
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, &full_bar[s], n0 + j * 64, k0);
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers (phase 1): main loop, accumulator -> shared memory =====================
    const int ew = warp - 4;
    float acc[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    consume_ktiles<BN>(acc, smem, STAGES, full_bar, empty_bar, s, ph, num_kt, p.a_mn, p.b_mn, ew >> 2);
    named_bar_sync(1, CONSUMER_THREADS);        // both warpgroups' MMAs retired: the ring may be overwritten
    float* part = reinterpret_cast<float*>(smem);
    wg_store_acc<BN>(acc, part, L::PART_PITCH, 64 * (ew >> 2));
    if constexpr (!CLUSTER) {
      named_bar_sync(1, CONSUMER_THREADS);
      const int q = ew & 3;
      constexpr int NCHUNK = BN / 32;
      const int c_begin = (ew < 4 ? 0 : (NCHUNK + 1) / 2) * 32, c_end = (ew < 4 ? (NCHUNK + 1) / 2 : NCHUNK) * 32;
      const int lrow = q * 32 + static_cast<int>(lane_id());
      const int row = m0 + lrow;
      const size_t elt = p.out_fp32 ? 4 : 2;
      const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && ((p.ldd * elt) % 16 == 0);
#pragma unroll 1
      for (int c = c_begin; c < c_end; c += 32) {
        const int col0 = n0 + c;
        if (row >= p.M || col0 >= p.N) continue;
        uint32_t r[32];
        acc_ld_row32(part + lrow * L::PART_PITCH + c, r);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
        store_row_chunk<32, AFFINE>(p, row, col0, v, vec_ok);
      }
    }
  }

  if constexpr (CLUSTER) {
    // ===================== cluster split-K: reduce the S partial tiles through DSMEM =====================
    const int S = p.cluster_k;
    cluster_sync_all();  // every CTA's partial tile is in its shared memory
    if (warp >= 4 && warp < 8) {                 // four warps of the first consumer warpgroup
      const uint32_t me = cluster_ctarank();
      const int rows_per = BM / S;                 // S in {2, 4, 8}
      constexpr int CG = BN / 8;                   // 8-column groups per row
      const int t = threadIdx.x - 128;             // 0..127
      const size_t elt = p.out_fp32 ? 4 : 2;
      const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && ((p.ldd * elt) % 16 == 0);
      const bool want_stats = p.col_stats != nullptr;
      // 128 % CG == 0: a thread always lands on the same 8 columns, so its statistics stay in registers
      float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, cq[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int item = t; item < rows_per * CG; item += 128) {
        const int lrow = static_cast<int>(me) * rows_per + item / CG;
        const int c = (item % CG) * 8;
        const uint32_t laddr = smem_u32(smem) + static_cast<uint32_t>((lrow * L::PART_PITCH + c) * 4);
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int r = 0; r < S; ++r) {              // fixed order: deterministic sum
          const float4 a = ld_dsmem_f4(laddr, r), b = ld_dsmem_f4(laddr + 16, r);
          v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
          v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
        }
        const int row = m0 + lrow, col0 = n0 + c;
        if (want_stats) {                          // rows >= M are exact zeros (TMA zero fill)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float rnd = __bfloat162float(__float2bfloat16_rn(v[j]));
            cs[j] += rnd;
            cq[j] = fmaf(rnd, rnd, cq[j]);
          }
        }
        if (row < p.M && col0 < p.N) store_row_chunk<8, AFFINE>(p, row, col0, v, vec_ok);
      }
      if (want_stats) {
        // threads t, t + CG, t + 2 CG ... own the same 8 columns: fold the lanes of a warp with shuffles, park one
        // row of partials per warp in shared memory (plain stores), then one thread per column adds the four warps
        // and issues the global atomics.  (A shared-memory atomicAdd version serialises 16-way on a CAS loop.)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int o = CG; o < 32; o <<= 1) {
            cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], o);
            cq[j] += __shfl_xor_sync(0xffffffffu, cq[j], o);
          }
        }
        const int wq = t >> 5, ln = t & 31;
        if (ln < CG) {                               // CG <= 32: lanes 0..CG-1 hold the warp's sums of columns ln*8..+7
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            cstat[wq * 2 * BN + ln * 8 + j] = cs[j];
            cstat[wq * 2 * BN + BN + ln * 8 + j] = cq[j];
          }
        }
        named_bar_sync(2, 128);                         // the four reducing warps only
        for (int i = t; i < 2 * BN; i += 128) {
          const int col = i < BN ? i : i - BN;
          if (n0 + col < p.N) {
            const float v = cstat[i] + cstat[2 * BN + i] + cstat[4 * BN + i] + cstat[6 * BN + i];
            atomicAdd(p.col_stats + (i < BN ? 0 : p.N) + n0 + col, v);
          }
        }
      }
    }
    cluster_sync_all();  // nobody leaves (and frees its smem) while a peer may still read it
  }
}


// --------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  // cuTensorMapEncodeTiled is a DRIVER entry point: it needs a current context on the calling
  // thread.  Autograd worker threads may not have touched the runtime yet -> bind the primary
  // context once per thread (cudaFree(0) is the canonical no-op that does so).
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 2-D bf16 tensor map over a row-major [rows, cols] matrix with row pitch `ld` elements;
// box = [box_cols (inner), box_rows], 128B swizzle (box_cols must be 64) unless `swizzle` is another mode (its span
// bounds box_cols).
static int make_map(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, int box_cols,
                    int box_rows, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// 4-D bf16 tensor map: [outer][inner][rows][cols] with element strides; box = [box_cols, box_rows, 1, 1]
static int make_map4(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, long long inner,
                     long long s_inner, long long outer, long long s_outer, int box_cols, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[4] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(inner),
                        static_cast<cuuint64_t>(outer)};
  cuuint64_t gstr[3] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(s_inner) * 2,
                        static_cast<cuuint64_t>(s_outer) * 2};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows), 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// BN wider than 128 is not instantiated (see the top of the file): a requested 256 runs as 128.
static int clamp_bn(int bn) { return bn > 128 ? 128 : bn; }

static void set_sgd_epilogue(GemmParams& p, const B200SgdEpilogue& s) {
  p.sgd_hyper = s.hyper; p.sgd_theta = s.theta; p.sgd_wb = reinterpret_cast<__nv_bfloat16*>(s.theta_bf16);
  p.sgd_mom = s.mom; p.sgd_nesterov = s.nesterov; p.sgd_anchor = s.anchor; p.sgd_corr = s.corr; p.sgd_v = s.v;
}

static void set_affine_epilogue(GemmParams& p, const B200AffineEpilogue& a) {
  p.bn_scale = a.scale; p.bn_shift = a.shift; p.residual = reinterpret_cast<const __nv_bfloat16*>(a.residual);
  p.ldr = a.ldr; p.act = a.relu ? 1 : 0;
}

// what the affine epilogue needs of its output and operands (see affine_chunk)
static bool affine_ok(const B200AffineEpilogue& a, int N) {
  return a.scale != nullptr && a.shift != nullptr && N % 8 == 0 &&
         ((reinterpret_cast<uintptr_t>(a.scale) | reinterpret_cast<uintptr_t>(a.shift) |
           reinterpret_cast<uintptr_t>(a.residual)) & 15) == 0 &&
         (a.residual == nullptr || (a.ldr % 8 == 0 && a.ldr >= N));
}

template <int BN, int STAGES, int CONV = 0, bool SGD = false, bool AFFINE = false, bool PROX = false, bool SCAF = false,
          bool ADAM = false>
static int launch_fixed(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid,
                      cudaStream_t stream) {
  constexpr int smem = STAGES * SmemLayout<BN>::STAGE_BYTES + 2 * STAGES * 8 + 8 * BN * 4 + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_fixed_kernel<BN, STAGES, CONV, SGD, AFFINE, PROX, SCAF, ADAM>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  cudaError_t le = launch_pdl(gemm_bf16_fixed_kernel<BN, STAGES, CONV, SGD, AFFINE, PROX, SCAF, ADAM>, grid, GEMM_THREADS, smem, stream,
                              ta, tb, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

// the optimizer-epilogue instantiation, in its FedProx form when the step has an anchor, in its SCAFFOLD form when it
// has a correction, in its AdamW form when it has a second moment
template <int BN, int STAGES, int CONV>
static int launch_fixed_sgd(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid,
                            cudaStream_t stream) {
  if (p.sgd_anchor != nullptr && p.sgd_corr != nullptr) return -2;
  if (p.sgd_v != nullptr) {
    if (p.sgd_anchor != nullptr || p.sgd_corr != nullptr || p.sgd_mom == nullptr) return -2;
    return launch_fixed<BN, STAGES, CONV, true, false, false, false, true>(ta, tb, p, grid, stream);
  }
  if (p.sgd_corr != nullptr) return launch_fixed<BN, STAGES, CONV, true, false, false, true>(ta, tb, p, grid, stream);
  return p.sgd_anchor != nullptr ? launch_fixed<BN, STAGES, CONV, true, false, true>(ta, tb, p, grid, stream)
                                 : launch_fixed<BN, STAGES, CONV, true>(ta, tb, p, grid, stream);
}

// the LoRA instantiation: its dynamic shared memory grows with the staged U and factor rows (lora_stage)
template <int BN, int STAGES>
static int launch_fixed_lora(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid,
                             cudaStream_t stream) {
  constexpr int base = STAGES * SmemLayout<BN>::STAGE_BYTES + 2 * STAGES * 8 + 8 * BN * 4 + 1024;
  constexpr int cap = base + (BM + BN) * (B200_LORA_MAX_R + 8) * 2;
  static_assert(cap <= 227 * 1024, "LoRA GEMM exceeds the 227 KB of shared memory a block may use");
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_fixed_kernel<BN, STAGES, 0, false, false, false, false, false, true>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  const int smem = base + (BM * (p.lora_R + 8) + BN * (p.lora_rs + 8)) * 2;
  cudaError_t le = launch_pdl(gemm_bf16_fixed_kernel<BN, STAGES, 0, false, false, false, false, false, true>, grid,
                              GEMM_THREADS, smem, stream, ta, tb, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

template <int BN, int STAGES>
static int launch_persistent(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int num_tiles,
                             cudaStream_t stream) {
  constexpr int smem = STAGES * SmemLayout<BN>::STAGE_BYTES + SmemLayout<BN>::PART_BYTES + 2 * STAGES * 8 +
                       CONSUMER_WARPS * EPI_WARP_BYTES + 1024;
  static_assert(smem <= 227 * 1024, "persistent GEMM exceeds the 227 KB of shared memory a block may use");
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_persistent_kernel<BN, STAGES>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  const int grid = num_tiles < device_sm_count() ? num_tiles : device_sm_count();
  cudaError_t le = launch_pdl(gemm_bf16_persistent_kernel<BN, STAGES>, dim3(grid), GEMM_THREADS, smem, stream, ta, tb, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

template <int BN, int CONV = 0, bool AFFINE = false>
static int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid,
                      cudaStream_t stream) {
  using L = SmemLayout<BN>;
  constexpr int max_stages = BN == 128 ? 6 : 8;
  constexpr int max_smem = max_stages * L::STAGE_BYTES + 2 * MAX_STAGES * 8 + 8 * BN * 4 + 1024;
  static bool configured = false;
  if (!configured) {
    const int cap = max_smem > L::PART_BYTES + 4096 ? max_smem : L::PART_BYTES + 4096;
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_splitk_kernel<BN, false, CONV, AFFINE>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_bf16_splitk_kernel<BN, true, CONV, AFFINE>,
                               cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  int ring = p.stages * L::STAGE_BYTES;
  if (L::PART_BYTES > ring) ring = L::PART_BYTES;
  int smem = ring + 2 * MAX_STAGES * 8 + 8 * BN * 4 + 1024;
  // occupancy cap: CTAs of this kernel per SM (shared memory is the limiter we control)
  constexpr int max_ctas = 2;
  // atomic epilogues (wgrad): one CTA per SM, co-resident CTAs only contend for the same output lines
  const int ctas_here = p.atomic_out ? 1 : max_ctas;
  const int floor_smem = (227 * 1024) / (ctas_here + 1) + 1024;   // > 1/(ctas+1) of the SM
  if (smem < floor_smem && floor_smem <= max_smem) smem = floor_smem;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (p.cluster_k > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = 1;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = p.cluster_k;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaError_t le = p.cluster_k > 1 ? cudaLaunchKernelEx(&cfg, gemm_bf16_splitk_kernel<BN, true, CONV, AFFINE>, ta, tb, p)
                                   : cudaLaunchKernelEx(&cfg, gemm_bf16_splitk_kernel<BN, false, CONV, AFFINE>, ta, tb, p);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace b200

// D = act(alpha * A B^T + bias).  a/b: bf16 device pointers.
//   a_mn == 0: A is row-major [M, K] with pitch lda;  a_mn == 1: A is row-major [K, M] with pitch lda
//   b_mn == 0: B is row-major [N, K] with pitch ldb;  b_mn == 1: B is row-major [K, N] with pitch ldb
//   split_k > 1 with accumulate / fp32 atomic output -> atomic split-K; split_k < 0 -> cluster split-K of
//   size -split_k (2, 4 or 8) for any output type.
// Returns 0 on success, a CUDA / driver error code otherwise, -2 on unsupported alignment.
// tensor-map encoders for other translation units (attention.cu)
extern "C" int b200_encode_map2_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     int box_cols, int box_rows) {
  return b200::make_map(reinterpret_cast<CUtensorMap*>(map), base, rows, cols, ld, box_cols, box_rows);
}
// the same with a 64-byte swizzle (conv_halo.cu: the MN-major [64 cout] x [32 cin] weight slab of a 32-column tile)
extern "C" int b200_encode_map2_sw64_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                          int box_cols, int box_rows) {
  return b200::make_map(reinterpret_cast<CUtensorMap*>(map), base, rows, cols, ld, box_cols, box_rows,
                        CU_TENSOR_MAP_SWIZZLE_64B);
}
extern "C" int b200_encode_map4_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     long long inner, long long s_inner, long long outer, long long s_outer,
                                     int box_cols, int box_rows) {
  return b200::make_map4(reinterpret_cast<CUtensorMap*>(map), base, rows, cols, ld, inner, s_inner, outer, s_outer,
                         box_cols, box_rows);
}
// 4-D bf16 tensor map with an arbitrary box (conv_halo.cu: one halo box of whole images); dims innermost first,
// `stride_bytes` of dims 1..3, 128B swizzle, out-of-bounds elements read as zero
extern "C" int b200_encode_map4_box_bf16(void* map, const void* base, const long long* dims, const long long* stride_bytes,
                                         const int* box) {
  b200::EncodeTiledFn fn = b200::get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[4], gstr[3];
  cuuint32_t bx[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) {
    gdim[i] = static_cast<cuuint64_t>(dims[i]);
    bx[i] = static_cast<cuuint32_t>(box[i]);
    if (i < 3) gstr[i] = static_cast<cuuint64_t>(stride_bytes[i]);
  }
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(map), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim,
                  gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

extern "C" int b200_gemm_bf16(const void* a, const void* b, void* d, const float* bias, int M, int N, int K,
                              long long lda, long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32, int act,
                              int split_k, int accumulate, float alpha, const uint32_t* tile_flags,
                              uint32_t flag_epoch, long long flag_elem_off, int flag_tile_elems,
                              long long flag_bias_off, int force_bn, float* col_stats, const uint32_t* flag_epoch_ptr,
                              const B200SgdEpilogue* sgd, const B200AffineEpilogue* affine, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  // optimizer epilogue: only a weight gradient (MN-major operands, plain fp32 accumulation) qualifies
  if (sgd != nullptr && (!accumulate || !out_fp32 || !a_mn || !b_mn || bias != nullptr || act != 0 || alpha != 1.0f ||
                         col_stats != nullptr || tile_flags != nullptr))
    return B200_SGD_EPILOGUE_DECLINED;
  // eval-mode BatchNorm epilogue: a plain bf16 forward GEMM, one K pass per CTA or a cluster split-K
  if (affine != nullptr && (sgd != nullptr || accumulate || out_fp32 || bias != nullptr || act != 0 || alpha != 1.0f ||
                            col_stats != nullptr || tile_flags != nullptr || split_k > 1 || !affine_ok(*affine, N)))
    return B200_AFFINE_EPILOGUE_DECLINED;
  // fused BatchNorm statistics: plain single-pass GEMM only (no split-K partials, no bias / activation / scaling)
  if (col_stats != nullptr && (split_k > 1 || bias != nullptr || act != 0 || alpha != 1.0f || accumulate)) return -3;
  if ((lda % 8) || (ldb % 8) || (reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15))
    return -2;
  const int bn = clamp_bn(force_bn > 0 ? force_bn : (N > 64 ? 128 : 64));
  if (tile_flags != nullptr && (b_mn || flag_tile_elems <= 0)) return -4;
  CUtensorMap ta, tb;
  int rc;
  if (!a_mn)
    rc = make_map(&ta, a, M, K, lda, BK, BM);
  else
    rc = make_map(&ta, a, K, M, lda, 64, BK);
  if (rc) return rc;
  if (!b_mn)
    rc = make_map(&tb, b, N, K, ldb, BK, bn);
  else
    rc = make_map(&tb, b, K, N, ldb, 64, BK);
  if (rc) return rc;

  const int k_tiles = (K + BK - 1) / BK;
  int cluster_k = 1;
  if (split_k < 0) {  // cluster split-K: every z-slice must own at least one k tile
    cluster_k = -split_k;
    if (cluster_k != 2 && cluster_k != 4 && cluster_k != 8) return -5;
    while (cluster_k > 1 && (cluster_k - 1) * ((k_tiles + cluster_k - 1) / cluster_k) >= k_tiles) cluster_k >>= 1;
    split_k = cluster_k;
  }
  if (split_k < 1) split_k = 1;
  if (split_k > k_tiles) split_k = k_tiles;
  int per = (k_tiles + split_k - 1) / split_k;
  if (cluster_k == 1) split_k = (k_tiles + per - 1) / per;  // no empty z-slices
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.D = d; p.ldd = ldd; p.bias = bias; p.out_fp32 = out_fp32; p.act = act;
  p.a_mn = a_mn; p.b_mn = b_mn; p.k_tiles_per_split = per;
  p.cluster_k = cluster_k;
  p.atomic_out = (accumulate || (split_k > 1 && cluster_k == 1)) ? 1 : 0;
  p.col_stats = col_stats;
  p.tile_flags = tile_flags; p.flag_epoch = flag_epoch; p.alpha = alpha;
  p.flag_elem_off = flag_elem_off; p.flag_tile_elems = flag_tile_elems; p.ldb = ldb;
  p.flag_bias_off = (tile_flags != nullptr && bias != nullptr) ? flag_bias_off : -1;
  p.flag_epoch_ptr = tile_flags != nullptr ? flag_epoch_ptr : nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  if (p.atomic_out && (!out_fp32 || bias != nullptr || act != 0)) return -3;
  const int max_stages = bn == 128 ? 6 : 8;
  p.stages = per < max_stages ? (per < 2 ? 2 : per) : max_stages;
  dim3 grid((N + bn - 1) / bn, (M + BM - 1) / BM, split_k);
  // large plain GEMMs (>= one wave of tiles, single K pass): persistent kernel with overlapped epilogue
  const int num_tiles = static_cast<int>(grid.x * grid.y);
  // the affine epilogue runs on the fixed-depth kernel where the persistent one would be picked
  const bool persistent = split_k == 1 && tile_flags == nullptr && num_tiles >= device_sm_count() && bn == 128 &&
                          affine == nullptr;
  if (sgd != nullptr) {
    // the optimizer epilogue lives in the fixed-depth kernel and needs each tile's complete gradient in one CTA
    if (split_k != 1 || cluster_k != 1 || persistent) return B200_SGD_EPILOGUE_DECLINED;
    set_sgd_epilogue(p, *sgd);
  }
  const bool shallow = per <= 4 && !p.batched;
  if (affine != nullptr) {
    set_affine_epilogue(p, *affine);
    if (cluster_k > 1)
      return bn == 128 ? launch_cfg<128, 0, true>(ta, tb, p, grid, stream) : launch_cfg<64, 0, true>(ta, tb, p, grid, stream);
    if (bn == 128)
      return shallow ? launch_fixed<128, 3, 0, false, true>(ta, tb, p, grid, stream)
                     : launch_fixed<128, 6, 0, false, true>(ta, tb, p, grid, stream);
    return shallow ? launch_fixed<64, 4, 0, false, true>(ta, tb, p, grid, stream)
                   : launch_fixed<64, 8, 0, false, true>(ta, tb, p, grid, stream);
  }
  if (cluster_k > 1) {
    if (bn == 128) return launch_cfg<128>(ta, tb, p, grid, stream);
    return launch_cfg<64>(ta, tb, p, grid, stream);
  }
  if (persistent) return launch_persistent<128, 3>(ta, tb, p, num_tiles, stream);
  // short K loops (stem convolution: 3 k tiles, 1x1 shortcuts: 1-4) do not need a deep ring: a shallow one asks for
  // little shared memory
  if (sgd != nullptr) {
    if (bn == 128)
      return shallow ? launch_fixed_sgd<128, 3, 0>(ta, tb, p, grid, stream) : launch_fixed_sgd<128, 6, 0>(ta, tb, p, grid, stream);
    return shallow ? launch_fixed_sgd<64, 4, 0>(ta, tb, p, grid, stream) : launch_fixed_sgd<64, 8, 0>(ta, tb, p, grid, stream);
  }
  if (bn == 128) return shallow ? launch_fixed<128, 3>(ta, tb, p, grid, stream) : launch_fixed<128, 6>(ta, tb, p, grid, stream);
  return shallow ? launch_fixed<64, 4>(ta, tb, p, grid, stream) : launch_fixed<64, 8>(ta, tb, p, grid, stream);
}

// D = act(alpha * (A B^T + s U F^T) + bias) with the LoRA term of B200LoraEpilogue (csrc/launch.h) in the epilogue of
// the fixed-depth kernel, one K pass per CTA.  Operand conventions as b200_gemm_bf16; D is written, not accumulated.
extern "C" int b200_gemm_bf16_lora(const void* a, const void* b, void* d, const float* bias, int M, int N, int K,
                                   long long lda, long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32,
                                   int act, float alpha, const B200LoraEpilogue* lora, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (lora == nullptr || lora->u == nullptr || lora->f == nullptr) return -3;
  const B200LoraEpilogue& l = *lora;
  if (l.R < 8 || l.R > B200_LORA_MAX_R || l.R % 8 || l.rs < 8 || l.rs % 8 || l.rs > l.R || l.ds < 32 || l.ds % 32 ||
      N > 3 * l.ds || l.ldu < l.R || l.ldu % 8 || (reinterpret_cast<uintptr_t>(l.u) & 15))
    return -3;
  for (int i = 0; i < 3; ++i)
    if (l.slot[i] < -1 || (l.slot[i] + 1) * l.rs > l.R) return -3;
  if ((lda % 8) || (ldb % 8) || (reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15))
    return -2;
  const int bn = N > 64 ? 128 : 64;
  CUtensorMap ta, tb;
  int rc = !a_mn ? make_map(&ta, a, M, K, lda, BK, BM) : make_map(&ta, a, K, M, lda, 64, BK);
  if (rc) return rc;
  rc = !b_mn ? make_map(&tb, b, N, K, ldb, BK, bn) : make_map(&tb, b, K, N, ldb, 64, BK);
  if (rc) return rc;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.D = d; p.ldd = ldd; p.bias = bias; p.out_fp32 = out_fp32; p.act = act;
  p.col_stats = nullptr; p.a_mn = a_mn; p.b_mn = b_mn; p.k_tiles_per_split = (K + BK - 1) / BK;
  p.atomic_out = 0; p.cluster_k = 1; p.tile_flags = nullptr; p.flag_epoch = 0; p.flag_elem_off = 0;
  p.flag_tile_elems = 0; p.flag_bias_off = -1; p.ldb = ldb; p.alpha = alpha; p.flag_epoch_ptr = nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  p.lora_u = reinterpret_cast<const __nv_bfloat16*>(l.u); p.lora_f = reinterpret_cast<const __nv_bfloat16*>(l.f);
  p.lora_ldu = l.ldu; p.lora_fs_n = l.fs_n; p.lora_fs_j = l.fs_j; p.lora_R = l.R; p.lora_rs = l.rs; p.lora_ds = l.ds;
  for (int i = 0; i < 3; ++i) p.lora_slot[i] = l.slot[i];
  p.lora_s = l.s;
  dim3 grid((N + bn - 1) / bn, (M + BM - 1) / BM, 1);
  if (bn == 128) { p.stages = 3; return launch_fixed_lora<128, 3>(ta, tb, p, grid, stream); }
  p.stages = 4;
  return launch_fixed_lora<64, 4>(ta, tb, p, grid, stream);
}

// Strided-batched GEMM (attention): for z = outer * n_inner + inner
//     D[z] = act(alpha * A[z] B[z]^T),  X[z] = X + outer * x_outer + inner * x_inner   (element strides)
// Same operand-major conventions as b200_gemm_bf16; every stride must be a multiple of 8 elements.
extern "C" int b200_gemm_bf16_batched(const void* a, const void* b, void* d, int M, int N, int K, long long lda,
                                      long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32, int act,
                                      float alpha, int n_outer, int n_inner, long long a_outer, long long a_inner,
                                      long long b_outer, long long b_inner, long long d_outer, long long d_inner,
                                      int accumulate, cudaStream_t stream) {
  using namespace b200;
  if (M <= 0 || N <= 0 || K <= 0 || n_outer <= 0 || n_inner <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (a_outer % 8) || (a_inner % 8) || (b_outer % 8) || (b_inner % 8) ||
      (reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15))
    return -2;
  // degenerate strides (size-1 dims) still need a non-zero multiple-of-16-byte stride for the encoder
  auto fix = [](long long s) { return s > 0 ? s : 8; };
  const int bn = N > 64 ? 128 : 64;
  CUtensorMap ta, tb;
  int rc;
  if (!a_mn)
    rc = make_map4(&ta, a, M, K, lda, n_inner, fix(a_inner), n_outer, fix(a_outer), BK, BM);
  else
    rc = make_map4(&ta, a, K, M, lda, n_inner, fix(a_inner), n_outer, fix(a_outer), 64, BK);
  if (rc) return rc;
  if (!b_mn)
    rc = make_map4(&tb, b, N, K, ldb, n_inner, fix(b_inner), n_outer, fix(b_outer), BK, bn);
  else
    rc = make_map4(&tb, b, K, N, ldb, n_inner, fix(b_inner), n_outer, fix(b_outer), 64, BK);
  if (rc) return rc;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.D = d; p.ldd = ldd; p.bias = nullptr; p.out_fp32 = out_fp32; p.act = act;
  p.a_mn = a_mn; p.b_mn = b_mn; p.k_tiles_per_split = (K + BK - 1) / BK; p.cluster_k = 1;
  p.atomic_out = accumulate ? 1 : 0;
  p.col_stats = nullptr;
  p.tile_flags = nullptr; p.flag_epoch = 0; p.alpha = alpha; p.flag_elem_off = 0; p.flag_tile_elems = 0;
  p.ldb = ldb; p.flag_bias_off = -1; p.flag_epoch_ptr = nullptr; p.stages = 4;
  p.batched = 1; p.batch_inner = n_inner; p.d_outer = d_outer; p.d_inner = d_inner;
  if (p.atomic_out && !out_fp32) return -3;
  dim3 grid((N + bn - 1) / bn, (M + BM - 1) / BM, n_outer * n_inner);
  p.batch_count = n_outer * n_inner;
  // attention-sized batches are thousands of one- or two-k-tile problems: a CTA per problem is all
  // prologue (barrier init, first TMA round trip).  Persistent CTAs amortise that and overlap
  // the epilogue of problem i with the loads + MMAs of problem i+1.
  const long long total_tiles = static_cast<long long>(grid.x) * grid.y * grid.z;
  if (total_tiles >= 2 * device_sm_count() && total_tiles < (1ll << 30)) {
    const int nt = static_cast<int>(total_tiles);
    if (bn == 128) return launch_persistent<128, 3>(ta, tb, p, nt, stream);
    return launch_persistent<64, 5>(ta, tb, p, nt, stream);
  }
  if (bn == 128) return launch_fixed<128, 6>(ta, tb, p, grid, stream);
  return launch_fixed<64, 8>(ta, tb, p, grid, stream);
}

// ---- implicit-GEMM convolution ----
extern "C" int b200_encode_map_im2col_bf16(void* map, const void* x, int N, int H, int W, int C, int KH, int KW,
                                            int stride, int pad, int channels, int pixels);

// forward: y[N*Ho*Wo, Cout] = im2col(x) w^T with x NHWC bf16 (Cin % 64 == 0), w [Cout, KH*KW*Cin] (channels_last)
extern "C" int b200_conv_igemm_fwd(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, int KH,
                                   int KW, int stride, int pad, int Ho, int Wo, int cluster_k, int force_bn,
                                   float* col_stats, const B200AffineEpilogue* affine, cudaStream_t stream) {
  using namespace b200;
  const long long M = static_cast<long long>(N) * Ho * Wo;
  const int K = KH * KW * Cin;
  if (M <= 0 || Cout <= 0) return 0;
  if (Cin % 64 != 0 || Cout % 8 != 0 || M > (1ll << 30) || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return -2;
  if (affine != nullptr && (col_stats != nullptr || !affine_ok(*affine, Cout))) return B200_AFFINE_EPILOGUE_DECLINED;
  const int bn = clamp_bn(force_bn > 0 ? force_bn : (Cout > 64 ? 128 : 64));
  CUtensorMap ta, tb;
  int rc = b200_encode_map_im2col_bf16(&ta, x, N, H, W, Cin, KH, KW, stride, pad, 64, BM);
  if (rc) return rc;
  rc = make_map(&tb, w, Cout, K, K, BK, bn);
  if (rc) return rc;
  const int k_tiles = K / BK;
  if (cluster_k != 1 && cluster_k != 2 && cluster_k != 4 && cluster_k != 8) return -5;
  while (cluster_k > 1 && (cluster_k - 1) * ((k_tiles + cluster_k - 1) / cluster_k) >= k_tiles) cluster_k >>= 1;
  const int per = (k_tiles + cluster_k - 1) / cluster_k;
  GemmParams p;
  p.M = static_cast<int>(M); p.N = Cout; p.K = K; p.D = y; p.ldd = Cout; p.bias = nullptr; p.out_fp32 = 0; p.act = 0;
  p.a_mn = 0; p.b_mn = 0; p.k_tiles_per_split = per; p.cluster_k = cluster_k; p.atomic_out = 0;
  p.col_stats = col_stats;
  p.tile_flags = nullptr; p.flag_epoch = 0; p.alpha = 1.0f; p.flag_elem_off = 0; p.flag_tile_elems = 0; p.ldb = K;
  p.flag_bias_off = -1; p.flag_epoch_ptr = nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  const int max_stages = bn == 128 ? 6 : 8;
  p.stages = per < max_stages ? (per < 2 ? 2 : per) : max_stages;
  p.conv_ho = Ho; p.conv_wo = Wo; p.conv_stride = stride; p.conv_pad = pad; p.conv_kw = KW; p.conv_cin = Cin;
  p.conv_taps = KH * KW; p.conv_ncol = Cin;
  dim3 grid((Cout + bn - 1) / bn, static_cast<unsigned>((M + BM - 1) / BM), cluster_k);
  const bool shallow = per <= 4;
  if (affine != nullptr) {
    set_affine_epilogue(p, *affine);
    if (cluster_k > 1)
      return bn == 128 ? launch_cfg<128, 1, true>(ta, tb, p, grid, stream) : launch_cfg<64, 1, true>(ta, tb, p, grid, stream);
    if (bn == 128)
      return shallow ? launch_fixed<128, 3, 1, false, true>(ta, tb, p, grid, stream)
                     : launch_fixed<128, 6, 1, false, true>(ta, tb, p, grid, stream);
    return shallow ? launch_fixed<64, 4, 1, false, true>(ta, tb, p, grid, stream)
                   : launch_fixed<64, 8, 1, false, true>(ta, tb, p, grid, stream);
  }
  if (cluster_k > 1) {
    if (bn == 128) return launch_cfg<128, 1>(ta, tb, p, grid, stream);
    return launch_cfg<64, 1>(ta, tb, p, grid, stream);
  }
  if (bn == 128) return shallow ? launch_fixed<128, 3, 1>(ta, tb, p, grid, stream) : launch_fixed<128, 6, 1>(ta, tb, p, grid, stream);
  return shallow ? launch_fixed<64, 4, 1>(ta, tb, p, grid, stream) : launch_fixed<64, 8, 1>(ta, tb, p, grid, stream);
}

// input gradient of a STRIDE-1 convolution: dx[N*H*W, Cin] = im2col_{pad' = K-1-pad}(dy) * flip(w), dy NHWC bf16
// [N, Ho, Wo, Cout] (Cout % 64 == 0), w [Cout, KH*KW*Cin] channels_last (Cin % 64 == 0 so that a 64-wide N atom never
// straddles two taps).  No col buffer, no col2im, no weight transpose.
extern "C" int b200_conv_igemm_dgrad(const void* dy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout,
                                     int KH, int KW, int pad, int Ho, int Wo, int cluster_k, int force_bn,
                                     cudaStream_t stream) {
  using namespace b200;
  const long long M = static_cast<long long>(N) * H * W;
  const int K = KH * KW * Cout;
  if (M <= 0 || Cin <= 0) return 0;
  const int padp = KH - 1 - pad, padq = KW - 1 - pad;
  if (Cout % 64 != 0 || Cin % 64 != 0 || M > (1ll << 30) || padp < 0 || padq < 0 || padp != padq ||
      Ho + 2 * padp - (KH - 1) != H || Wo + 2 * padq - (KW - 1) != W || (reinterpret_cast<uintptr_t>(dy) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(dx) & 15))
    return -2;
  const int bn = clamp_bn(force_bn > 0 ? force_bn : (Cin > 64 ? 128 : 64));
  CUtensorMap ta, tb;
  int rc = b200_encode_map_im2col_bf16(&ta, dy, N, Ho, Wo, Cout, KH, KW, 1, padp, 64, BM);
  if (rc) return rc;
  rc = make_map(&tb, w, Cout, static_cast<long long>(KH) * KW * Cin, static_cast<long long>(KH) * KW * Cin, 64, BK);
  if (rc) return rc;
  const int k_tiles = K / BK;
  if (cluster_k != 1 && cluster_k != 2 && cluster_k != 4 && cluster_k != 8) return -5;
  while (cluster_k > 1 && (cluster_k - 1) * ((k_tiles + cluster_k - 1) / cluster_k) >= k_tiles) cluster_k >>= 1;
  const int per = (k_tiles + cluster_k - 1) / cluster_k;
  GemmParams p;
  p.M = static_cast<int>(M); p.N = Cin; p.K = K; p.D = dx; p.ldd = Cin; p.bias = nullptr; p.out_fp32 = 0; p.act = 0;
  p.a_mn = 0; p.b_mn = 1; p.k_tiles_per_split = per; p.cluster_k = cluster_k; p.atomic_out = 0;
  p.col_stats = nullptr;
  p.tile_flags = nullptr; p.flag_epoch = 0; p.alpha = 1.0f; p.flag_elem_off = 0; p.flag_tile_elems = 0;
  p.ldb = static_cast<long long>(KH) * KW * Cin;
  p.flag_bias_off = -1; p.flag_epoch_ptr = nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  const int max_stages = bn == 128 ? 6 : 8;
  p.stages = per < max_stages ? (per < 2 ? 2 : per) : max_stages;
  p.conv_ho = H; p.conv_wo = W; p.conv_stride = 1; p.conv_pad = padp; p.conv_kw = KW; p.conv_cin = Cout;
  p.conv_taps = KH * KW; p.conv_ncol = Cin;
  dim3 grid((Cin + bn - 1) / bn, static_cast<unsigned>((M + BM - 1) / BM), cluster_k);
  if (cluster_k > 1) {
    if (bn == 128) return launch_cfg<128, 3>(ta, tb, p, grid, stream);
    return launch_cfg<64, 3>(ta, tb, p, grid, stream);
  }
  if (bn == 128) return launch_fixed<128, 6, 3>(ta, tb, p, grid, stream);
  return launch_fixed<64, 8, 3>(ta, tb, p, grid, stream);
}

// input gradient of a STRIDE-2 convolution by sub-pixel decomposition (see s2_class): dx[N, H, W, Cin] from dy NHWC bf16
// [N, Ho, Wo, Cout] and w [Cout, KH*KW*Cin] channels_last, both channel counts multiples of 64.  `ntaps[c]` taps of
// class c are `taps[c * S2_MAX_TAPS + t]` (filter tap | dp << 16 | dq << 24, ops/functional.py conv_s2_dgrad_taps).
// One launch for all four classes; every element of dx is written.
extern "C" int b200_conv_igemm_dgrad_s2(const void* dy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout,
                                        int KH, int KW, int Ho, int Wo, const int* ntaps, const int* taps, int force_bn,
                                        cudaStream_t stream) {
  using namespace b200;
  const long long M = static_cast<long long>(N) * Ho * Wo;   // GEMM rows of one class
  if (static_cast<long long>(N) * H * W <= 0 || Cin <= 0) return 0;
  if (Cout % 64 != 0 || Cin % 64 != 0 || M <= 0 || static_cast<long long>(N) * H * W > (1ll << 30) ||
      (H + 1) / 2 > Ho || (W + 1) / 2 > Wo || (reinterpret_cast<uintptr_t>(dy) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(dx) & 15))
    return -2;
  const long long tiles_m = (M + BM - 1) / BM;
  if (4 * tiles_m > 65535) return -2;
  GemmParams p;
  int max_taps = 0;
  for (int c = 0; c < 4; ++c) {
    if (ntaps[c] < 0 || ntaps[c] > S2_MAX_TAPS) return -2;
    for (int t = 0; t < ntaps[c]; ++t) {
      const int tw = taps[c * S2_MAX_TAPS + t];
      if (tw < 0 || (tw & 0xffff) >= KH * KW) return -2;
      p.s2_tap[c][t] = tw;
    }
    p.s2_ntaps[c] = ntaps[c];
    max_taps = ntaps[c] > max_taps ? ntaps[c] : max_taps;
  }
  if (max_taps == 0) return -2;
  const int bn = clamp_bn(force_bn > 0 ? force_bn : (Cin > 64 ? 128 : 64));
  CUtensorMap ta, tb;
  // dy traversed pixel by pixel over its own extent; the tap offsets (dq, dp) shift each gather, zero outside dy
  int rc = b200_encode_map_im2col_bf16(&ta, dy, N, Ho, Wo, Cout, 1, 1, 1, 0, 64, BM);
  if (rc) return rc;
  rc = make_map(&tb, w, Cout, static_cast<long long>(KH) * KW * Cin, static_cast<long long>(KH) * KW * Cin, 64, BK);
  if (rc) return rc;
  // single K pass per CTA: these GEMMs are short (at most 4 taps x Cout / 64 k tiles) and run on the dgrad chain
  // beside the weight-gradient branch, where a cluster split would take SMs from it
  const int k_tiles = max_taps * (Cout / 64);
  p.M = static_cast<int>(M); p.N = Cin; p.K = k_tiles * BK; p.D = dx; p.ldd = Cin; p.bias = nullptr; p.out_fp32 = 0;
  p.act = 0; p.a_mn = 0; p.b_mn = 1; p.k_tiles_per_split = k_tiles; p.cluster_k = 1; p.atomic_out = 0;
  p.col_stats = nullptr;
  p.tile_flags = nullptr; p.flag_epoch = 0; p.alpha = 1.0f; p.flag_elem_off = 0; p.flag_tile_elems = 0;
  p.ldb = static_cast<long long>(KH) * KW * Cin;
  p.flag_bias_off = -1; p.flag_epoch_ptr = nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  p.conv_ho = Ho; p.conv_wo = Wo; p.conv_stride = 2; p.conv_pad = 0; p.conv_kw = KW; p.conv_cin = Cout;
  p.conv_taps = KH * KW; p.conv_ncol = Cin; p.conv_h = H; p.conv_w = W;
  dim3 grid((Cin + bn - 1) / bn, static_cast<unsigned>(4 * tiles_m), 1);
  if (bn == 128) return launch_fixed<128, 6, 4>(ta, tb, p, grid, stream);
  return launch_fixed<64, 8, 4>(ta, tb, p, grid, stream);
}

// weight gradient: dw[Cout, KH*KW*Cin] (fp32, accumulated with red.add) += dy[N*Ho*Wo, Cout]^T im2col(x)
extern "C" int b200_conv_igemm_wgrad(const void* dy, const void* x, float* dw, int N, int H, int W, int Cin, int Cout,
                                     int KH, int KW, int stride, int pad, int Ho, int Wo, int split_k, int force_bn,
                                     const B200SgdEpilogue* sgd, cudaStream_t stream) {
  using namespace b200;
  const long long Mp = static_cast<long long>(N) * Ho * Wo;      // reduction length (output pixels)
  const int Kc = KH * KW * Cin;                                    // GEMM N
  if (Mp <= 0 || Cout <= 0) return 0;
  if (Cin % 64 != 0 || Cout % 8 != 0 || Mp > (1ll << 30) || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(dy) & 15) || (reinterpret_cast<uintptr_t>(dw) & 15))
    return -2;
  const int bn = clamp_bn(force_bn > 0 ? force_bn : (Kc > 64 ? 128 : 64));
  CUtensorMap ta, tb;
  int rc = make_map(&ta, dy, Mp, Cout, Cout, 64, BK);              // MN-major A: rows = pixels (K), cols = Cout (M)
  if (rc) return rc;
  rc = b200_encode_map_im2col_bf16(&tb, x, N, H, W, Cin, KH, KW, stride, pad, 64, 64);
  if (rc) return rc;
  const int k_tiles = static_cast<int>((Mp + BK - 1) / BK);
  if (split_k < 1) split_k = 1;
  if (split_k > k_tiles) split_k = k_tiles;
  const int per = (k_tiles + split_k - 1) / split_k;
  split_k = (k_tiles + per - 1) / per;
  if (sgd != nullptr && split_k != 1) return B200_SGD_EPILOGUE_DECLINED;
  GemmParams p;
  if (sgd != nullptr) set_sgd_epilogue(p, *sgd);
  p.M = Cout; p.N = Kc; p.K = static_cast<int>(Mp); p.D = dw; p.ldd = Kc; p.bias = nullptr; p.out_fp32 = 1; p.act = 0;
  p.a_mn = 1; p.b_mn = 1; p.k_tiles_per_split = per; p.cluster_k = 1; p.atomic_out = 1;
  p.col_stats = nullptr;
  p.tile_flags = nullptr; p.flag_epoch = 0; p.alpha = 1.0f; p.flag_elem_off = 0; p.flag_tile_elems = 0; p.ldb = Kc;
  p.flag_bias_off = -1; p.flag_epoch_ptr = nullptr;
  p.batched = 0; p.batch_inner = 1; p.batch_count = 1; p.d_outer = 0; p.d_inner = 0;
  p.stages = 4;
  p.conv_ho = Ho; p.conv_wo = Wo; p.conv_stride = stride; p.conv_pad = pad; p.conv_kw = KW; p.conv_cin = Cin;
  p.conv_taps = KH * KW; p.conv_ncol = Cin;
  dim3 grid((Kc + bn - 1) / bn, (Cout + BM - 1) / BM, split_k);
  if (sgd != nullptr) {
    if (bn == 128) return launch_fixed_sgd<128, 6, 2>(ta, tb, p, grid, stream);
    return launch_fixed_sgd<64, 8, 2>(ta, tb, p, grid, stream);
  }
  if (bn == 128) return launch_fixed<128, 6, 2>(ta, tb, p, grid, stream);
  return launch_fixed<64, 8, 2>(ta, tb, p, grid, stream);
}

B200_TRACE_REGISTER(gemm_wgmma)
