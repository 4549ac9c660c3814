// Fused attention (forward here, backward further down) for one (batch, head) per CTA, S = 128 keys/queries, d_head = 64 (BERT-base at
// sequence length 128):   P = softmax(scale * Q K^T)   O = P V
//
//   TMA   Q [128 x 64], K [128 x 64] (K-major operands), V [128 keys x 64] (MN-major B operand) -> smem
//   MMA 1 S = Q K^T            wgmma, two consumer warpgroups x (64 x 128 x 64)  -> fp32 tile in shared memory
//   softmax: one thread per query row reads its row of the staged tile -- row max and row sum need no shuffles:
//            (A) max, (B) exp -> un-normalised bf16 P~ written to shared memory in the 128B-swizzled K-major layout
//            wgmma expects for an A operand, row sum; (C) normalised P to global memory (saved for backward).
//   MMA 2 O~ = P~ V            wgmma, two warpgroups x (64 x 64 x 128)  -> fp32 tile in shared memory
//   epilogue O = O~ / rowsum   -> out[b*S + q, h*64 : h*64+64]
//
// The S x S scores never touch HBM and P is written exactly once (the unfused path writes S, reads S,
// writes P, reads P).  It runs whenever S = 128, d_head = 64 and there is no mask; tests/test_gpu_bert.py checks it
// against the multi-kernel path and an fp32 reference.
//
// PAD: the same tiles for a runtime S < 128 (ViT sequence lengths such as 8 x 8 patches + a class token = 65), no
// mask, no dropout.  The TMA maps carry the tensor dimension S, so query / key / value / dO rows >= S arrive as zeros.
// Key columns >= S are left out of the row max and the row sum and get P~ = 0; no row >= S of out or dqkv is written
// (the next image's tokens live there).  probs is [B*H, S, Sp] with Sp = round_up(S, 8), columns S..Sp-1 written as 0;
// the backward loads its P tile through a 3-D map, so rows >= S and columns >= Sp arrive as zeros and every product
// that reaches a padded row or column multiplies finite values.
#define B200_TU_TAG 4
#include "dropout.cuh"
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"

extern "C" int b200_encode_map4_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     long long inner, long long s_inner, long long outer, long long s_outer,
                                     int box_cols, int box_rows);

namespace b200 {

constexpr int AT_S = 128;      // queries == keys per CTA
constexpr int AT_D = 64;       // head dimension
constexpr int AT_THREADS = 384;                    // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma + softmax
constexpr int AT_CONSUMERS = 256;
constexpr int AT_Q_BYTES = AT_S * AT_D * 2;        // 16 KB, K-major, 128 B rows
constexpr int AT_P_BYTES = AT_S * AT_S * 2;        // 32 KB = two 64-key k-tiles of 16 KB
constexpr int AT_SP = AT_S + 4;                    // fp32 pitch of a staged 128-column tile (skews banks)
constexpr int AT_OP = AT_D + 4;                    // fp32 pitch of a staged 64-column tile
constexpr int AT_WIDE_BYTES = AT_S * AT_SP * 4;
constexpr int AT_NARROW_BYTES = AT_S * AT_OP * 4;

struct AttnParams {
  __nv_bfloat16* out;      // [B*S, D]
  __nv_bfloat16* probs;    // [B*H*S, S]; PAD: [B*H, S, Sp]
  int H, D;                // heads, model width (H * 64)
  float scale_log2e;       // softmax scale * log2(e)
  int S;                   // PAD: sequence length (< 128); probs row pitch Sp = round_up(S, 8)
};

// DROP: dropout on the probabilities.  Pass B zeroes the dropped entries of P~ before MMA 2 and the epilogue scales by
// inv * s; the saved probs stay the undropped P.  Element i of the mask is the index into probs.
template <bool DROP, bool PAD = false>
__global__ void __launch_bounds__(AT_THREADS, 1)
attention_fwd_s128_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const AttnParams p, const DropArgs da) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + AT_Q_BYTES;
  uint8_t* sV = sK + AT_Q_BYTES;
  uint8_t* sP = sV + AT_Q_BYTES;
  float* sS = reinterpret_cast<float*>(sP + AT_P_BYTES);                 // scores, fp32 [128][AT_SP]
  float* sO = reinterpret_cast<float*>(sP + AT_P_BYTES + AT_WIDE_BYTES); // O~, fp32 [128][AT_OP]
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(sP + AT_P_BYTES + AT_WIDE_BYTES + AT_NARROW_BYTES);

  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int bh = blockIdx.x;
  const int b = bh / p.H, h = bh - b * p.H;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(bar_load, 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();

  if (warp == 0) {
    if (elect_one()) {
      mbar_expect_tx(bar_load, 3 * AT_Q_BYTES);
      tma_load_4d(sQ, &tmQ, bar_load, 0, 0, h, b);                 // box [64 d][128 queries]
      tma_load_4d(sK, &tmK, bar_load, 0, 0, h, b);                 // box [64 d][128 keys]
      tma_load_4d(sV, &tmV, bar_load, 0, 0, h, b);                 // box [64 d][64 keys]  (MN-major atom 0)
      tma_load_4d(sV + 8192, &tmV, bar_load, 0, 64, h, b);         // keys 64..127
    }
  } else if (warp >= 4) {
    const int ew = warp - 4, g = ew >> 2;                          // warpgroup g computes query rows 64 g .. 64 g + 63
    mbar_wait(bar_load, 0);
    {
      // MMA 1: S = Q K^T (both K-major)
      float acc[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.f;
      const uint32_t q = smem_u32(sQ) + g * 8192, k = smem_u32(sK);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < AT_D / 16; ++kk)
        wgmma_bf16_n128<0, 0>(acc, gmma_desc_sw128(q + kk * 32, 16, 1024), gmma_desc_sw128(k + kk * 32, 16, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      wg_store_acc<128>(acc, sS, AT_SP, 64 * g);
    }
    named_bar_sync(1, AT_CONSUMERS);
    // softmax: thread == query row (warps 4..7), row max and row sum need no shuffles
    const int lane = static_cast<int>(lane_id());
    const int r = (ew & 3) * 32 + lane;
    const float* srow = sS + r * AT_SP;
    float mb = 0.f, inv = 0.f;
    if (ew < 4) {
      DropCtr dc;
      if constexpr (DROP) dc = drop_ctr(da);
      // pass A: row maximum
      float m = -INFINITY;
#pragma unroll 1
      for (int c = 0; c < AT_S; c += 32) {
        uint32_t x[32];
        acc_ld_row32(srow + c, x);
#pragma unroll
        for (int j = 0; j < 32; ++j) m = fmaxf(m, PAD && c + j >= p.S ? -INFINITY : __uint_as_float(x[j]));
      }
      mb = m * p.scale_log2e;
      // pass B: P~ = exp2(scale*log2e*x - mb) -> bf16 -> swizzled shared memory (K-major A operand); row sum
      float sum = 0.f;
      uint8_t* prow = sP + r * 128;
#pragma unroll 1
      for (int c = 0; c < AT_S; c += 32) {
        uint32_t x[32];
        acc_ld_row32(srow + c, x);
        float e[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          e[j] = PAD && c + j >= p.S ? 0.f : exp2f(fmaf(__uint_as_float(x[j]), p.scale_log2e, -mb));
          sum += e[j];
        }
        if constexpr (DROP) {
          const unsigned long long i0 = (static_cast<unsigned long long>(bh) * AT_S + r) * AT_S + c;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            const uint32_t bits = drop_keep8(dc, i0 + j);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) e[j + jj] = kept(bits, jj, e[j + jj], 1.f);
          }
        }
        uint8_t* tile = prow + (c >> 6) * 16384;                     // 64-key k-tile
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const int chunk = ((c & 63) + j) >> 3;                     // 16-byte chunk inside the 128-byte row
          *reinterpret_cast<uint4*>(tile + ((chunk ^ (r & 7)) << 4)) =
              make_uint4(pack_bf16x2(e[j], e[j + 1]), pack_bf16x2(e[j + 2], e[j + 3]), pack_bf16x2(e[j + 4], e[j + 5]),
                         pack_bf16x2(e[j + 6], e[j + 7]));
        }
      }
      inv = 1.f / sum;
      fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core (async proxy)
    }
    named_bar_sync(1, AT_CONSUMERS);
    {
      // MMA 2: O~ = P~ V   (A = P~ K-major in two 64-key halves, B = V MN-major: d contiguous)
      float acc[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = 0.f;
      const uint32_t pp = smem_u32(sP) + g * 8192, v = smem_u32(sV);
      wgmma_fence();
#pragma unroll
      for (int kt = 0; kt < 2; ++kt)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_bf16_n64<0, 1>(acc, gmma_desc_sw128(pp + kt * 16384 + kk * 32, 16, 1024),
                               gmma_desc_sw128(v + kt * 8192 + kk * 2048, 8192, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      wg_store_acc<64>(acc, sO, AT_OP, 64 * g);
    }
    named_bar_sync(1, AT_CONSUMERS);
    const int S = PAD ? p.S : AT_S, Sp = PAD ? (p.S + 7) & ~7 : AT_S;
    if (ew < 4 && (!PAD || r < S)) {
      // normalised probabilities to global memory (saved for backward)
      __nv_bfloat16* grow = p.probs + (static_cast<size_t>(bh) * S + r) * Sp;
#pragma unroll 1
      for (int c = 0; c < Sp; c += 32) {
        uint32_t x[32];
        acc_ld_row32(srow + c, x);
        float e[32];
#pragma unroll
        for (int j = 0; j < 32; ++j)
          e[j] = PAD && c + j >= S ? 0.f : exp2f(fmaf(__uint_as_float(x[j]), p.scale_log2e, -mb)) * inv;
#pragma unroll
        for (int j = 0; j < 32; j += 8)
          if (!PAD || c + j < Sp)
            *reinterpret_cast<uint4*>(grow + c + j) =
                make_uint4(pack_bf16x2(e[j], e[j + 1]), pack_bf16x2(e[j + 2], e[j + 3]), pack_bf16x2(e[j + 4], e[j + 5]),
                           pack_bf16x2(e[j + 6], e[j + 7]));
      }
      // epilogue: O = O~ / rowsum (times s with dropout)
      if constexpr (DROP) inv *= da.scale;
      __nv_bfloat16* orow = p.out + (static_cast<size_t>(b) * S + r) * p.D + h * AT_D;
#pragma unroll 1
      for (int c = 0; c < AT_D; c += 32) {
        uint32_t x[32];
        acc_ld_row32(sO + r * AT_OP + c, x);
#pragma unroll
        for (int j = 0; j < 32; j += 8)
          *reinterpret_cast<uint4*>(orow + c + j) =
              make_uint4(pack_bf16x2(__uint_as_float(x[j]) * inv, __uint_as_float(x[j + 1]) * inv),
                         pack_bf16x2(__uint_as_float(x[j + 2]) * inv, __uint_as_float(x[j + 3]) * inv),
                         pack_bf16x2(__uint_as_float(x[j + 4]) * inv, __uint_as_float(x[j + 5]) * inv),
                         pack_bf16x2(__uint_as_float(x[j + 6]) * inv, __uint_as_float(x[j + 7]) * inv));
      }
    }
  }
}


// ---- backward, same tiling: one CTA per (batch, head), S = 128, d = 64 ------------------------------------------
//   dV = P^T dO          (A = P^T  MN-major view of the K-major P tile, B = dO MN-major)
//   dP = dO V^T          (A = dO K-major, B = V K-major)
//   dS = P o (dP - rowsum(dP o P))      thread == query row; written IN PLACE over P in shared memory
//   dQ = scale * dS K    (A = dS K-major, B = K MN-major)
//   dK = scale * dS^T Q  (A = dS^T MN-major view of the same tile, B = Q MN-major)
// Every operand tile is a plain [128 rows x 128 B] swizzled block; "K-major" vs "MN-major" is only the descriptor
// (k-step = 32 B inside a row vs 16 rows = 2048 B; the two 64-key halves of P / dS are 16384 B apart).  Each
// consumer warpgroup computes 64 output rows; results are staged in fp32 shared-memory tiles for the row-per-thread
// passes.  The unfused path reads P twice, writes dP, reads it back, writes dS and reads it twice (all S x S, through
// HBM); here P is read once and nothing S x S is written.  It runs wherever the fused forward did.
struct AttnBwdParams {
  __nv_bfloat16* dqkv;     // [B*S, 3*D]
  const __nv_bfloat16* probs;   // [B*H*S, S]: re-read by the row pass of the dropout form
  int H, D;
  float scale;
  int S;                   // PAD: sequence length (< 128)
};

// DROP: with M the mask and s the scale, dV = (P o M s)^T dO, dP = M s o (dO V^T), delta = rowsum(P o dP),
// dS = P o (dP - delta).  Before the first MMAs each row owner turns its row of the P tile into bf16(P o M s) in place
// and keeps its 128 keep bits in registers; the row pass then re-reads the undropped P row from global memory (L2).
template <bool DROP, bool PAD = false>
__global__ void __launch_bounds__(AT_THREADS, 1)
attention_bwd_s128_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                          const __grid_constant__ CUtensorMap tmP, const AttnBwdParams p, const DropArgs da) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + AT_Q_BYTES;
  uint8_t* sV = sK + AT_Q_BYTES;
  uint8_t* sdO = sV + AT_Q_BYTES;
  uint8_t* sP = sdO + AT_Q_BYTES;                   // [2 key halves][128 q x 64 keys]; becomes dS in place
  float* sW = reinterpret_cast<float*>(sP + AT_P_BYTES);                  // dP, later [dQ | dK], fp32 [128][AT_SP]
  float* sN = reinterpret_cast<float*>(sP + AT_P_BYTES + AT_WIDE_BYTES);  // dV, fp32 [128][AT_OP]
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(sP + AT_P_BYTES + AT_WIDE_BYTES + AT_NARROW_BYTES);

  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int bh = blockIdx.x;
  const int b = bh / p.H, h = bh - b * p.H;
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmdO); tma_prefetch_desc(&tmP);
    mbar_init(bar_load, 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();

  if (warp == 0) {
    if (elect_one()) {
      mbar_expect_tx(bar_load, 4 * AT_Q_BYTES + AT_P_BYTES);
      tma_load_4d(sQ, &tmQ, bar_load, 0, 0, h, b);
      tma_load_4d(sK, &tmK, bar_load, 0, 0, h, b);
      tma_load_4d(sV, &tmV, bar_load, 0, 0, h, b);
      tma_load_4d(sdO, &tmdO, bar_load, 0, 0, h, b);
      if constexpr (PAD) {
        tma_load_4d(sP, &tmP, bar_load, 0, 0, bh, 0);                // [B*H][S][Sp] map: rows >= S, keys >= Sp -> 0
        tma_load_4d(sP + 16384, &tmP, bar_load, 64, 0, bh, 0);
      } else {
        tma_load_2d(sP, &tmP, bar_load, 0, bh * AT_S);               // keys 0..63   x 128 query rows
        tma_load_2d(sP + 16384, &tmP, bar_load, 64, bh * AT_S);      // keys 64..127
      }
    }
  } else if (warp >= 4) {
    const int ew = warp - 4, g = ew >> 2;
    const uint32_t q = smem_u32(sQ), k = smem_u32(sK), v = smem_u32(sV), d_o = smem_u32(sdO), pp = smem_u32(sP);
    mbar_wait(bar_load, 0);
    uint32_t keep[AT_S / 32];     // DROP: keep bits of this thread's row (warpgroup 1)
    if constexpr (DROP) {
      if (ew < 4) {
        const DropCtr dc = drop_ctr(da);
        const int rr = (ew & 3) * 32 + static_cast<int>(lane_id());
        const unsigned long long i0 = (static_cast<unsigned long long>(bh) * AT_S + rr) * AT_S;
        uint8_t* prow = sP + rr * 128;
#pragma unroll
        for (int c = 0; c < AT_S; c += 32) {
          uint32_t bits = 0;
#pragma unroll
          for (int j = 0; j < 32; j += 8) bits |= drop_keep8(dc, i0 + c + j) << j;
          keep[c >> 5] = bits;
          uint8_t* tile = prow + (c >> 6) * 16384;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            uint4* slot = reinterpret_cast<uint4*>(tile + (((((c & 63) + j) >> 3) ^ (rr & 7)) << 4));
            float f[8];
            const uint4 pv = *slot;
            const float2 p0 = unpack_bf16x2(pv.x), p1 = unpack_bf16x2(pv.y), p2 = unpack_bf16x2(pv.z), p3 = unpack_bf16x2(pv.w);
            f[0] = p0.x; f[1] = p0.y; f[2] = p1.x; f[3] = p1.y; f[4] = p2.x; f[5] = p2.y; f[6] = p3.x; f[7] = p3.y;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) f[jj] = kept(bits, j + jj, f[jj], da.scale);
            *slot = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                               pack_bf16x2(f[6], f[7]));
          }
        }
        fence_proxy_async();        // the dropped tile (generic-proxy writes) -> visible to the tensor core
      }
      named_bar_sync(1, AT_CONSUMERS);
    }
    {
      // dV[key, d] = sum_q P[q, key] dO[q, d]: both operands MN-major, reduction over the 128 query rows;
      // warpgroup g owns keys 64 g .. 64 g + 63 = the g-th 64-key half of P
      float dv[32], dp[64];
#pragma unroll
      for (int j = 0; j < 32; ++j) dv[j] = 0.f;
#pragma unroll
      for (int j = 0; j < 64; ++j) dp[j] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_bf16_n64<1, 1>(dv, gmma_desc_sw128(pp + g * 16384 + kk * 2048, 16384, 1024),
                             gmma_desc_sw128(d_o + kk * 2048, 8192, 1024), 1u);
      // dP[q, key] = sum_d dO[q, d] V[key, d]: both K-major
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_bf16_n128<0, 0>(dp, gmma_desc_sw128(d_o + g * 8192 + kk * 32, 16, 1024),
                              gmma_desc_sw128(v + kk * 32, 16, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(dv);
      wgmma_fence_operands(dp);
      wg_store_acc<64>(dv, sN, AT_OP, 64 * g);
      wg_store_acc<128>(dp, sW, AT_SP, 64 * g);
    }
    named_bar_sync(1, AT_CONSUMERS);
    const int lane = static_cast<int>(lane_id());
    const int r = (ew & 3) * 32 + lane;                            // query row (dP, dQ) / key row (dV, dK)
    const int S = PAD ? p.S : AT_S;
    __nv_bfloat16* grow = p.dqkv + (static_cast<size_t>(b) * S + r) * (3 * static_cast<size_t>(p.D)) + h * AT_D;
    if (ew < 4) {
      uint8_t* prow = sP + r * 128;
      const float* wrow = sW + r * AT_SP;
      const __nv_bfloat16* gprow = p.probs + (static_cast<size_t>(bh) * AT_S + r) * AT_S;   // DROP: undropped P
      // pass 1: delta = sum_key P[r, key] * dP[r, key]
      float delta = 0.f;
#pragma unroll 1
      for (int c = 0; c < AT_S; c += 32) {
        uint32_t x[32];
        acc_ld_row32(wrow + c, x);
        if constexpr (DROP) {
          const uint32_t kb = c == 0 ? keep[0] : c == 32 ? keep[1] : c == 64 ? keep[2] : keep[3];   // static indices
#pragma unroll
          for (int j = 0; j < 32; ++j) x[j] = __float_as_uint(kept(kb, j, __uint_as_float(x[j]), da.scale));
        }
        const uint8_t* tile = prow + (c >> 6) * 16384;
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const int chunk = ((c & 63) + j) >> 3;
          const uint4 pv = DROP ? *reinterpret_cast<const uint4*>(gprow + c + j)
                                : *reinterpret_cast<const uint4*>(tile + ((chunk ^ (r & 7)) << 4));
          const float2 p0 = unpack_bf16x2(pv.x), p1 = unpack_bf16x2(pv.y), p2 = unpack_bf16x2(pv.z), p3 = unpack_bf16x2(pv.w);
          delta = fmaf(p0.x, __uint_as_float(x[j]), delta);     delta = fmaf(p0.y, __uint_as_float(x[j + 1]), delta);
          delta = fmaf(p1.x, __uint_as_float(x[j + 2]), delta); delta = fmaf(p1.y, __uint_as_float(x[j + 3]), delta);
          delta = fmaf(p2.x, __uint_as_float(x[j + 4]), delta); delta = fmaf(p2.y, __uint_as_float(x[j + 5]), delta);
          delta = fmaf(p3.x, __uint_as_float(x[j + 6]), delta); delta = fmaf(p3.y, __uint_as_float(x[j + 7]), delta);
        }
      }
      // pass 2: dS = P * (dP - delta), bf16, in place over P (this thread owns row r of both halves)
#pragma unroll 1
      for (int c = 0; c < AT_S; c += 32) {
        uint32_t x[32];
        acc_ld_row32(wrow + c, x);
        if constexpr (DROP) {
          const uint32_t kb = c == 0 ? keep[0] : c == 32 ? keep[1] : c == 64 ? keep[2] : keep[3];   // static indices
#pragma unroll
          for (int j = 0; j < 32; ++j) x[j] = __float_as_uint(kept(kb, j, __uint_as_float(x[j]), da.scale));
        }
        uint8_t* tile = prow + (c >> 6) * 16384;
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const int chunk = ((c & 63) + j) >> 3;
          uint4* slot = reinterpret_cast<uint4*>(tile + ((chunk ^ (r & 7)) << 4));
          const uint4 pv = DROP ? *reinterpret_cast<const uint4*>(gprow + c + j) : *slot;
          const float2 p0 = unpack_bf16x2(pv.x), p1 = unpack_bf16x2(pv.y), p2 = unpack_bf16x2(pv.z), p3 = unpack_bf16x2(pv.w);
          *slot = make_uint4(pack_bf16x2(p0.x * (__uint_as_float(x[j]) - delta), p0.y * (__uint_as_float(x[j + 1]) - delta)),
                             pack_bf16x2(p1.x * (__uint_as_float(x[j + 2]) - delta), p1.y * (__uint_as_float(x[j + 3]) - delta)),
                             pack_bf16x2(p2.x * (__uint_as_float(x[j + 4]) - delta), p2.y * (__uint_as_float(x[j + 5]) - delta)),
                             pack_bf16x2(p3.x * (__uint_as_float(x[j + 6]) - delta), p3.y * (__uint_as_float(x[j + 7]) - delta)));
        }
      }
      fence_proxy_async();            // dS (generic-proxy writes) -> visible to the tensor core
    } else if (!PAD || r < S) {
      // dV row r (= key index) is complete: the second warpgroup stores it while the first computes dS
#pragma unroll 1
      for (int c = 0; c < AT_D; c += 32) {
        uint32_t x[32];
        acc_ld_row32(sN + r * AT_OP + c, x);
#pragma unroll
        for (int j = 0; j < 32; j += 8)
          *reinterpret_cast<uint4*>(grow + 2 * p.D + c + j) =
              make_uint4(pack_bf16x2(__uint_as_float(x[j]), __uint_as_float(x[j + 1])),
                         pack_bf16x2(__uint_as_float(x[j + 2]), __uint_as_float(x[j + 3])),
                         pack_bf16x2(__uint_as_float(x[j + 4]), __uint_as_float(x[j + 5])),
                         pack_bf16x2(__uint_as_float(x[j + 6]), __uint_as_float(x[j + 7])));
      }
    }
    named_bar_sync(1, AT_CONSUMERS);
    {
      // dQ[q, d] = sum_key dS[q, key] K[key, d]: A K-major (two 64-key halves), B = K MN-major
      // dK[key, d] = sum_q dS[q, key] Q[q, d]: A = dS^T (MN-major view, key half g), B = Q MN-major
      float dq[32], dk[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) { dq[j] = 0.f; dk[j] = 0.f; }
      wgmma_fence();
#pragma unroll
      for (int kt = 0; kt < 2; ++kt)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_bf16_n64<0, 1>(dq, gmma_desc_sw128(pp + kt * 16384 + g * 8192 + kk * 32, 16, 1024),
                               gmma_desc_sw128(k + (kt * 4 + kk) * 2048, 8192, 1024), 1u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_bf16_n64<1, 1>(dk, gmma_desc_sw128(pp + g * 16384 + kk * 2048, 16384, 1024),
                             gmma_desc_sw128(q + kk * 2048, 8192, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(dq);
      wgmma_fence_operands(dk);
      wg_store_acc<64>(dq, sW, AT_SP, 64 * g);          // dP is consumed: columns [0,64) dQ, [64,128) dK
      wg_store_acc<64>(dk, sW + AT_D, AT_SP, 64 * g);
    }
    named_bar_sync(1, AT_CONSUMERS);
    // dQ row r (query) from columns [0,64), dK row r (key) from columns [64,128), both scaled by the softmax scale;
    // the two warpgroups take one half each
    const int c = (ew < 4 ? 0 : AT_D);
#pragma unroll 1
    for (int cc = c; cc < (PAD && r >= S ? c : c + AT_D); cc += 32) {
      uint32_t x[32];
      acc_ld_row32(sW + r * AT_SP + cc, x);
      __nv_bfloat16* dst = grow + (cc < AT_D ? cc : p.D + (cc - AT_D));
#pragma unroll
      for (int j = 0; j < 32; j += 8)
        *reinterpret_cast<uint4*>(dst + j) =
            make_uint4(pack_bf16x2(__uint_as_float(x[j]) * p.scale, __uint_as_float(x[j + 1]) * p.scale),
                       pack_bf16x2(__uint_as_float(x[j + 2]) * p.scale, __uint_as_float(x[j + 3]) * p.scale),
                       pack_bf16x2(__uint_as_float(x[j + 4]) * p.scale, __uint_as_float(x[j + 5]) * p.scale),
                       pack_bf16x2(__uint_as_float(x[j + 6]) * p.scale, __uint_as_float(x[j + 7]) * p.scale));
    }
  }
}

}  // namespace b200

using namespace b200;

// qkv: packed [B*S, 3*H*64] bf16; out [B*S, H*64]; probs [B*H*S, S] (PAD: [B*H, S, round_up(S, 8)]).  Returns -2
// for unsupported shapes.
template <bool DROP, bool PAD = false>
static int attention_fwd_launch(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                                const DropArgs& da, cudaStream_t stream) {
  if (B <= 0) return 0;
  if ((PAD ? S <= 0 || S >= AT_S : S != AT_S) || dh != AT_D) return -2;
  const long long D = static_cast<long long>(H) * dh;
  if ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(probs)) & 15) return -2;
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(qkv);
  CUtensorMap tq, tk, tv;
  int rc = b200_encode_map4_bf16(&tq, base, S, dh, 3 * D, H, dh, B, static_cast<long long>(S) * 3 * D, 64, 128);
  if (rc == 0) rc = b200_encode_map4_bf16(&tk, base + D, S, dh, 3 * D, H, dh, B, static_cast<long long>(S) * 3 * D, 64, 128);
  if (rc == 0) rc = b200_encode_map4_bf16(&tv, base + 2 * D, S, dh, 3 * D, H, dh, B, static_cast<long long>(S) * 3 * D, 64, 64);
  if (rc) return rc;
  AttnParams p;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.probs = reinterpret_cast<__nv_bfloat16*>(probs);
  p.H = H;
  p.D = static_cast<int>(D);
  p.scale_log2e = scale * 1.4426950408889634f;
  p.S = S;
  constexpr int smem = 3 * AT_Q_BYTES + AT_P_BYTES + AT_WIDE_BYTES + AT_NARROW_BYTES + 8 + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(attention_fwd_s128_kernel<DROP, PAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  cudaError_t le = launch_pdl(attention_fwd_s128_kernel<DROP, PAD>, dim3(static_cast<unsigned>(B) * H), AT_THREADS, smem,
                              stream, tq, tk, tv, p, da);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_encode_map2_bf16(void* map, const void* base, long long rows, long long cols, long long ld,
                                     int box_cols, int box_rows);

// qkv [B*S, 3D], dout [B*S, D], probs [B*H*S, S] (PAD: [B*H, S, round_up(S, 8)]; saved by the forward) -> dqkv [B*S, 3D]
template <bool DROP, bool PAD = false>
static int attention_bwd_launch(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S, int H,
                                int dh, float scale, const DropArgs& da, cudaStream_t stream) {
  if (B <= 0) return 0;
  if ((PAD ? S <= 0 || S >= AT_S : S != AT_S) || dh != AT_D) return -2;
  const long long D = static_cast<long long>(H) * dh;
  if ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(probs) |
       reinterpret_cast<uintptr_t>(dqkv)) & 15)
    return -2;
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(qkv);
  CUtensorMap tq, tk, tv, tdo, tp;
  const long long so = static_cast<long long>(S) * 3 * D;
  int rc = b200_encode_map4_bf16(&tq, base, S, dh, 3 * D, H, dh, B, so, 64, 128);
  if (rc == 0) rc = b200_encode_map4_bf16(&tk, base + D, S, dh, 3 * D, H, dh, B, so, 64, 128);
  if (rc == 0) rc = b200_encode_map4_bf16(&tv, base + 2 * D, S, dh, 3 * D, H, dh, B, so, 64, 128);
  if (rc == 0) rc = b200_encode_map4_bf16(&tdo, dout, S, dh, D, H, dh, B, static_cast<long long>(S) * D, 64, 128);
  if (PAD) {
    const long long sp = (S + 7) & ~7, bh = static_cast<long long>(B) * H;
    if (rc == 0) rc = b200_encode_map4_bf16(&tp, probs, S, sp, sp, bh, S * sp, 1, bh * S * sp, 64, 128);
  } else if (rc == 0) {
    rc = b200_encode_map2_bf16(&tp, probs, static_cast<long long>(B) * H * S, S, S, 64, 128);
  }
  if (rc) return rc;
  AttnBwdParams p;
  p.dqkv = reinterpret_cast<__nv_bfloat16*>(dqkv);
  p.probs = reinterpret_cast<const __nv_bfloat16*>(probs);
  p.H = H;
  p.D = static_cast<int>(D);
  p.scale = scale;
  p.S = S;
  constexpr int smem = 4 * AT_Q_BYTES + AT_P_BYTES + AT_WIDE_BYTES + AT_NARROW_BYTES + 8 + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_s128_kernel<DROP, PAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  cudaError_t le = launch_pdl(attention_bwd_s128_kernel<DROP, PAD>, dim3(static_cast<unsigned>(B) * H), AT_THREADS, smem,
                              stream, tq, tk, tv, tdo, tp, p, da);
  if (le != cudaSuccess) return static_cast<int>(le);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_attention_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                                  cudaStream_t stream) {
  return attention_fwd_launch<false>(qkv, out, probs, B, S, H, dh, scale, DropArgs{}, stream);
}
extern "C" int b200_attention_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S, int H,
                                  int dh, float scale, cudaStream_t stream) {
  return attention_bwd_launch<false>(qkv, dout, probs, dqkv, B, S, H, dh, scale, DropArgs{}, stream);
}

extern "C" int b200_attention_drop_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                                       const B200Dropout* drop, cudaStream_t stream) {
  return attention_fwd_launch<true>(qkv, out, probs, B, S, H, dh, scale, drop_args(drop), stream);
}
extern "C" int b200_attention_drop_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S,
                                       int H, int dh, float scale, const B200Dropout* drop, cudaStream_t stream) {
  return attention_bwd_launch<true>(qkv, dout, probs, dqkv, B, S, H, dh, scale, drop_args(drop), stream);
}

// S < 128 (not a multiple of 8 in practice: other lengths take the multi-kernel path), d_head = 64, no mask, no dropout
extern "C" int b200_attention_short_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                                        cudaStream_t stream) {
  return attention_fwd_launch<false, true>(qkv, out, probs, B, S, H, dh, scale, DropArgs{}, stream);
}
extern "C" int b200_attention_short_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S,
                                        int H, int dh, float scale, cudaStream_t stream) {
  return attention_bwd_launch<false, true>(qkv, dout, probs, dqkv, B, S, H, dh, scale, DropArgs{}, stream);
}

B200_TRACE_REGISTER(attention)
