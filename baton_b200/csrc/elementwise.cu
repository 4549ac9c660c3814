// HBM-bound elementwise / reduction kernels over flat buffers: fused arena SGD (K4), multi-source
// weighted sum (manager-side FedAvg, K1 fallback), casts, batch row gather (K8), column sums
// (bias gradients), ReLU / GELU pieces.  All use 16-byte vectors and grid-stride loops sized to
// the device's SMs x a few resident CTAs.
#define B200_TU_TAG 8
#include <cuda_fp16.h>

#include "dp.cuh"
#include "launch.h"
#include "pdl.cuh"
#include "ptx.cuh"
#include "rows.cuh"
#include "sgd.cuh"

namespace b200 {

constexpr int EW_THREADS = 256;
static inline int ew_grid(long long n_vec, int max_ctas = device_sm_count() * 8) {
  long long g = (n_vec + EW_THREADS - 1) / EW_THREADS;
  if (g < 1) g = 1;
  if (g > max_ctas) g = max_ctas;
  return static_cast<int>(g);
}

// fp32 product and sum rounded to nearest, each on its own and without flushing subnormals (the build's fast-math flag
// turns __fmul_rn / __fadd_rn into their .ftz forms; torch on the host keeps subnormals)
__device__ __forceinline__ float mul_rn(float a, float b) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float add_rn(float a, float b) {
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float rcp_rn(float a) {
  float r;
  asm("rcp.rn.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}

// ------------------------------------------------------------------ fused SGD over the arena
// One pass over {w, g, m}: the update of sgd.cuh ; g = 0 (so split-K wgrad GEMMs can red.add into it next step) ;
// bf16 shadow = bf16(w).
// K4 "emit the upload copy" (SURVEY 2.6): the LAST step of a local epoch can also write this client's wire copy for the
// round-end collective -- bf16 / fp32 of (w_new - global) * scale -- while w_new is still in registers, so the
// collective's own pack phase (one more read of theta + global, ~10 B / element) disappears.  The wire address is
// read from a device word (`wire_slot`): the collective double-buffers its wire by round parity and the captured
// epoch graph must follow without being re-captured.  Elements [n, n_pack) are float BUFFERS (BatchNorm running
// statistics): not optimised, only packed.
struct SgdPack {
  const unsigned long long* wire_slot;   // device word holding the wire base address, or nullptr = no pack
  const float* global_w;                 // delta upload: wire = w - global_w; nullptr: wire = w
  const float* scale;                    // device scalar multiplied into the wire value (NVLS: n_k; P2P: 1)
  long long n_pack;                      // elements to pack (>= n)
  int wire_fp32;                         // 0: bf16 wire, 1: fp32 wire
};

// The upload copy of one 4-element group of new weights (SgdPack; `i` indexes float4 groups)
__device__ __forceinline__ void sgd_pack4(const SgdPack& pk, uint8_t* wire, float pscale, long long i, float4 d) {
  if (pk.global_w != nullptr) {
    const float4 gl = reinterpret_cast<const float4*>(pk.global_w)[i];
    d.x -= gl.x; d.y -= gl.y; d.z -= gl.z; d.w -= gl.w;
  }
  d.x *= pscale; d.y *= pscale; d.z *= pscale; d.w *= pscale;
  if (pk.wire_fp32) reinterpret_cast<float4*>(wire)[i] = d;
  else reinterpret_cast<uint2*>(wire)[i] = make_uint2(pack_bf16x2(d.x, d.y), pack_bf16x2(d.z, d.w));
}

// The gradient of a clipped step, g' = fl32(g * coef) (clip_grad_norm_ multiplies even when coef is 1)
__device__ __forceinline__ float4 clip4(float4 g, float c) {
  return make_float4(mul_rn(g.x, c), mul_rn(g.y, c), mul_rn(g.z, c), mul_rn(g.w, c));
}
// The clip coefficient, written by the norm kernel this kernel waits on (programmatic dependent launch).  A plain load
// through the `const __restrict__` hyper pointer may be issued as a read-only load ahead of griddep_wait(); this one
// cannot move across it.
__device__ __forceinline__ float load_clip_coef(const float* p) {
  float r;
  asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(r) : "l"(p) : "memory");
  return r;
}
// float4 group i of the gradient, clipped when CLIP
template <bool CLIP>
__device__ __forceinline__ float4 load_grad4(float* g, long long i, float coef) {
  if constexpr (CLIP) return clip4(reinterpret_cast<float4*>(g)[i], coef);
  return reinterpret_cast<float4*>(g)[i];
}

// Body of the AdamW form of fused_sgd_kernel: the same passes (update + gradient zeroing + bf16 shadow + upload copy,
// then the pack-only float buffers, then the scalar tail) with adamw_update in place of the SGD step.  CLIP: the
// gradient is multiplied by `coef` as it is loaded.
template <bool CLIP>
__device__ __forceinline__ void adamw_arena(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, __nv_bfloat16* __restrict__ wb, long long n,
                                            const AdamHyper h, float coef, int zero_grad, const SgdPack& pk) {
  const long long nv = n >> 2;
  uint8_t* wire = nullptr;
  float pscale = 1.f;
  if (pk.wire_slot != nullptr) {
    wire = reinterpret_cast<uint8_t*>(*pk.wire_slot);
    if (pk.scale != nullptr) pscale = *pk.scale;
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv; i += stride) {
    float4 mv = reinterpret_cast<const float4*>(m)[i], vv = reinterpret_cast<const float4*>(v)[i];
    const float4 wv = adamw_update4(h, reinterpret_cast<const float4*>(w)[i], load_grad4<CLIP>(g, i, coef), mv, vv);
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    reinterpret_cast<float4*>(w)[i] = wv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (wb != nullptr) reinterpret_cast<uint2*>(wb)[i] = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    if (wire != nullptr) sgd_pack4(pk, wire, pscale, i, wv);
  }
  if (wire != nullptr) {      // float buffers behind the parameters: pack only (n and n_pack are multiples of 8)
    for (long long i = nv + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < (pk.n_pack >> 2);
         i += stride)
      sgd_pack4(pk, wire, pscale, i, reinterpret_cast<const float4*>(w)[i]);
  }
  if (blockIdx.x == 0) {
    for (long long i = (nv << 2) + threadIdx.x; i < n; i += blockDim.x) {
      const float wv = adamw_update(h, w[i], CLIP ? mul_rn(g[i], coef) : g[i], m[i], v[i]);
      w[i] = wv;
      if (zero_grad) g[i] = 0.f;
      if (wb != nullptr) wb[i] = __float2bfloat16_rn(wv);
    }
  }
}

// PROX: FedProx step toward the anchor `aux` (indexed like w).  SCAF: SCAFFOLD step, `aux` is the correction c - c_i
// (indexed like w).  The two are exclusive; with neither, `aux` is not read.  One pointer serves both so the plain and
// FedProx instantiations keep their parameter list.
// ADAM: the AdamW step of sgd.cuh instead of SGD.  `hyper` is then the step's AdamW row (ADAMW_ROW floats), `mom` the
// first moment m and `aux` the second moment v, which this form also writes (each element is read once, by the thread
// that writes it); `nesterov` is not read.
// CLIP: gradient-norm clipping -- g is multiplied by the coefficient hyper[SGD_HYPER_CLIP] (AdamW: row[ADAMW_ROW_CLIP])
// as it is loaded, before any other term; everything else is the unclipped form's.
template <bool PROX, bool SCAF = false, bool ADAM = false, bool CLIP = false>
__global__ void __launch_bounds__(EW_THREADS)
fused_sgd_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ mom,
                 __nv_bfloat16* __restrict__ wb, long long n, const float* __restrict__ hyper, int zero_grad,
                 int nesterov, const SgdPack pk, const float* __restrict__ aux) {
  static_assert(!(PROX && SCAF), "FedProx and SCAFFOLD are exclusive");
  static_assert(!(ADAM && (PROX || SCAF)), "AdamW takes neither the FedProx nor the SCAFFOLD term");
  griddep_launch_dependents();
  griddep_wait();
  if constexpr (ADAM) {
    adamw_arena<CLIP>(w, g, mom, const_cast<float*>(aux), wb, n, load_adam_hyper(hyper),
                      CLIP ? load_clip_coef(hyper + ADAMW_ROW_CLIP) : 1.f, zero_grad, pk);
    return;
  }
  const SgdHyper h = PROX ? load_sgd_hyper_prox(hyper) : load_sgd_hyper(hyper);
  const float coef = CLIP ? load_clip_coef(hyper + SGD_HYPER_CLIP) : 1.f;
  const long long nv = n >> 2;
  uint8_t* wire = nullptr;
  float pscale = 1.f;
  if (pk.wire_slot != nullptr) {
    wire = reinterpret_cast<uint8_t*>(*pk.wire_slot);
    if (pk.scale != nullptr) pscale = *pk.scale;
  }
  // delta upload of a FedProx step: the anchor IS the global copy the wire value is taken against -- read it once
  const bool anchor_is_global = PROX && aux == pk.global_w;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 mv = mom != nullptr ? reinterpret_cast<float4*>(mom)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 wv;
    if constexpr (PROX) {
      av = reinterpret_cast<const float4*>(aux)[i];
      wv = sgd_update4_prox(h, reinterpret_cast<float4*>(w)[i], load_grad4<CLIP>(g, i, coef), av, mv,
                            mom != nullptr, nesterov);
    } else if constexpr (SCAF) {
      wv = sgd_update4_scaf(h, reinterpret_cast<float4*>(w)[i], load_grad4<CLIP>(g, i, coef),
                            reinterpret_cast<const float4*>(aux)[i], mv, mom != nullptr, nesterov);
    } else {
      wv = sgd_update4(h, reinterpret_cast<float4*>(w)[i], load_grad4<CLIP>(g, i, coef), mv, mom != nullptr,
                       nesterov);
    }
    if (mom != nullptr) reinterpret_cast<float4*>(mom)[i] = mv;
    reinterpret_cast<float4*>(w)[i] = wv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (wb != nullptr) reinterpret_cast<uint2*>(wb)[i] = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    if (wire != nullptr) {
      float4 d = wv;
      if (pk.global_w != nullptr) {
        const float4 gl = anchor_is_global ? av : reinterpret_cast<const float4*>(pk.global_w)[i];
        d.x -= gl.x; d.y -= gl.y; d.z -= gl.z; d.w -= gl.w;
      }
      d.x *= pscale; d.y *= pscale; d.z *= pscale; d.w *= pscale;
      if (pk.wire_fp32) reinterpret_cast<float4*>(wire)[i] = d;
      else reinterpret_cast<uint2*>(wire)[i] = make_uint2(pack_bf16x2(d.x, d.y), pack_bf16x2(d.z, d.w));
    }
  }
  if (wire != nullptr) {      // float buffers behind the parameters: pack only (n and n_pack are multiples of 8)
    const long long npv = pk.n_pack >> 2;
    for (long long i = nv + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < npv;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      float4 d = reinterpret_cast<const float4*>(w)[i];
      if (pk.global_w != nullptr) {
        const float4 gl = reinterpret_cast<const float4*>(pk.global_w)[i];
        d.x -= gl.x; d.y -= gl.y; d.z -= gl.z; d.w -= gl.w;
      }
      d.x *= pscale; d.y *= pscale; d.z *= pscale; d.w *= pscale;
      if (pk.wire_fp32) reinterpret_cast<float4*>(wire)[i] = d;
      else reinterpret_cast<uint2*>(wire)[i] = make_uint2(pack_bf16x2(d.x, d.y), pack_bf16x2(d.z, d.w));
    }
  }
  // scalar tail (n is normally padded to a multiple of 4 by the arena)
  if (blockIdx.x == 0) {
    for (long long i = (nv << 2) + threadIdx.x; i < n; i += blockDim.x) {
      float mv = mom != nullptr ? mom[i] : 0.f;
      const float wv = PROX ? sgd_update_prox(h, w[i], CLIP ? mul_rn(g[i], coef) : g[i], aux[i], mv, mom != nullptr,
                                              nesterov)
                       : SCAF ? sgd_update_scaf(h, w[i], CLIP ? mul_rn(g[i], coef) : g[i], aux[i], mv, mom != nullptr,
                                                nesterov)
                              : sgd_update(h, w[i], CLIP ? mul_rn(g[i], coef) : g[i], mv, mom != nullptr, nesterov);
      if (mom != nullptr) mom[i] = mv;
      w[i] = wv;
      if (zero_grad) g[i] = 0.f;
      if (wb != nullptr) wb[i] = __float2bfloat16_rn(wv);
    }
  }
}

__device__ __forceinline__ bool same_bits4(float4 a, float4 b) {
  return __float_as_uint(a.x) == __float_as_uint(b.x) && __float_as_uint(a.y) == __float_as_uint(b.y) &&
         __float_as_uint(a.z) == __float_as_uint(b.z) && __float_as_uint(a.w) == __float_as_uint(b.w);
}

// Body of the AdamW form of fused_sgd_segments_kernel.  A kind-1 element has g = 0 at every step, so its m and v are
// 0 from the first step of a run on (the first step ignores what is stored), and its step is w *= (1 - lr*wd): the
// identity exactly when that factor rounds to 1, i.e. with weight decay 0.  Kind-1 chunks are then skipped -- except
// at the first step, where they are processed once so that their stored m and v really are 0 for the whole-arena
// steps of the run (the momentum buffer may hold an earlier SGD run's momentum).  The skip is decided from the step
// row in device memory, so a captured epoch stays exact.  Kind-1 weights are stored only where their bits change.
// CLIP: kind-0 gradients are multiplied by `coef` as they are loaded.
template <bool CLIP>
__device__ __forceinline__ void adamw_segments(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m,
                                               float* __restrict__ v, __nv_bfloat16* __restrict__ wb,
                                               const long long* __restrict__ seg, int n_seg, const AdamHyper h,
                                               float coef) {
  const bool nograd_is_identity = h.decay == 1.f && !h.first;
  for (int s = blockIdx.x; s < n_seg; s += gridDim.x) {
    const long long off = seg[3 * s], len = seg[3 * s + 1];
    const bool has_grad = seg[3 * s + 2] == 0;
    if (!has_grad && nograd_is_identity) continue;      // block-uniform
    long long done = 0;
    if ((off & 3) == 0) {
      const long long nv = len >> 2;
      for (long long i = threadIdx.x; i < nv; i += blockDim.x) {
        const long long e = off + (i << 2);
        float4 mv = *reinterpret_cast<const float4*>(m + e), vv = *reinterpret_cast<const float4*>(v + e);
        float4 gv = has_grad ? *reinterpret_cast<const float4*>(g + e) : make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (CLIP) gv = has_grad ? clip4(gv, coef) : gv;
        const float4 w0 = *reinterpret_cast<const float4*>(w + e);
        const float4 wv = adamw_update4(h, w0, gv, mv, vv);
        *reinterpret_cast<float4*>(m + e) = mv;
        *reinterpret_cast<float4*>(v + e) = vv;
        if (!has_grad && same_bits4(w0, wv)) continue;
        *reinterpret_cast<float4*>(w + e) = wv;
        if (has_grad) *reinterpret_cast<float4*>(g + e) = make_float4(0.f, 0.f, 0.f, 0.f);
        if (wb != nullptr) *reinterpret_cast<uint2*>(wb + e) = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
      }
      done = nv << 2;
    }
    for (long long i = done + threadIdx.x; i < len; i += blockDim.x) {
      const long long e = off + i;
      const float w0 = w[e];
      const float wv = adamw_update(h, w0, has_grad ? (CLIP ? mul_rn(g[e], coef) : g[e]) : 0.f, m[e], v[e]);
      if (!has_grad && __float_as_uint(w0) == __float_as_uint(wv)) continue;
      w[e] = wv;
      if (has_grad) g[e] = 0.f;
      if (wb != nullptr) wb[e] = __float2bfloat16_rn(wv);
    }
  }
}

// ------------------------------------------------------------------ leftover SGD of a step with an optimizer epilogue
// When the weight-gradient GEMMs of a step applied SGD in their epilogue (gemm_wgmma.cu), what is left is a set of
// arena ranges, given as a device table of chunks {offset, length, kind} -- one chunk per CTA iteration.
//   kind 0: parameters with a gradient -- the update of fused_sgd_kernel, gradient zeroed afterwards;
//   kind 1: parameters whose gradient is identically zero (the off-centre taps of a k x k convolution on a 1x1 map) --
//           the update with g = 0, gradient never read.  With weight decay 0, no momentum buffer and no proximal term
//           that update is the identity, and the chunk is skipped; this is decided here from `hyper`, so a captured
//           graph stays exact when it is replayed with new hyper-parameters.
// With an anchor (FedProx) a kind-1 element moves only by prox*(w - a) [+ wd*w]: without a momentum buffer it is stored
// only where its bits change.  In engine rounds these taps equal the global model all round, so nothing is written.
// SCAF (`aux` = the correction c - c_i, as in fused_sgd_kernel): a kind-1 element moves by -lr * (corr [+ wd*w]), so
// kind-1 chunks are never skipped; they use the same sparse store (a zero correction writes nothing).
// ADAM (`hyper` = the AdamW step row, `mom` = m, `aux` = v, as in fused_sgd_kernel): see adamw_segments.
// CLIP (as in fused_sgd_kernel): kind-0 gradients are multiplied by the clip coefficient as they are loaded; a kind-1
// gradient is 0 and stays 0, so kind-1 chunks are skipped (or not) exactly as without clipping.
template <bool PROX, bool SCAF = false, bool ADAM = false, bool CLIP = false>
__global__ void __launch_bounds__(EW_THREADS)
fused_sgd_segments_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ mom,
                          __nv_bfloat16* __restrict__ wb, const long long* __restrict__ seg, int n_seg,
                          const float* __restrict__ hyper, int nesterov, const float* __restrict__ aux) {
  static_assert(!(PROX && SCAF), "FedProx and SCAFFOLD are exclusive");
  static_assert(!(ADAM && (PROX || SCAF)), "AdamW takes neither the FedProx nor the SCAFFOLD term");
  griddep_launch_dependents();
  griddep_wait();
  if constexpr (ADAM) {
    adamw_segments<CLIP>(w, g, mom, const_cast<float*>(aux), wb, seg, n_seg, load_adam_hyper(hyper),
                         CLIP ? load_clip_coef(hyper + ADAMW_ROW_CLIP) : 1.f);
    return;
  }
  const SgdHyper h = PROX ? load_sgd_hyper_prox(hyper) : load_sgd_hyper(hyper);
  const float coef = CLIP ? load_clip_coef(hyper + SGD_HYPER_CLIP) : 1.f;
  const bool has_mom = mom != nullptr;
  const bool nograd_is_identity = !SCAF && h.prox == 0.f && h.wd == 0.f && !has_mom;
  for (int s = blockIdx.x; s < n_seg; s += gridDim.x) {
    const long long off = seg[3 * s], len = seg[3 * s + 1];
    const bool has_grad = seg[3 * s + 2] == 0;
    if (!has_grad && nograd_is_identity) continue;      // block-uniform
    const bool sparse_store = (PROX || SCAF) && !has_grad && !has_mom;
    long long done = 0;
    if ((off & 3) == 0) {
      const long long nv = len >> 2;
      for (long long i = threadIdx.x; i < nv; i += blockDim.x) {
        const long long e = off + (i << 2);
        float4 mv = has_mom ? *reinterpret_cast<float4*>(mom + e) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 gv = has_grad ? *reinterpret_cast<float4*>(g + e) : make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (CLIP) gv = has_grad ? clip4(gv, coef) : gv;
        const float4 w0 = *reinterpret_cast<float4*>(w + e);
        const float4 wv = PROX ? sgd_update4_prox(h, w0, gv, *reinterpret_cast<const float4*>(aux + e), mv, has_mom,
                                                  nesterov)
                          : SCAF ? sgd_update4_scaf(h, w0, gv, *reinterpret_cast<const float4*>(aux + e), mv, has_mom,
                                                    nesterov)
                                 : sgd_update4(h, w0, gv, mv, has_mom, nesterov);
        if (has_mom) *reinterpret_cast<float4*>(mom + e) = mv;
        if (sparse_store && same_bits4(w0, wv)) continue;
        *reinterpret_cast<float4*>(w + e) = wv;
        if (has_grad) *reinterpret_cast<float4*>(g + e) = make_float4(0.f, 0.f, 0.f, 0.f);
        if (wb != nullptr) *reinterpret_cast<uint2*>(wb + e) = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
      }
      done = nv << 2;
    }
    for (long long i = done + threadIdx.x; i < len; i += blockDim.x) {
      const long long e = off + i;
      float mv = has_mom ? mom[e] : 0.f;
      const float gv = has_grad ? (CLIP ? mul_rn(g[e], coef) : g[e]) : 0.f;
      const float w0 = w[e];
      const float wv = PROX ? sgd_update_prox(h, w0, gv, aux[e], mv, has_mom, nesterov)
                       : SCAF ? sgd_update_scaf(h, w0, gv, aux[e], mv, has_mom, nesterov)
                              : sgd_update(h, w0, gv, mv, has_mom, nesterov);
      if (has_mom) mom[e] = mv;
      if (sparse_store && __float_as_uint(w0) == __float_as_uint(wv)) continue;
      w[e] = wv;
      if (has_grad) g[e] = 0.f;
      if (wb != nullptr) wb[e] = __float2bfloat16_rn(wv);
    }
  }
}

// ------------------------------------------------------------------ gradient-norm clipping (clip_grad_norm_)
// norm = ||g[0, n)|| over a FIXED grid of B200_GRAD_NORM_BLOCKS CTAs (independent of the SM count): squares and sums in
// fp64, one fp64 partial per CTA in work[0, B), and the last CTA to arrive (counter work[B], reset by it) sums them in
// index order -- dp_clip_factor_kernel's pattern, so the norm is a pure function of the gradient's values and n, graph
// or eager.  work[B + 1] keeps the fp64 sum of squares.  Then, as torch computes it from its fp32 norm,
//     coef = clamp(fl32(fl32(1 / fl32(norm + 1e-6)) * max_norm), max = 1)
// with IEEE-rounded, non-flushing operations (a NaN norm gives NaN, an infinite one 0).  `max_norm` is read from device
// memory so a captured step follows a new threshold; norm and coef are written to device memory.
constexpr int GRAD_NORM_THREADS = 256;
__device__ __forceinline__ double add_squares4(float4 a, double d) {
  const double x = a.x, y = a.y, z = a.z, w = a.w;
  return fma(w, w, fma(z, z, fma(y, y, fma(x, x, d))));
}
__global__ void __launch_bounds__(GRAD_NORM_THREADS)
grad_norm_clip_kernel(const float* __restrict__ g, long long n, const float* __restrict__ max_norm,
                      unsigned long long* __restrict__ work, float* __restrict__ norm_out, float* __restrict__ coef_out) {
  __shared__ double red[GRAD_NORM_THREADS / 32];
  __shared__ bool last;
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  const long long stride = static_cast<long long>(B200_GRAD_NORM_BLOCKS) * GRAD_NORM_THREADS;
  double d0 = 0.0, d1 = 0.0;        // two loads in flight per thread
  long long i = blockIdx.x * static_cast<long long>(GRAD_NORM_THREADS) + threadIdx.x;
  for (; i + stride < nv; i += 2 * stride) {
    const float4 a = reinterpret_cast<const float4*>(g)[i], b = reinterpret_cast<const float4*>(g)[i + stride];
    d0 = add_squares4(a, d0);
    d1 = add_squares4(b, d1);
  }
  if (i < nv) d0 = add_squares4(reinterpret_cast<const float4*>(g)[i], d0);
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {     // scalar tail
    const double t = g[(nv << 2) + threadIdx.x];
    d1 = fma(t, t, d1);
  }
  double d = d0 + d1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < GRAD_NORM_THREADS / 32; ++w) b += red[w];
    reinterpret_cast<double*>(work)[blockIdx.x] = b;
    __threadfence();
    last = atomicAdd(work + B200_GRAD_NORM_BLOCKS, 1ull) == B200_GRAD_NORM_BLOCKS - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double sq = 0.0;
  for (int b = 0; b < B200_GRAD_NORM_BLOCKS; ++b) sq += reinterpret_cast<const volatile double*>(work)[b];
  work[B200_GRAD_NORM_BLOCKS] = 0ull;
  reinterpret_cast<double*>(work)[B200_GRAD_NORM_BLOCKS + 1] = sq;
  const float norm = static_cast<float>(sqrt(sq));
  const float c = mul_rn(rcp_rn(add_rn(norm, 1e-6f)), *max_norm);
  norm_out[0] = norm;
  coef_out[0] = c > 1.f ? 1.f : c;
}

// ------------------------------------------------------------------ logical-client fold (time-sliced clients on one GPU)
// One pass per co-resident logical client:  acc (+)= n_k * (theta - global)   and, if another client follows on this GPU,
// reset the replica to the global model (theta = global, bf16 shadow, momentum = 0).  mode: 0 = accumulate, 1 = first
// client (acc = ...), 2 = finish: theta = global + acc / total (no accumulate; `nk` carries 1 / total).
__global__ void __launch_bounds__(EW_THREADS)
fold_client_kernel(float* __restrict__ acc, float* __restrict__ theta, const float* __restrict__ global_w,
                   __nv_bfloat16* __restrict__ wb, float* __restrict__ mom, long long n_mom, long long n, float nk,
                   int mode, int reset) {
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 g = reinterpret_cast<const float4*>(global_w)[i];
    if (mode == 2) {
      const float4 a = reinterpret_cast<const float4*>(acc)[i];
      reinterpret_cast<float4*>(theta)[i] = make_float4(fmaf(a.x, nk, g.x), fmaf(a.y, nk, g.y), fmaf(a.z, nk, g.z),
                                                        fmaf(a.w, nk, g.w));
      continue;
    }
    const float4 t = reinterpret_cast<const float4*>(theta)[i];
    float4 a = mode == 1 ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<const float4*>(acc)[i];
    a.x = fmaf(nk, t.x - g.x, a.x); a.y = fmaf(nk, t.y - g.y, a.y);
    a.z = fmaf(nk, t.z - g.z, a.z); a.w = fmaf(nk, t.w - g.w, a.w);
    reinterpret_cast<float4*>(acc)[i] = a;
    if (reset) {
      reinterpret_cast<float4*>(theta)[i] = g;
      if (wb != nullptr) reinterpret_cast<uint2*>(wb)[i] = make_uint2(pack_bf16x2(g.x, g.y), pack_bf16x2(g.z, g.w));
      if (mom != nullptr && (i << 2) < n_mom) reinterpret_cast<float4*>(mom)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// ------------------------------------------------------------------ SCAFFOLD control variates (n = the parameters)
// Before client i trains: corr = c - c_i (the correction its SGD steps add to the gradient).
__global__ void __launch_bounds__(EW_THREADS)
scaffold_corr_kernel(float* __restrict__ corr, const float* __restrict__ c, const float* __restrict__ ci, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(c)[i], b = reinterpret_cast<const float4*>(ci)[i];
    reinterpret_cast<float4*>(corr)[i] = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
  }
}

// After client i trained K steps at lr eta (option II of the paper): dc = (global - theta) * inv_k_eta - c with
// inv_k_eta = 1 / (K eta); c_i += dc; and the rank's upload of the control-variate segment up = dc (first hosted
// client of the round) or up += dc (later ones).  Runs before the logical-client fold resets theta.
__global__ void __launch_bounds__(EW_THREADS)
scaffold_dc_kernel(float* __restrict__ up, float* __restrict__ ci, const float* __restrict__ c,
                   const float* __restrict__ global_w, const float* __restrict__ theta, long long n, float inv_k_eta,
                   int first) {
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 g = reinterpret_cast<const float4*>(global_w)[i], t = reinterpret_cast<const float4*>(theta)[i];
    const float4 cv = reinterpret_cast<const float4*>(c)[i];
    const float4 d = make_float4(fmaf(g.x - t.x, inv_k_eta, -cv.x), fmaf(g.y - t.y, inv_k_eta, -cv.y),
                                 fmaf(g.z - t.z, inv_k_eta, -cv.z), fmaf(g.w - t.w, inv_k_eta, -cv.w));
    float4 a = reinterpret_cast<const float4*>(ci)[i];
    a.x += d.x; a.y += d.y; a.z += d.z; a.w += d.w;
    reinterpret_cast<float4*>(ci)[i] = a;
    float4 u = d;
    if (!first) {
      const float4 p = reinterpret_cast<const float4*>(up)[i];
      u.x += p.x; u.y += p.y; u.z += p.z; u.w += p.w;
    }
    reinterpret_cast<float4*>(up)[i] = u;
  }
}

// ------------------------------------------------------------------ multi-source weighted sum
struct WsumArgs {
  const void* src[B200_MAX_RANKS];
  float w[B200_MAX_RANKS];
  int n_src;
};
template <bool BF16>
__global__ void __launch_bounds__(EW_THREADS) weighted_sum_kernel(void* __restrict__ dst, WsumArgs a, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int VEC = BF16 ? 8 : 4;
  const long long nv = n / VEC;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
    for (int k = 0; k < a.n_src; ++k) {
      const uint4 u = reinterpret_cast<const uint4*>(a.src[k])[i];
      const float wk = a.w[k];
      if constexpr (BF16) {
        const float2 p0 = unpack_bf16x2(u.x), p1 = unpack_bf16x2(u.y), p2 = unpack_bf16x2(u.z), p3 = unpack_bf16x2(u.w);
        acc[0] = fmaf(wk, p0.x, acc[0]); acc[1] = fmaf(wk, p0.y, acc[1]);
        acc[2] = fmaf(wk, p1.x, acc[2]); acc[3] = fmaf(wk, p1.y, acc[3]);
        acc[4] = fmaf(wk, p2.x, acc[4]); acc[5] = fmaf(wk, p2.y, acc[5]);
        acc[6] = fmaf(wk, p3.x, acc[6]); acc[7] = fmaf(wk, p3.y, acc[7]);
      } else {
        acc[0] = fmaf(wk, __uint_as_float(u.x), acc[0]); acc[1] = fmaf(wk, __uint_as_float(u.y), acc[1]);
        acc[2] = fmaf(wk, __uint_as_float(u.z), acc[2]); acc[3] = fmaf(wk, __uint_as_float(u.w), acc[3]);
      }
    }
    uint4 o;
    if constexpr (BF16) {
      o = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                     pack_bf16x2(acc[6], acc[7]));
    } else {
      o = make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3]));
    }
    reinterpret_cast<uint4*>(dst)[i] = o;
  }
  if (blockIdx.x == 0) {
    for (long long i = nv * VEC + threadIdx.x; i < n; i += blockDim.x) {
      float acc = 0.f;
      for (int k = 0; k < a.n_src; ++k) {
        const float v = BF16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.src[k])[i])
                             : reinterpret_cast<const float*>(a.src[k])[i];
        acc = fmaf(a.w[k], v, acc);
      }
      if (BF16)
        reinterpret_cast<__nv_bfloat16*>(dst)[i] = __float2bfloat16_rn(acc);
      else
        reinterpret_cast<float*>(dst)[i] = acc;
    }
  }
}

// ------------------------------------------------------------------ casts
__global__ void __launch_bounds__(EW_THREADS) cast_f32_bf16_kernel(const float* __restrict__ s,
                                                                    __nv_bfloat16* __restrict__ d, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(s)[i];
    reinterpret_cast<uint2*>(d)[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0)
    for (long long i = (nv << 2) + threadIdx.x; i < n; i += blockDim.x) d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void __launch_bounds__(EW_THREADS) cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ s,
                                                                    float* __restrict__ d, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint2 u = reinterpret_cast<const uint2*>(s)[i];
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
    reinterpret_cast<float4*>(d)[i] = make_float4(a.x, a.y, b.x, b.y);
  }
  if (blockIdx.x == 0)
    for (long long i = (nv << 2) + threadIdx.x; i < n; i += blockDim.x) d[i] = __bfloat162float(s[i]);
}

// ------------------------------------------------------------------ batch gather (X[idx]) on a resident shard
__global__ void __launch_bounds__(EW_THREADS)
gather_rows_kernel(const uint4* __restrict__ src, const long long* __restrict__ idx, uint4* __restrict__ dst,
                   long long n_rows, int row_vecs) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = n_rows * row_vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / row_vecs;
    const int c = static_cast<int>(i - r * row_vecs);
    dst[i] = __ldg(src + idx[r] * row_vecs + c);
  }
}
// ------------------------------------------------------------------ augmenting batch gather (random crop + flip)
// dst[s] = augment(src[idx[s]]) for NHWC images.  Output position p = s0 + s draws from ONE Philox4x32-10 output,
// counter (p, epoch, stream_lo, stream_hi), key `key`: oy = x.x % (2 pad + 1), ox = x.y % (2 pad + 1) (0 without
// crop), flip = x.z & 1 (0 without flip); out[h, w] = src[h + oy - pad, w' + ox - pad] (w' = W - 1 - w when flipped),
// 0 outside the image.  The per-epoch words {epoch, stream_lo, stream_hi} are read from device memory so a replayed
// graph picks up a new epoch without a recapture.
//
// One work item = a tile of up to `rows_per_tile` output rows of one image.  Its source rows are one contiguous byte
// range (the crop shifts rows as a whole), which the CTA stages into shared memory with V-byte vector loads; each
// thread then composes V output bytes from single-element shared-memory reads (the pixel order is reversed and
// shifted by a non-vector amount) and writes them with one V-byte store.  Global traffic is V-byte vectors only.
template <int N> struct AugVec;
template <> struct AugVec<2> { using T = uint16_t; };
template <> struct AugVec<4> { using T = uint32_t; };
template <> struct AugVec<8> { using T = uint2; };
template <> struct AugVec<16> { using T = uint4; };

constexpr int AUG_THREADS = 256;
constexpr int AUG_TILE_BYTES = 8192;    // shared memory per work item (more when one image row is larger)
constexpr int AUG_MAX_ROW_BYTES = 48 * 1024;   // one image row must fit the default dynamic shared memory

template <int ES, int V>
__global__ void __launch_bounds__(AUG_THREADS)
gather_augment_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ idx, uint8_t* __restrict__ dst,
                      const uint32_t* __restrict__ words, long long n_rows, long long s0, uint2 key, int pad,
                      int crop, int flip, int H, int W, int C, int rows_per_tile) {
  using E = typename AugVec<ES>::T;
  using Vt = typename AugVec<V>::T;
  constexpr int EPV = V / ES;
  extern __shared__ uint4 aug_smem[];
  const E* se = reinterpret_cast<const E*>(aug_smem);
  griddep_launch_dependents();
  griddep_wait();
  const uint32_t epoch = words[0], st_lo = words[1], st_hi = words[2];
  const int row_e = W * C;
  const long long row_bytes = static_cast<long long>(row_e) * ES, img_bytes = row_bytes * H;
  const int tiles = (H + rows_per_tile - 1) / rows_per_tile;
  const int items = static_cast<int>(n_rows) * tiles;     // < 2^31 (checked at launch)
  const uint32_t span = 2u * static_cast<uint32_t>(pad) + 1u;
  for (int it = blockIdx.x; it < items; it += gridDim.x) {
    const int s = it / tiles;
    const int h0 = (it - s * tiles) * rows_per_tile;
    const int hn = min(rows_per_tile, H - h0);
    const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>(s0 + s), epoch, st_lo, st_hi), key);
    const int dy = crop ? static_cast<int>(x.x % span) - pad : 0;
    const int dx = crop ? static_cast<int>(x.y % span) - pad : 0;
    const bool fl = flip && (x.z & 1u);
    const int lo = max(0, h0 + dy), hi = min(H, h0 + hn + dy);    // source rows this tile reads
    if (hi > lo) {
      const Vt* g = reinterpret_cast<const Vt*>(src + idx[s] * img_bytes + lo * row_bytes);
      Vt* d = reinterpret_cast<Vt*>(aug_smem);
      const int nv = static_cast<int>((hi - lo) * row_bytes / V);
      for (int i = threadIdx.x; i < nv; i += AUG_THREADS) d[i] = __ldg(g + i);
    }
    __syncthreads();
    Vt* out = reinterpret_cast<Vt*>(dst + static_cast<long long>(s) * img_bytes + h0 * row_bytes);
    const int out_v = static_cast<int>(hn * row_bytes / V);
    for (int i = threadIdx.x; i < out_v; i += AUG_THREADS) {
      const int e = i * EPV;
      int r = e / row_e;
      int w = (e - r * row_e) / C;
      int c = e - r * row_e - w * C;
      uint32_t wd[(V + 3) / 4] = {};     // the output vector as 32-bit words (kept in registers)
#pragma unroll
      for (int k = 0; k < EPV; ++k) {
        const int sh = h0 + r + dy, sw = (fl ? W - 1 - w : w) + dx;
        const uint32_t val = (sh >= lo && sh < hi && sw >= 0 && sw < W) ? se[(sh - lo) * row_e + sw * C + c] : 0u;
        wd[k * ES / 4] |= val << (8 * ((k * ES) & 3));
        if (++c == C) {
          c = 0;
          if (++w == W) { w = 0; ++r; }
        }
      }
      if constexpr (V == 16) out[i] = make_uint4(wd[0], wd[1], wd[2], wd[3]);
      else if constexpr (V == 8) out[i] = make_uint2(wd[0], wd[1]);
      else out[i] = static_cast<Vt>(wd[0]);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ mixing batch gather (mixup / CutMix)
// gather_augment_kernel, then each output image mixed with its batch partner (torchvision's batch.roll(1, 0)): within
// the batch of `batch` positions holding s (the call covers whole batches, s0 % batch == 0; the last may be ragged, of L
// rows), row j pairs with (j - 1 + L) % L.  Both images are augmented with their own draws first.  The batch's mix row
// rows[(s0 + s) / batch] (data/mix.py) holds lam, lam1 (fp32 bits), the kind and the box y0, y1, x0, x1:
//   mixup:  out = round(fp32(fp32(a lam) + fp32(b lam1)))   (mul_rn / add_rn: no contracted FMA)
//   CutMix: out = b inside the box, a outside (data movement only)
// A work item stages its own and its partner's source rows into two halves of shared memory (the partner's only when
// the tile meets the box, for CutMix), then composes as gather_augment_kernel does.
constexpr int MIX_ROW = 8;
constexpr int MIX_CUTMIX = 1;

template <int ES>
__device__ __forceinline__ uint32_t mix_elem(uint32_t a, uint32_t b, float lam, float lam1, int fp16) {
  if constexpr (ES == 4) {
    return __float_as_uint(add_rn(mul_rn(__uint_as_float(a), lam), mul_rn(__uint_as_float(b), lam1)));
  } else {
    if (fp16) {
      const float f = add_rn(mul_rn(__half2float(__ushort_as_half(static_cast<unsigned short>(a))), lam),
                                mul_rn(__half2float(__ushort_as_half(static_cast<unsigned short>(b))), lam1));
      return __half_as_ushort(__float2half_rn(f));
    }
    const float f = add_rn(mul_rn(__bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(a))), lam),
                              mul_rn(__bfloat162float(__ushort_as_bfloat16(static_cast<unsigned short>(b))), lam1));
    return __bfloat16_as_ushort(__float2bfloat16_rn(f));
  }
}

template <int ES, int V>
__global__ void __launch_bounds__(AUG_THREADS)
gather_mix_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ idx, uint8_t* __restrict__ dst,
                  const uint32_t* __restrict__ words, const int* __restrict__ mix_rows, long long n_rows, long long s0,
                  int batch, uint2 key, int pad, int crop, int flip, int fp16, int H, int W, int C, int rows_per_tile,
                  int half_bytes) {
  using E = typename AugVec<ES>::T;
  using Vt = typename AugVec<V>::T;
  constexpr int EPV = V / ES;
  extern __shared__ uint4 aug_smem[];
  const E* sa = reinterpret_cast<const E*>(aug_smem);
  const E* sb = reinterpret_cast<const E*>(reinterpret_cast<const uint8_t*>(aug_smem) + half_bytes);
  griddep_launch_dependents();
  griddep_wait();
  const uint32_t epoch = words[0], st_lo = words[1], st_hi = words[2];
  const int row_e = W * C;
  const long long row_bytes = static_cast<long long>(row_e) * ES, img_bytes = row_bytes * H;
  const int tiles = (H + rows_per_tile - 1) / rows_per_tile;
  const int items = static_cast<int>(n_rows) * tiles;     // < 2^31 (checked at launch)
  const uint32_t span = 2u * static_cast<uint32_t>(pad) + 1u;
  for (int it = blockIdx.x; it < items; it += gridDim.x) {
    const int s = it / tiles;
    const int h0 = (it - s * tiles) * rows_per_tile;
    const int hn = min(rows_per_tile, H - h0);
    const int b0 = s / batch * batch;                       // first row of s's batch in this call
    const int L = static_cast<int>(min(static_cast<long long>(batch), n_rows - b0));
    const int sp = b0 + (s == b0 ? L - 1 : s - b0 - 1);     // the partner
    const int* mr = mix_rows + (s0 + s) / batch * MIX_ROW;
    const float lam = __int_as_float(mr[0]), lam1 = __int_as_float(mr[1]);
    const bool cut = mr[2] == MIX_CUTMIX;
    const int y0 = mr[3], y1 = mr[4], x0 = mr[5], x1 = mr[6];
    const bool need_b = !cut || (y0 < h0 + hn && y1 > h0 && x1 > x0);
    const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>(s0 + s), epoch, st_lo, st_hi), key);
    const uint4 xp = philox4x32_10(make_uint4(static_cast<uint32_t>(s0 + sp), epoch, st_lo, st_hi), key);
    const int dy = crop ? static_cast<int>(x.x % span) - pad : 0;
    const int dx = crop ? static_cast<int>(x.y % span) - pad : 0;
    const bool fl = flip && (x.z & 1u);
    const int dyb = crop ? static_cast<int>(xp.x % span) - pad : 0;
    const int dxb = crop ? static_cast<int>(xp.y % span) - pad : 0;
    const bool flb = flip && (xp.z & 1u);
    const int lo = max(0, h0 + dy), hi = min(H, h0 + hn + dy);        // source rows of the own image
    const int lob = max(0, h0 + dyb), hib = min(H, h0 + hn + dyb);    // and of the partner
    if (hi > lo) {
      const Vt* g = reinterpret_cast<const Vt*>(src + idx[s] * img_bytes + lo * row_bytes);
      Vt* d = reinterpret_cast<Vt*>(aug_smem);
      const int nv = static_cast<int>((hi - lo) * row_bytes / V);
      for (int i = threadIdx.x; i < nv; i += AUG_THREADS) d[i] = __ldg(g + i);
    }
    if (need_b && hib > lob) {
      const Vt* g = reinterpret_cast<const Vt*>(src + idx[sp] * img_bytes + lob * row_bytes);
      Vt* d = reinterpret_cast<Vt*>(reinterpret_cast<uint8_t*>(aug_smem) + half_bytes);
      const int nv = static_cast<int>((hib - lob) * row_bytes / V);
      for (int i = threadIdx.x; i < nv; i += AUG_THREADS) d[i] = __ldg(g + i);
    }
    __syncthreads();
    Vt* out = reinterpret_cast<Vt*>(dst + static_cast<long long>(s) * img_bytes + h0 * row_bytes);
    const int out_v = static_cast<int>(hn * row_bytes / V);
    for (int i = threadIdx.x; i < out_v; i += AUG_THREADS) {
      const int e = i * EPV;
      int r = e / row_e;
      int w = (e - r * row_e) / C;
      int c = e - r * row_e - w * C;
      uint32_t wd[(V + 3) / 4] = {};
#pragma unroll
      for (int k = 0; k < EPV; ++k) {
        const int oh = h0 + r;
        const int sh = oh + dy, sw = (fl ? W - 1 - w : w) + dx;
        uint32_t val = (sh >= lo && sh < hi && sw >= 0 && sw < W) ? static_cast<uint32_t>(sa[(sh - lo) * row_e + sw * C + c]) : 0u;
        if (need_b && (!cut || (oh >= y0 && oh < y1 && w >= x0 && w < x1))) {
          const int shb = oh + dyb, swb = (flb ? W - 1 - w : w) + dxb;
          const uint32_t vb =
              (shb >= lob && shb < hib && swb >= 0 && swb < W) ? static_cast<uint32_t>(sb[(shb - lob) * row_e + swb * C + c]) : 0u;
          val = cut ? vb : mix_elem<ES>(val, vb, lam, lam1, fp16);
        }
        wd[k * ES / 4] |= val << (8 * ((k * ES) & 3));
        if (++c == C) {
          c = 0;
          if (++w == W) { w = 0; ++r; }
        }
      }
      if constexpr (V == 16) out[i] = make_uint4(wd[0], wd[1], wd[2], wd[3]);
      else if constexpr (V == 8) out[i] = make_uint2(wd[0], wd[1]);
      else out[i] = static_cast<Vt>(wd[0]);
    }
    __syncthreads();
  }
}

__global__ void gather_i64_kernel(const long long* __restrict__ src, const long long* __restrict__ idx,
                                  long long* __restrict__ dst, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = src[idx[i]];
}

// ------------------------------------------------------------------ column sum of a bf16 [rows, cols] matrix
// (bias gradient).  Block = 32 x 8: 32 consecutive columns, 8 row lanes; grid.x over column groups,
// grid.y over row chunks; partial sums are combined with fp32 atomics.
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, long long rows, int cols) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  float acc = 0.f;
  if (c < cols)
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + ty; r < rows; r += static_cast<long long>(gridDim.y) * 8)
      acc += __bfloat162float(x[r * cols + c]);
  s[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += s[j][tx];
    atomicAdd(out + c, t);
  }
}

// 16-byte version (cols % 8 == 0): block = 32 column groups (256 columns) x 8 row lanes, 4 rows in flight per
// thread; grid.x over column chunks, grid.y over row chunks
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const uint4* __restrict__ x, float* __restrict__ out, long long rows, int cols8, int rows_per_cta) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s[8][32][9];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int cg = blockIdx.x * 32 + tx;
  const long long r0 = static_cast<long long>(blockIdx.y) * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  if (r1 > rows) r1 = rows;
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (cg < cols8) {
    for (long long r = r0 + ty; r < r1; r += 32) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r + 8 * u < r1) v[u] = __ldcs(x + (r + 8 * u) * cols8 + cg);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r + 8 * u < r1) {
          const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = unpack_bf16x2(w[j]);
            a[2 * j] += f.x;
            a[2 * j + 1] += f.y;
          }
        }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s[ty][tx][j] = a[j];
  __syncthreads();
  // 256 threads -> 256 columns of this chunk
  const int col = threadIdx.x, g = col >> 3, j = col & 7;
  if (blockIdx.x * 32 + g < cols8) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += s[y][g][j];
    atomicAdd(out + (static_cast<long long>(blockIdx.x) * 32 + g) * 8 + j, t);
  }
}

// ------------------------------------------------------------------ small bf16 elementwise ops
__global__ void __launch_bounds__(EW_THREADS)
add_bf16_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ o, long long nv, int relu) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 x = a[i], y = b[i];
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
    uint32_t r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 p = unpack_bf16x2(xs[j]), q = unpack_bf16x2(ys[j]);
      float u = p.x + q.x, v = p.y + q.y;
      if (relu) { u = fmaxf(u, 0.f); v = fmaxf(v, 0.f); }
      r[j] = pack_bf16x2(u, v);
    }
    o[i] = make_uint4(r[0], r[1], r[2], r[3]);
  }
}
// dx = dy * (y > 0)
__global__ void __launch_bounds__(EW_THREADS)
relu_bwd_kernel(const uint4* __restrict__ y, const uint4* __restrict__ dy, uint4* __restrict__ dx, long long nv) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 a = y[i], b = dy[i];
    const uint32_t as[4] = {a.x, a.y, a.z, a.w}, bs[4] = {b.x, b.y, b.z, b.w};
    uint32_t r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 p = unpack_bf16x2(as[j]), q = unpack_bf16x2(bs[j]);
      r[j] = pack_bf16x2(p.x > 0.f ? q.x : 0.f, p.y > 0.f ? q.y : 0.f);
    }
    dx[i] = make_uint4(r[0], r[1], r[2], r[3]);
  }
}
__device__ __forceinline__ float gelu_f(float v) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * v * (1.f + tanhf(k0 * (v + k1 * v * v * v)));
}
__device__ __forceinline__ float gelu_grad_f(float v) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (v + k1 * v * v * v);
  const float t = tanhf(u);
  return 0.5f * (1.f + t) + 0.5f * v * (1.f - t * t) * k0 * (1.f + 3.f * k1 * v * v);
}
__global__ void __launch_bounds__(EW_THREADS)
gelu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __float2bfloat16_rn(gelu_f(__bfloat162float(x[i])));
}
__global__ void __launch_bounds__(EW_THREADS)
gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                __nv_bfloat16* __restrict__ dx, long long n) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dx[i] = __float2bfloat16_rn(__bfloat162float(dy[i]) * gelu_grad_f(__bfloat162float(x[i])));
}
// 16-byte versions (n % 8 == 0, aligned): 8 elements per thread, streaming loads
__global__ void __launch_bounds__(EW_THREADS)
gelu_vec_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long nv) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 u = __ldcs(x + i);
    const uint32_t in[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = unpack_bf16x2(in[j]);
      o[j] = pack_bf16x2(gelu_f(v.x), gelu_f(v.y));
    }
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
__global__ void __launch_bounds__(EW_THREADS)
gelu_bwd_vec_kernel(const uint4* __restrict__ x, const uint4* __restrict__ dy, uint4* __restrict__ dx, long long nv) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 u = __ldcs(x + i), g = __ldcs(dy + i);
    const uint32_t xs[4] = {u.x, u.y, u.z, u.w}, gs[4] = {g.x, g.y, g.z, g.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = unpack_bf16x2(xs[j]), d = unpack_bf16x2(gs[j]);
      o[j] = pack_bf16x2(d.x * gelu_grad_f(v.x), d.y * gelu_grad_f(v.y));
    }
    dx[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
// exact GELU, x Phi(x) (torch.nn.GELU() / approximate="none"), and its derivative Phi(x) + x phi(x)
__device__ __forceinline__ float gelu_erf_f(float v) { return 0.5f * v * (1.f + erff(v * 0.7071067811865476f)); }
__device__ __forceinline__ float gelu_erf_grad_f(float v) {
  return 0.5f * (1.f + erff(v * 0.7071067811865476f)) + v * 0.3989422804014327f * expf(-0.5f * v * v);
}
__global__ void __launch_bounds__(EW_THREADS)
gelu_erf_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long nv) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v[8];
    unpack8(__ldcs(x + i), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = gelu_erf_f(v[j]);
    y[i] = pack8(v);
  }
}
__global__ void __launch_bounds__(EW_THREADS)
gelu_erf_bwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ dy, uint4* __restrict__ dx, long long nv) {
  griddep_launch_dependents();
  griddep_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v[8], g[8];
    unpack8(__ldcs(x + i), v);
    unpack8(__ldcs(dy + i), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= gelu_erf_grad_f(v[j]);
    dx[i] = pack8(g);
  }
}

// dst[r, 0:kp] = src[r, 0:k] zero padded (weights whose K is not a multiple of 8, e.g. 7x7x3 = 147)
__global__ void __launch_bounds__(EW_THREADS)
pad_rows_kernel(const __nv_bfloat16* __restrict__ s, __nv_bfloat16* __restrict__ d, long long rows, int k, int kp,
                const uint32_t* __restrict__ flags, const uint32_t* __restrict__ epoch_word, long long elem_off, int granule) {
  // gated mode: do NOT let the dependent GEMM become resident early -- its large CTAs would sit on the SMs while this
  // kernel spins, and the collective that publishes the flags might be the one still waiting for those SMs
  if (flags == nullptr) griddep_launch_dependents();
  griddep_wait();
  if (flags != nullptr) {
    // bcast_gemm staging: the source is a slice of the bf16 arena that the FedAvg collective may still be writing on
    // another stream -- acquire the arrival flags of the granules under it first (bounded spin)
    if (threadIdx.x == 0) {
      const uint32_t need = *reinterpret_cast<const volatile uint32_t*>(epoch_word);
      for (long long t = elem_off / granule; t <= (elem_off + rows * k - 1) / granule; ++t) {
        unsigned long long spins = 0;
        while (static_cast<int32_t>(ld_acquire_sys(flags + t) - need) < 0)
          if (++spins > (1ull << 26)) break;
      }
    }
    __syncthreads();
  }
  const long long total = rows * kp;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / kp;
    const int c = static_cast<int>(i - r * kp);
    d[i] = c < k ? s[r * k + c] : __float2bfloat16_rn(0.f);
  }
}

// embedding backward: grad_table[idx[r], :] += dy[r, :]  (fp32 atomics; rows of 8-element vectors)
__global__ void __launch_bounds__(EW_THREADS)
embedding_bwd_kernel(const uint4* __restrict__ dy, const long long* __restrict__ idx, float* __restrict__ grad,
                     long long n_rows, int row_vecs) {
  griddep_launch_dependents();
  griddep_wait();
  const long long total = n_rows * row_vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / row_vecs;
    const int c = static_cast<int>(i - r * row_vecs);
    const uint4 v = dy[i];
    float* g = grad + (idx[r] * row_vecs + c) * 8;
    const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), cc = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g), "f"(a.x), "f"(a.y), "f"(b.x), "f"(b.y) : "memory");
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g + 4), "f"(cc.x), "f"(cc.y), "f"(d.x), "f"(d.y) : "memory");
  }
}

}  // namespace b200

using namespace b200;
#define RET_LAST() return static_cast<int>(cudaGetLastError())

extern "C" int b200_fused_sgd(float* w, float* g, float* mom, void* w_bf16, long long n, const float* hyper,
                              int zero_grad, int nesterov, const unsigned long long* wire_slot,
                              const float* pack_global, const float* pack_scale, long long n_pack, int wire_fp32,
                              const float* prox_anchor, const float* corr, float* adam_v, int clip,
                              cudaStream_t stream) {
  if (n <= 0) return 0;
  SgdPack pk;
  pk.wire_slot = wire_slot; pk.global_w = pack_global; pk.scale = pack_scale;
  pk.n_pack = n_pack > n ? n_pack : n; pk.wire_fp32 = wire_fp32;
  if (wire_slot != nullptr && ((n & 7) || (pk.n_pack & 7))) return -2;
  if (prox_anchor != nullptr && corr != nullptr) return -2;
  if (adam_v != nullptr && (prox_anchor != nullptr || corr != nullptr || mom == nullptr)) return -2;
  // read as float4 at the offsets of w
  if ((reinterpret_cast<uintptr_t>(prox_anchor) | reinterpret_cast<uintptr_t>(corr) |
       reinterpret_cast<uintptr_t>(adam_v)) & 15)
    return -2;
  auto kernel = clip ? (adam_v != nullptr        ? fused_sgd_kernel<false, false, true, true>
                       : prox_anchor != nullptr ? fused_sgd_kernel<true, false, false, true>
                       : corr != nullptr        ? fused_sgd_kernel<false, true, false, true>
                                                : fused_sgd_kernel<false, false, false, true>)
                     : (adam_v != nullptr        ? fused_sgd_kernel<false, false, true>
                       : prox_anchor != nullptr ? fused_sgd_kernel<true>
                       : corr != nullptr        ? fused_sgd_kernel<false, true>
                                                : fused_sgd_kernel<false>);
  launch_pdl(kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, w, g, mom, reinterpret_cast<__nv_bfloat16*>(w_bf16), n,
             hyper, zero_grad, nesterov, pk,
             adam_v != nullptr ? adam_v : prox_anchor != nullptr ? prox_anchor : corr);
  RET_LAST();
}
extern "C" int b200_fused_sgd_segments(float* w, float* g, float* mom, void* w_bf16, const long long* segments, int n_seg,
                                       const float* hyper, int nesterov, const float* prox_anchor, const float* corr,
                                       float* adam_v, int clip, cudaStream_t stream) {
  if (n_seg <= 0) return 0;
  if ((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(mom) |
       reinterpret_cast<uintptr_t>(prox_anchor) | reinterpret_cast<uintptr_t>(corr) |
       reinterpret_cast<uintptr_t>(adam_v)) & 15 ||
      reinterpret_cast<uintptr_t>(w_bf16) & 7)
    return -2;
  if (prox_anchor != nullptr && corr != nullptr) return -2;
  if (adam_v != nullptr && (prox_anchor != nullptr || corr != nullptr || mom == nullptr)) return -2;
  auto kernel = clip ? (adam_v != nullptr        ? fused_sgd_segments_kernel<false, false, true, true>
                       : prox_anchor != nullptr ? fused_sgd_segments_kernel<true, false, false, true>
                       : corr != nullptr        ? fused_sgd_segments_kernel<false, true, false, true>
                                                : fused_sgd_segments_kernel<false, false, false, true>)
                     : (adam_v != nullptr        ? fused_sgd_segments_kernel<false, false, true>
                       : prox_anchor != nullptr ? fused_sgd_segments_kernel<true>
                       : corr != nullptr        ? fused_sgd_segments_kernel<false, true>
                                                : fused_sgd_segments_kernel<false>);
  launch_pdl(kernel, ew_grid(n_seg * static_cast<long long>(EW_THREADS)), EW_THREADS, 0, stream, w, g, mom,
             reinterpret_cast<__nv_bfloat16*>(w_bf16), segments, n_seg, hyper, nesterov,
             adam_v != nullptr ? adam_v : prox_anchor != nullptr ? prox_anchor : corr);
  RET_LAST();
}
extern "C" int b200_grad_norm_clip(const float* g, long long n, const float* max_norm, void* work, float* norm_out,
                                   float* coef_out, cudaStream_t stream) {
  if (n < 0 || max_norm == nullptr || work == nullptr || norm_out == nullptr || coef_out == nullptr) return -2;
  if (reinterpret_cast<uintptr_t>(g) & 15) return -2;
  launch_pdl(grad_norm_clip_kernel, B200_GRAD_NORM_BLOCKS, GRAD_NORM_THREADS, 0, stream, g, n, max_norm,
             static_cast<unsigned long long*>(work), norm_out, coef_out);
  RET_LAST();
}
extern "C" int b200_scaffold_corr(float* corr, const float* c, const float* ci, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if ((n & 3) || ((reinterpret_cast<uintptr_t>(corr) | reinterpret_cast<uintptr_t>(c) |
                   reinterpret_cast<uintptr_t>(ci)) & 15))
    return -2;
  launch_pdl(scaffold_corr_kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, corr, c, ci, n);
  RET_LAST();
}
extern "C" int b200_scaffold_dc(float* up, float* ci, const float* c, const float* global_w, const float* theta,
                                long long n, float inv_k_eta, int first, cudaStream_t stream) {
  if (n <= 0) return 0;
  if ((n & 3) || ((reinterpret_cast<uintptr_t>(up) | reinterpret_cast<uintptr_t>(ci) | reinterpret_cast<uintptr_t>(c) |
                   reinterpret_cast<uintptr_t>(global_w) | reinterpret_cast<uintptr_t>(theta)) & 15))
    return -2;
  launch_pdl(scaffold_dc_kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, up, ci, c, global_w, theta, n, inv_k_eta, first);
  RET_LAST();
}
extern "C" int b200_fold_client(float* acc, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom,
                                long long n, float nk, int mode, int reset, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n & 3) return -2;
  launch_pdl(fold_client_kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, acc, theta, global_w,
             reinterpret_cast<__nv_bfloat16*>(w_bf16), mom, n_mom, n, nk, mode, reset);
  RET_LAST();
}
extern "C" int b200_weighted_sum(void* dst, const void* const* srcs, const float* weights, int n_src, long long n,
                                 int dtype, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n_src > B200_MAX_RANKS || n_src < 1) return -2;
  WsumArgs a;
  a.n_src = n_src;
  for (int k = 0; k < n_src; ++k) { a.src[k] = srcs[k]; a.w[k] = weights[k]; }
  if (dtype == 1)
    launch_pdl(weighted_sum_kernel<true>, ew_grid(n / 8), EW_THREADS, 0, stream, dst, a, n);
  else
    launch_pdl(weighted_sum_kernel<false>, ew_grid(n / 4), EW_THREADS, 0, stream, dst, a, n);
  RET_LAST();
}
extern "C" int b200_cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  launch_pdl(cast_f32_bf16_kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  RET_LAST();
}
extern "C" int b200_cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  launch_pdl(cast_bf16_f32_kernel, ew_grid(n >> 2), EW_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(src), dst, n);
  RET_LAST();
}
extern "C" int b200_gather_rows(const void* src, const long long* idx, void* dst, long long n_rows,
                                long long row_bytes, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (row_bytes % 16) return -2;
  const int rv = static_cast<int>(row_bytes / 16);
  launch_pdl(gather_rows_kernel, ew_grid(n_rows * rv), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(src), idx,
                                                                      reinterpret_cast<uint4*>(dst), n_rows, rv);
  RET_LAST();
}
template <int ES, int V>
static void launch_gather_augment(const void* src, const long long* idx, void* dst, const uint32_t* words,
                                  long long n_rows, long long s0, uint2 key, int pad, int crop, int flip, int H, int W,
                                  int C, int rows_per_tile, cudaStream_t stream) {
  const long long row_bytes = static_cast<long long>(W) * C * ES;
  const size_t smem = static_cast<size_t>((rows_per_tile * row_bytes + 15) / 16 * 16);
  const long long items = n_rows * ((H + rows_per_tile - 1) / rows_per_tile);
  const int grid = static_cast<int>(items < device_sm_count() * 8LL ? items : device_sm_count() * 8LL);
  launch_pdl(gather_augment_kernel<ES, V>, grid, AUG_THREADS, smem, stream, static_cast<const uint8_t*>(src), idx,
             static_cast<uint8_t*>(dst), words, n_rows, s0, key, pad, crop, flip, H, W, C, rows_per_tile);
}
// Vector width and rows per tile of an augmenting gather; false when the shape or the addresses are not supported.
static bool gather_augment_plan(const void* src, const void* dst, long long n_rows, int H, int W, int C, int elem_bytes,
                                int pad, int* vec, int* rows_per_tile) {
  if ((elem_bytes != 2 && elem_bytes != 4) || H < 1 || W < 1 || C < 1 || pad < 0) return false;
  const long long row_bytes = static_cast<long long>(W) * C * elem_bytes;
  if (row_bytes > AUG_MAX_ROW_BYTES || n_rows * H >= (1LL << 31)) return false;
  // widest vector dividing the row pitch and both base addresses: every staged range and output tile starts on a row
  int v = 16;
  while (v > elem_bytes && (row_bytes % v || reinterpret_cast<uintptr_t>(src) % v || reinterpret_cast<uintptr_t>(dst) % v))
    v >>= 1;
  if (row_bytes % v || reinterpret_cast<uintptr_t>(src) % v || reinterpret_cast<uintptr_t>(dst) % v) return false;
  long long r = AUG_TILE_BYTES / row_bytes;
  *vec = v;
  *rows_per_tile = static_cast<int>(r < 1 ? 1 : (r > H ? H : r));
  return true;
}
extern "C" int b200_gather_augment(const void* src, const long long* idx, void* dst, const unsigned* words,
                                   long long n_rows, long long s0, unsigned long long key, int pad, int crop, int flip,
                                   int H, int W, int C, int elem_bytes, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  int v, rows_per_tile;
  if (!gather_augment_plan(src, dst, n_rows, H, W, C, elem_bytes, pad, &v, &rows_per_tile)) return -2;
  const uint2 k = make_uint2(static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32));
  const uint32_t* w = reinterpret_cast<const uint32_t*>(words);
#define B200_AUG(ES, V)                                                                                               \
  launch_gather_augment<ES, V>(src, idx, dst, w, n_rows, s0, k, pad, crop, flip, H, W, C, rows_per_tile, stream)
  if (elem_bytes == 2) {
    if (v == 16) B200_AUG(2, 16);
    else if (v == 8) B200_AUG(2, 8);
    else if (v == 4) B200_AUG(2, 4);
    else B200_AUG(2, 2);
  } else {
    if (v == 16) B200_AUG(4, 16);
    else if (v == 8) B200_AUG(4, 8);
    else B200_AUG(4, 4);
  }
#undef B200_AUG
  RET_LAST();
}
template <int ES, int V>
static cudaError_t launch_gather_mix(const void* src, const long long* idx, void* dst, const uint32_t* words,
                                     const int* rows, long long n_rows, long long s0, int batch, uint2 key, int pad,
                                     int crop, int flip, int fp16, int H, int W, int C, int rows_per_tile,
                                     cudaStream_t stream) {
  const long long row_bytes = static_cast<long long>(W) * C * ES;
  const int half = static_cast<int>((rows_per_tile * row_bytes + 15) / 16 * 16);
  const size_t smem = 2 * static_cast<size_t>(half);
  static size_t configured = 0;              // two images of up to AUG_MAX_ROW_BYTES rows may exceed the default 48 KB
  if (smem > 48 * 1024 && smem > configured) {
    const cudaError_t e = cudaFuncSetAttribute(gather_mix_kernel<ES, V>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    configured = smem;
  }
  const long long items = n_rows * ((H + rows_per_tile - 1) / rows_per_tile);
  const int grid = static_cast<int>(items < device_sm_count() * 8LL ? items : device_sm_count() * 8LL);
  return launch_pdl(gather_mix_kernel<ES, V>, grid, AUG_THREADS, smem, stream, static_cast<const uint8_t*>(src), idx,
                    static_cast<uint8_t*>(dst), words, rows, n_rows, s0, batch, key, pad, crop, flip, fp16, H, W, C,
                    rows_per_tile, half);
}
extern "C" int b200_gather_mix(const void* src, const long long* idx, void* dst, const unsigned* words, const int* rows,
                               long long n_rows, long long s0, int batch, unsigned long long key, int pad, int crop,
                               int flip, int H, int W, int C, int elem_bytes, int fp16, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (batch < 1 || s0 < 0 || s0 % batch) return -2;
  int v, rows_per_tile;
  if (!gather_augment_plan(src, dst, n_rows, H, W, C, elem_bytes, pad, &v, &rows_per_tile)) return -2;
  const uint2 k = make_uint2(static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32));
  const uint32_t* w = reinterpret_cast<const uint32_t*>(words);
  cudaError_t e;
#define B200_MIX(ES, V)                                                                                               \
  e = launch_gather_mix<ES, V>(src, idx, dst, w, rows, n_rows, s0, batch, k, pad, crop, flip, fp16, H, W, C,           \
                               rows_per_tile, stream)
  if (elem_bytes == 2) {
    if (v == 16) B200_MIX(2, 16);
    else if (v == 8) B200_MIX(2, 8);
    else if (v == 4) B200_MIX(2, 4);
    else B200_MIX(2, 2);
  } else {
    if (v == 16) B200_MIX(4, 16);
    else if (v == 8) B200_MIX(4, 8);
    else B200_MIX(4, 4);
  }
#undef B200_MIX
  if (e != cudaSuccess) return static_cast<int>(e);
  RET_LAST();
}
extern "C" int b200_gather_rows_i64(const long long* src, const long long* idx, long long* dst, long long n,
                                    cudaStream_t stream) {
  if (n <= 0) return 0;
  launch_pdl(gather_i64_kernel, ew_grid(n, 64), EW_THREADS, 0, stream, src, idx, dst, n);
  RET_LAST();
}
extern "C" int b200_colsum(const void* x, float* out, long long rows, int cols, int accumulate, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return 0;
  if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float) * cols, stream);
  if (cols % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const int cols8 = cols / 8;
    const unsigned gx = static_cast<unsigned>((cols8 + 31) / 32);
    // ~2 waves of CTAs over the machine, at least one 32-row pass each
    long long want = (2 * device_sm_count() + gx - 1) / gx;
    long long rpc = (rows + want - 1) / want;
    rpc = (rpc + 31) / 32 * 32;
    if (rpc < 32) rpc = 32;
    dim3 gridv(gx, static_cast<unsigned>((rows + rpc - 1) / rpc));
    launch_pdl(colsum_vec_kernel, gridv, 256, 0, stream, reinterpret_cast<const uint4*>(x), out, rows, cols8,
               static_cast<int>(rpc));
    RET_LAST();
  }
  long long gy = (rows + 63) / 64;
  if (gy > 64) gy = 64;
  dim3 grid((cols + 31) / 32, static_cast<unsigned>(gy));
  launch_pdl(colsum_kernel, grid, 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), out, rows, cols);
  RET_LAST();
}
extern "C" int b200_add_bf16(const void* a, const void* b, void* out, long long n, int relu, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8) return -2;
  launch_pdl(add_bf16_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(a),
                                                             reinterpret_cast<const uint4*>(b),
                                                             reinterpret_cast<uint4*>(out), n / 8, relu);
  RET_LAST();
}
extern "C" int b200_relu_bwd_bf16(const void* y, const void* dy, void* dx, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8) return -2;
  launch_pdl(relu_bwd_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(y),
                                                             reinterpret_cast<const uint4*>(dy),
                                                             reinterpret_cast<uint4*>(dx), n / 8);
  RET_LAST();
}
extern "C" int b200_gelu_bf16(const void* x, void* y, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
    launch_pdl(gelu_vec_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(x),
               reinterpret_cast<uint4*>(y), n / 8);
    RET_LAST();
  }
  launch_pdl(gelu_kernel, ew_grid(n), EW_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                                                     reinterpret_cast<__nv_bfloat16*>(y), n);
  RET_LAST();
}
extern "C" int b200_gelu_bwd_bf16(const void* x, const void* dy, void* dx, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0) {
    launch_pdl(gelu_bwd_vec_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(x),
               reinterpret_cast<const uint4*>(dy), reinterpret_cast<uint4*>(dx), n / 8);
    RET_LAST();
  }
  launch_pdl(gelu_bwd_kernel, ew_grid(n), EW_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                                                         reinterpret_cast<const __nv_bfloat16*>(dy),
                                                         reinterpret_cast<__nv_bfloat16*>(dx), n);
  RET_LAST();
}
extern "C" int b200_gelu_erf_bf16(const void* x, void* y, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15)) return -2;
  launch_pdl(gelu_erf_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(x),
             reinterpret_cast<uint4*>(y), n / 8);
  RET_LAST();
}
extern "C" int b200_gelu_erf_bwd_bf16(const void* x, const void* dy, void* dx, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n % 8 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15))
    return -2;
  launch_pdl(gelu_erf_bwd_kernel, ew_grid(n / 8), EW_THREADS, 0, stream, reinterpret_cast<const uint4*>(x),
             reinterpret_cast<const uint4*>(dy), reinterpret_cast<uint4*>(dx), n / 8);
  RET_LAST();
}
extern "C" int b200_pad_rows_bf16(const void* src, void* dst, long long rows, int k, int kp, const uint32_t* flags,
                                  const uint32_t* epoch_word, long long elem_off, int granule, cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (flags != nullptr && (epoch_word == nullptr || granule <= 0)) return -2;
  launch_pdl(pad_rows_kernel, ew_grid(rows * kp), EW_THREADS, 0, stream, reinterpret_cast<const __nv_bfloat16*>(src),
                                                                 reinterpret_cast<__nv_bfloat16*>(dst), rows, k, kp, flags,
                                                                 epoch_word, elem_off, granule);
  RET_LAST();
}

extern "C" int b200_embedding_bwd(const void* dy, const long long* idx, float* grad, long long n_rows, int width,
                                  cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (width % 8) return -2;
  launch_pdl(embedding_bwd_kernel, ew_grid(n_rows * (width / 8)), EW_THREADS, 0, stream,
             reinterpret_cast<const uint4*>(dy), idx, grad, n_rows, width / 8);
  RET_LAST();
}

B200_TRACE_REGISTER(elementwise)
