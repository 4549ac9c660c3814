// The SGD update of one parameter element, shared by the arena optimizer (elementwise.cu) and the optimizer epilogue of
// the weight-gradient GEMM (gemm_wgmma.cu).  Both must produce the same bits from the same gradient, so the arithmetic
// lives here once:
//     g' = g + wd*w [+ prox*(w - a)] ;  m = mu*m + (1-damp)*g' ;  step = nesterov ? g' + mu*m : m ;  w -= lr*step
// (without a momentum buffer: step = g').  The bracketed term is FedProx's proximal pull toward the anchor `a`, the
// global model the round started from; only the *_prox forms add it.  The *_scaf forms instead add SCAFFOLD's
// correction c - c_i:  g' = (g + wd*w) + corr.  Hyper-parameters come from device memory so a
// captured CUDA graph can be replayed with a new lr or prox coefficient.
#pragma once

namespace b200 {

struct SgdHyper {
  float lr, mu, wd, damp;
  float prox;   // FedProx coefficient; 0 unless loaded with load_sgd_hyper_prox
};

// hyper = device float[4] {lr, momentum, weight_decay, dampening}
__device__ __forceinline__ SgdHyper load_sgd_hyper(const float* h) { return SgdHyper{h[0], h[1], h[2], h[3], 0.f}; }
// hyper = device float[5]: the four above, then the proximal coefficient.  Only callers given an anchor read h[4].
__device__ __forceinline__ SgdHyper load_sgd_hyper_prox(const float* h) {
  return SgdHyper{h[0], h[1], h[2], h[3], h[4]};
}
// Gradient-norm clipping: the coefficient g is multiplied by before the step (clip_grad_norm_), written on the device by
// the norm kernel into a spare float of the step's hyper-parameters -- hyper[SGD_HYPER_CLIP] of the SGD float[6], or
// [ADAMW_ROW_CLIP] of the AdamW row.  Only the CLIP instantiations of the arena kernels read it.
constexpr int SGD_HYPER_CLIP = 5;

// momentum and learning rate on the full gradient g' (weight decay and proximal term already added)
__device__ __forceinline__ float sgd_apply(const SgdHyper& h, float w, float g, float& m, bool has_mom, bool nesterov) {
  float st = g;
  if (has_mom) {
    m = fmaf(h.mu, m, (1.f - h.damp) * g);
    st = nesterov ? fmaf(h.mu, m, g) : m;
  }
  return fmaf(-h.lr, st, w);
}

// returns the new w; `m` is read and updated only when has_mom
__device__ __forceinline__ float sgd_update(const SgdHyper& h, float w, float g, float& m, bool has_mom, bool nesterov) {
  return sgd_apply(h, w, fmaf(h.wd, w, g), m, has_mom, nesterov);
}

// the same with the proximal term toward the anchor value `a`
__device__ __forceinline__ float sgd_update_prox(const SgdHyper& h, float w, float g, float a, float& m, bool has_mom,
                                                 bool nesterov) {
  return sgd_apply(h, w, fmaf(h.prox, w - a, fmaf(h.wd, w, g)), m, has_mom, nesterov);
}

// the same with SCAFFOLD's control-variate correction `corr` = c - c_i added to the gradient (after weight decay)
__device__ __forceinline__ float sgd_update_scaf(const SgdHyper& h, float w, float g, float corr, float& m, bool has_mom,
                                                 bool nesterov) {
  return sgd_apply(h, w, fmaf(h.wd, w, g) + corr, m, has_mom, nesterov);
}

__device__ __forceinline__ float4 sgd_update4(const SgdHyper& h, float4 w, float4 g, float4& m, bool has_mom,
                                              bool nesterov) {
  w.x = sgd_update(h, w.x, g.x, m.x, has_mom, nesterov);
  w.y = sgd_update(h, w.y, g.y, m.y, has_mom, nesterov);
  w.z = sgd_update(h, w.z, g.z, m.z, has_mom, nesterov);
  w.w = sgd_update(h, w.w, g.w, m.w, has_mom, nesterov);
  return w;
}

__device__ __forceinline__ float4 sgd_update4_prox(const SgdHyper& h, float4 w, float4 g, float4 a, float4& m,
                                                   bool has_mom, bool nesterov) {
  w.x = sgd_update_prox(h, w.x, g.x, a.x, m.x, has_mom, nesterov);
  w.y = sgd_update_prox(h, w.y, g.y, a.y, m.y, has_mom, nesterov);
  w.z = sgd_update_prox(h, w.z, g.z, a.z, m.z, has_mom, nesterov);
  w.w = sgd_update_prox(h, w.w, g.w, a.w, m.w, has_mom, nesterov);
  return w;
}

__device__ __forceinline__ float4 sgd_update4_scaf(const SgdHyper& h, float4 w, float4 g, float4 c, float4& m,
                                                   bool has_mom, bool nesterov) {
  w.x = sgd_update_scaf(h, w.x, g.x, c.x, m.x, has_mom, nesterov);
  w.y = sgd_update_scaf(h, w.y, g.y, c.y, m.y, has_mom, nesterov);
  w.z = sgd_update_scaf(h, w.z, g.z, c.z, m.z, has_mom, nesterov);
  w.w = sgd_update_scaf(h, w.w, g.w, c.w, m.w, has_mom, nesterov);
  return w;
}

// ------------------------------------------------------------------ AdamW (torch.optim.AdamW, one parameter group)
//     w = w * (1 - lr*wd) ;  m = b1*m + (1-b1)*g ;  v = b2*v + (1-b2)*g^2 ;
//     w -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps)
// The coefficients of local step t come as ONE row of device floats (ADAMW_ROW), written by the host in fp64 and rounded
// once: every kernel of a step reads the same row, so all three optimizer sites see the same fp32 coefficients, and a
// captured epoch reads its step's row at replay (the host refreshes the rows between replays).  At t == 1 (`first`) the
// stored m and v are ignored -- the state of a fresh optimizer -- so a new round, the next logical client and the
// captured warm-up steps need no reset pass.  The operations are the IEEE-rounded intrinsics so that fast-math builds
// cannot contract them differently at the three sites.
constexpr int ADAMW_ROW = 12;   // floats per step row (48 B): the fields of AdamHyper, then padding
constexpr int ADAMW_ROW_CLIP = 9;   // the clip coefficient of a clipped step (padding otherwise)

struct AdamHyper {
  float decay;          // 1 - lr*wd
  float b1, omb1;       // beta1, 1 - beta1
  float b2, omb2;       // beta2, 1 - beta2
  float eps;
  float step;           // lr / (1 - beta1^t)
  float inv_bc2;        // 1 / sqrt(1 - beta2^t)
  bool first;           // t == 1
};

__device__ __forceinline__ AdamHyper load_adam_hyper(const float* r) {
  return AdamHyper{r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], r[8] != 0.f};
}

// returns the new w; m and v are read (unless h.first) and updated
__device__ __forceinline__ float adamw_update(const AdamHyper& h, float w, float g, float& m, float& v) {
  const float m0 = h.first ? 0.f : m, v0 = h.first ? 0.f : v;
  m = fmaf(h.b1, m0, __fmul_rn(h.omb1, g));
  v = fmaf(h.b2, v0, __fmul_rn(__fmul_rn(h.omb2, g), g));
  const float denom = fmaf(__fsqrt_rn(v), h.inv_bc2, h.eps);
  return fmaf(-h.step, __fdiv_rn(m, denom), __fmul_rn(w, h.decay));
}

__device__ __forceinline__ float4 adamw_update4(const AdamHyper& h, float4 w, float4 g, float4& m, float4& v) {
  w.x = adamw_update(h, w.x, g.x, m.x, v.x);
  w.y = adamw_update(h, w.y, g.y, m.y, v.y);
  w.z = adamw_update(h, w.z, g.z, m.z, v.z);
  w.w = adamw_update(h, w.w, g.w, m.w, v.w);
  return w;
}

}  // namespace b200
