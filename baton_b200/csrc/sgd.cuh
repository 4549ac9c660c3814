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

}  // namespace b200
