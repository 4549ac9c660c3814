// The SGD update of one parameter element, shared by the arena optimizer (elementwise.cu) and the optimizer epilogue of
// the weight-gradient GEMM (gemm_wgmma.cu).  Both must produce the same bits from the same gradient, so the arithmetic
// lives here once:
//     g' = g + wd*w ;  m = mu*m + (1-damp)*g' ;  step = nesterov ? g' + mu*m : m ;  w -= lr*step
// (without a momentum buffer: step = g').  Hyper-parameters come from device memory so a captured CUDA graph can be
// replayed with a new lr.
#pragma once

namespace b200 {

struct SgdHyper {
  float lr, mu, wd, damp;
};

__device__ __forceinline__ SgdHyper load_sgd_hyper(const float* h) { return SgdHyper{h[0], h[1], h[2], h[3]}; }

// returns the new w; `m` is read and updated only when has_mom
__device__ __forceinline__ float sgd_update(const SgdHyper& h, float w, float g, float& m, bool has_mom, bool nesterov) {
  g = fmaf(h.wd, w, g);
  float st = g;
  if (has_mom) {
    m = fmaf(h.mu, m, (1.f - h.damp) * g);
    st = nesterov ? fmaf(h.mu, m, g) : m;
  }
  return fmaf(-h.lr, st, w);
}

__device__ __forceinline__ float4 sgd_update4(const SgdHyper& h, float4 w, float4 g, float4& m, bool has_mom,
                                              bool nesterov) {
  w.x = sgd_update(h, w.x, g.x, m.x, has_mom, nesterov);
  w.y = sgd_update(h, w.y, g.y, m.y, has_mom, nesterov);
  w.z = sgd_update(h, w.z, g.z, m.z, has_mom, nesterov);
  w.w = sgd_update(h, w.w, g.w, m.w, has_mom, nesterov);
  return w;
}

}  // namespace b200
